"""sfmrecon's k2/k4 radial undistortion (mve::image::image_undistort_k2k4<uint8_t>) against the reference's results in
tests/golden/undistort_ref.npz (every byte of small images; digest, shape and a sample of large ones), without a GPU:
the NumPy restatement, and the per-pixel function of the device kernel (mve_b200/csrc/undistort.cuh) compiled by g++.  Also the argument checks of b200mvs_set_view_distortion in a planning
context."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import undistort_reference as UR
from tests.util import ROOT

GOLD = os.path.join(ROOT, "tests", "golden", "undistort_ref.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("undistort_emu") / "libundistort_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "emu", "undistort_emu.cc"), "-o", lib])
    L = C.CDLL(lib)
    L.emu_undistort.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
    return L


def test_fixture_covers_cases(golden):
    keys = set()
    for case in UR.cases():
        keys |= set(UR.fixture_entries(case, np.zeros((case[2], case[1], case[3]), np.uint8)))
    assert keys == set(golden.files)
    assert {(c[1], c[2]) for c in UR.cases()} >= set(UR.SIZES)
    assert {c[3] for c in UR.cases()} == {1, 2, 3, 4}
    assert {c[4] for c in UR.cases()} == set(UR.FLENS)
    assert os.path.getsize(GOLD) < 200_000


def test_fixture_meets_the_borders():
    """Some source positions lie within 1e-4 px of -0.5 or w - 0.5 on both sides (a pixel left 0 and one sampled), and
    some fall in linear_at's clamp band (w - 1, w - 0.5]."""
    near_in = near_out = band = 0
    for name, w, h, c, flen, k2, k4, seed in UR.cases():
        if k2 == 0 and k4 == 0:
            continue
        ix, iy = UR.source_positions(w, h, flen, k2, k4)
        for p, n in ((ix.astype(np.float64), w), (iy.astype(np.float64), h)):
            for b in (-0.5, n - 0.5):
                near = np.abs(p - b) < 1e-4
                outside = (p < b) if b < 0 else (p > b)
                near_out += int((near & outside).sum())
                near_in += int((near & ~outside).sum())
            band += int(((p > n - 1) & (p <= n - 0.5)).sum())
    assert near_in > 0 and near_out > 0 and band > 0, (near_in, near_out, band)


def test_restatement_equals_reference(golden):
    for case in UR.cases():
        name, w, h, c, flen, k2, k4, seed = case
        UR.check(golden, case, UR.undistort_k2k4(UR.make_image(w, h, c, seed), flen, k2, k4))


def test_device_function_on_host_equals_reference(golden, emu):
    for case in UR.cases():
        name, w, h, c, flen, k2, k4, seed = case
        img = np.ascontiguousarray(UR.make_image(w, h, c, seed))
        out = np.full_like(img, 0xA5)
        emu.emu_undistort(img.ctypes.data, w, h, c, flen, k2, k4, out.ctypes.data)
        UR.check(golden, case, out)


def test_fma_emulation_is_exact():
    """fma64 / fma32 against exact rational arithmetic on random and cancelling operands."""
    from fractions import Fraction
    rng = np.random.default_rng(5)
    a = rng.normal(size=400) * np.exp2(rng.integers(-20, 20, 400))
    b = rng.normal(size=400)
    c = np.where(rng.random(400) < 0.5, -a * b, rng.normal(size=400))
    got = UR.fma64(a, b, c)
    for i in range(400):
        assert got[i] == float(Fraction(a[i]) * Fraction(b[i]) + Fraction(c[i])), i
    a32, b32, c32 = (v.astype(np.float32) for v in (a, b, c))
    got32 = UR.fma32(a32, b32, c32)
    for i in range(400):
        exact = Fraction(float(a32[i])) * Fraction(float(b32[i])) + Fraction(float(c32[i]))
        assert got32[i] == np.float32(_round_f32(exact)), i


def _round_f32(q):
    """A rational rounded to the nearest float32 (ties to even), through a float64 neighbour pair."""
    from fractions import Fraction
    d = np.float32(float(q))
    lo, hi = (d, np.nextafter(d, np.float32(np.inf))) if Fraction(float(d)) <= q else (np.nextafter(d, np.float32(-np.inf)), d)
    dl, dh = q - Fraction(float(lo)), Fraction(float(hi)) - q
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (lo.view(np.int32) & 1) == 0 else hi


def test_set_view_distortion_arguments_planning_context():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    sc = dmrecon.Scene(3, dmrecon.DEVICE_NONE)
    sc.set_view_distortion(0, 0.1, -0.02)                    # stores: no device needed
    sc.set_view_distortion(2, 0.0, 0.0)
    sc.set_view_distortion(1, -1e-7, 3.0)
    sc.set_view_distortion(1, -1e-7, 3.0)
    for vid, k2, k4 in ((-1, 0.1, 0.0), (3, 0.1, 0.0), (0, float("nan"), 0.0), (0, 0.0, float("inf")),
                        (0, float("-inf"), 0.0), (0, 0.0, float("nan"))):
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.set_view_distortion(vid, k2, k4)
        assert e.value.code == dmrecon.ERR_INVALID_ARG and "b200mvs_set_view_distortion: bad arguments" in str(e.value)
    assert L.b200mvs_set_view_distortion(None, 0, 0.1, 0.0) == dmrecon.ERR_INVALID_ARG
    # cameras and view selection are untouched by it
    cam = dict(flen=1.0, paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3, dtype=np.float32), trans=np.zeros(3, np.float32))
    sc.set_view_camera(0, 64, 48, **cam)
    sc.set_view_distortion(0, 0.3, 0.1)
    assert sc.num_levels(0) == 2
    sc.close()
