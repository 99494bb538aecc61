"""The rules of a relative prior (mve_b200/csrc/prior_align.cuh, the functions k_align_observe, k_align_fit and
k_align_apply call) compiled by g++ and run on the CPU, against tests/prior_align_reference.py: the observation of a
feature bit for bit, at the map's edges and behind the camera; the fit's start and refit rules for each kind on seeded
sets, and every way it fails; and the apply bit for bit, on maps of the view's size and of other sizes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import prior_align_reference as ref
from tests.util import golden_scene

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
KINDS = (ref.DISPARITY, ref.DEPTH, ref.DEPTH_SCALE)
STATUS = {0: None, 1: "observations", 2: "MAD", 3: "inliers", 4: "singular", 5: "scale"}


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("prior_align_emu") / "libprior_align_emu.so")
    # no contraction: the device rounds every product and sum on its own (prior_align.cuh a_mul, a_add)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + EMU,
                           os.path.join(EMU, "prior_align_emu.cc"), "-o", lib])
    L = C.CDLL(lib)
    L.emu_align_observe.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_align_fit.argtypes = [C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_align_fit.restype = C.c_int
    L.emu_align_apply.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_int,
                                  C.c_int, C.c_void_p]
    return L


def _ptr(a):
    return a.ctypes.data


def _observe(L, cam, X, values, kind):
    R, t, ax, ay, cx, cy, W0, H0 = cam
    X = np.ascontiguousarray(X, np.float32)
    values = np.ascontiguousarray(values, np.float32)
    n = len(X)
    px, py, dy = np.empty(n, np.int32), np.empty(n, np.int32), np.empty((n, 2))
    Rm, tv, calib = (np.ascontiguousarray(a, np.float64) for a in (R, t, [ax, ay, cx, cy]))
    L.emu_align_observe(n, _ptr(X), _ptr(Rm), _ptr(tv), _ptr(calib), W0, H0, _ptr(values), values.shape[1],
                        values.shape[0], kind, _ptr(px), _ptr(py), _ptr(dy))
    return px, py, dy


def _fit(L, d, y, kind):
    d, y = np.ascontiguousarray(d, np.float64), np.ascontiguousarray(y, np.float64)
    out, counts = np.zeros(3), np.zeros(2, np.uint32)
    status = L.emu_align_fit(len(d), _ptr(d), _ptr(y), kind, _ptr(out), _ptr(counts))
    return status, out, counts


def _apply(L, cam, values, kind, s, t):
    _, _, ax, ay, cx, cy, W0, H0 = cam
    values = np.ascontiguousarray(values, np.float32)
    out = np.empty_like(values)
    calib = np.array([ax, ay, cx, cy])
    L.emu_align_apply(_ptr(calib), W0, H0, kind, s, t, _ptr(values), values.shape[1], values.shape[0], _ptr(out))
    return out


def _check_observe(L, cam, X, values, kind):
    px, py, dy = _observe(L, cam, X, values, kind)
    d, y, rpx, rpy = ref.observations(cam, X, values, kind)
    assert (px == rpx).all() and (py == rpy).all()
    used = dy[:, 0] > 0
    assert dy[used, 0].tobytes() == d.tobytes() and dy[used, 1].tobytes() == y.tobytes()
    return dy


def _check_fit(L, d, y, kind, pad=0):
    """The device fit of (d, y) with `pad` empty slots interleaved equals the reference's; returns the reference fit."""
    want = ref.fit(d, y, kind)
    dd, yy = np.asarray(d, np.float64), np.asarray(y, np.float64)
    if pad:
        slots = np.random.default_rng(len(d)).permutation(len(d) + pad) < len(d)
        dd, yy = np.zeros(len(slots)), np.zeros(len(slots))
        dd[slots], yy[slots] = d, y
    status, out, counts = _fit(L, dd, yy, kind)
    assert STATUS[status] == want.get("reason"), (status, want)
    assert counts[0] == want["n_obs"]
    if want["ok"]:
        assert counts[1] == want["n_inliers"]
        # t near 0 is a difference of sums of size |y|: relative to that
        np.testing.assert_allclose(out[0], want["scale"], rtol=1e-12)
        np.testing.assert_allclose(out[1], want["shift"], rtol=1e-12, atol=1e-12 * np.abs(y).max())
        np.testing.assert_allclose(out[2], want["median_rel_err"], rtol=1e-9, atol=1e-12)
    return want


def test_observations_of_a_scene(emu):
    s = golden_scene("T1")
    rng = np.random.default_rng(3)
    for v in range(min(s.n_views, 4)):
        cam = ref.camera(s, v)
        X = ref.view_features(s, v)
        assert len(X) > 16
        W0, H0 = s.size(v)
        for w, h in ((W0, H0), (W0 // 4, H0 // 4), (7, 5), (W0 * 2 + 1, H0 + 3)):
            values = rng.uniform(0.1, 3.0, (h, w)).astype(np.float32)
            values[rng.random((h, w)) < 0.1] = np.nan
            for kind in KINDS:
                _check_observe(emu, cam, X, values, kind)


def test_observations_at_edges_and_behind(emu):
    """Points whose prior pixel lies just inside and just outside each edge of the map, on the optical axis' plane and
    behind the camera."""
    R, t = np.eye(3), np.zeros(3)
    W0, H0 = 640, 480
    cam = (R, t, 500.0, 500.0, 320.0, 240.0, W0, H0)
    pts = []
    for u in (0.0, -1e-9, 639.999, 640.0, 1e-300, 320.0):
        for v in (0.0, -1e-6, 479.99, 480.0, 240.0):
            pts.append([(u - 320.0) / 500.0 * 2.0, (v - 240.0) / 500.0 * 2.0, 2.0])
    pts += [[0.0, 0.0, -1.0], [0.1, 0.1, 0.0], [0.0, 0.0, -0.0], [0.0, 0.0, 1e-30], [0.3, -0.2, 1e30]]
    X = np.array(pts, np.float32)
    for w, h in ((W0, H0), (160, 120), (1, 1), (641, 479)):
        values = np.linspace(0.5, 2.0, w * h, dtype=np.float32).reshape(h, w)
        for kind in KINDS:
            dy = _check_observe(emu, cam, X, values, kind)
            assert (dy[-5:-2, 0] == 0).all()           # behind or on the camera plane: no observation
            assert (dy[-2:, 0] > 0).all()              # just in front, on the axis: one
    # a value that is not finite and > 0 gives no observation
    values = np.full((H0, W0), np.nan, np.float32)
    for bad in (np.nan, np.inf, -np.inf, 0.0, -1.0, -0.0):
        values[:] = bad
        _, _, dy = _observe(emu, cam, X, values, ref.DEPTH)
        assert (dy == 0).all()


def _planted(rng, n, kind, s, t, outliers=0.1, noise=0.0, dither=0.0):
    """n observations of d = (y - t) / s in float32, with multiplicative Gaussian noise, an additive uniform dither and a
    share of outliers (returned as a mask)."""
    z = rng.uniform(1.0, 6.0, n)
    y = 1.0 / z if kind == ref.DISPARITY else z
    d = (y - t) / s * (1.0 + noise * rng.standard_normal(n)) + dither * rng.uniform(-1, 1, n)
    bad = rng.random(n) < outliers
    d[bad] *= rng.uniform(1.5, 4.0, bad.sum())
    return d.astype(np.float32).astype(np.float64), y, bad


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(4))
def test_fit_on_seeded_sets(emu, kind, seed):
    rng = np.random.default_rng(seed)
    s, t = (0.7, 0.0) if kind == ref.DEPTH_SCALE else ((0.2, 0.05) if kind == ref.DISPARITY else (1.7, 0.4))
    for n, noise, dither in ((16, 0.0, 0.0), (40, 0.02, 0.0), (3000, 0.02, 0.0), (20000, 0.0, 0.0), (20000, 0.0, 1e-5)):
        d, y, bad = _planted(rng, n, kind, s, t, noise=noise, dither=dither)
        want = _check_fit(emu, d, y, kind, pad=n // 3)
        if noise == 0.0 and n > 1000:
            np.testing.assert_allclose([want["scale"], want["shift"]], [s, t], rtol=1e-6, atol=1e-7)
            # Exact values differ from the model by their float32 rounding alone, which grows with d: the 3 sigma cut of
            # that near-zero spread drops the largest of them.  A uniform dither above the rounding keeps every one.
            if dither:
                assert want["ok"] and want["n_inliers"] == n - bad.sum()
            else:
                assert want["ok"] and want["n_inliers"] <= n - bad.sum()


@pytest.mark.parametrize("kind", KINDS)
def test_fit_failures(emu, kind):
    rng = np.random.default_rng(9)
    # fewer than 16 observations
    d, y, _ = _planted(rng, 15, kind, 1.0, 0.0 if kind == ref.DEPTH_SCALE else 0.1)
    assert _check_fit(emu, d, y, kind, pad=20)["reason"] == "observations"
    assert _check_fit(emu, d[:0], y[:0], kind)["reason"] == "observations"
    # MAD(d) = 0: more than half the values equal (DEPTH_SCALE has no MAD and fits)
    d, y, _ = _planted(rng, 100, kind, 1.0, 0.0, outliers=0.0)
    d[:60] = 2.0
    want = _check_fit(emu, d, y, kind)
    if kind != ref.DEPTH_SCALE:
        assert want["reason"] == "MAD"
    # s <= 0: the values fall as the target rises
    d, y, _ = _planted(rng, 200, kind, 1.0, 0.0, outliers=0.0)
    want = _check_fit(emu, d.max() + d.min() - d, y, kind)
    if kind != ref.DEPTH_SCALE:
        assert want["reason"] == "scale"
    # a constant target: s = 0
    if kind != ref.DEPTH_SCALE:
        d = rng.uniform(1, 2, 100)
        assert _check_fit(emu, d, np.full(100, 3.0), kind)["reason"] == "scale"


def test_fit_skips_non_finite_values(emu):
    """Observations come from finite values > 0 only: a map of NaN, +-inf, 0 and negative values around the planted
    ones fits as the planted ones alone do."""
    s = golden_scene("T1")
    v = 0
    cam = ref.camera(s, v)
    X = ref.view_features(s, v)
    W0, H0 = s.size(v)
    h, w = H0 // 4, W0 // 4
    ok, u, vv, z = ref.project(cam, X)
    px, py = np.floor(u * w / W0).astype(int), np.floor(vv * h / H0).astype(int)
    rng = np.random.default_rng(2)
    for kind in KINDS:
        values = np.zeros((h, w), np.float32)
        y = 1.0 / z if kind == ref.DISPARITY else z
        values[py[ok], px[ok]] = (y[ok] / 0.5).astype(np.float32)
        junk = rng.random(len(X)) < 0.3
        for k, bad in enumerate((np.nan, np.inf, -np.inf, 0.0, -2.0)):
            sel = ok & junk & (np.arange(len(X)) % 5 == k)
            values[py[sel], px[sel]] = bad
        dy = _check_observe(emu, cam, X, values, kind)
        used = dy[:, 0] > 0
        assert used.sum() < ok.sum()
        _check_fit(emu, dy[used, 0], dy[used, 1], kind)


@pytest.mark.parametrize("kind", KINDS)
def test_apply_bit_for_bit(emu, kind):
    s = golden_scene("T2")
    rng = np.random.default_rng(kind)
    for v in range(min(s.n_views, 3)):
        cam = ref.camera(s, v)
        W0, H0 = s.size(v)
        for w, h in ((W0, H0), (W0 // 4, H0 // 4), (W0 // 3 + 1, H0 // 2 - 1), (3, 2), (W0 * 2, H0 * 2)):
            values = rng.uniform(0.05, 5.0, (h, w)).astype(np.float32)
            flat = values.reshape(-1)
            idx = rng.choice(flat.size, min(flat.size, 12), replace=False)
            flat[idx] = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.0, 1e-38, 3e38, 1e-45, 7.0, 1.0, 2.0],
                                 np.float32)[:len(idx)]
            for st in ((0.3, -0.5), (1.2, 0.01), (2.0, 0.0), (1e-30, 1e-30), (1e30, 0.0)):
                sc, sh = st if kind != ref.DEPTH_SCALE else (st[0], 0.0)
                got = _apply(emu, cam, values, kind, sc, sh)
                want = ref.apply(cam, values, kind, sc, sh)
                assert got.tobytes() == want.tobytes(), (v, w, h, st)
