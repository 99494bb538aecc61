"""The NumPy restatement of the depth-map operations (tests/dm_reference.py) against the reference binary's own results
(tests/golden/depthmap_ops_ref.npz and depthmap_edges_ref.npz, minted through oracle/_ref/ref_harness dmops), without a
GPU: the yardstick of tests/test_gpu_depthmap_edges.py is itself checked.

Exact: confidence_clean, cleanup at every threshold, vertex ids, faces, confidences.  Vertices within 1e-6 * absmax (the
restatement repeats the reference build's float32 operations, so they agree to the bit in practice), normals p99.9
<= 1e-4 (float64 here, float32 there), scale values within 3e-5 relative."""
import hashlib

import numpy as np
import pytest

from tests import dm_reference as R
from tests.test_gpu_depthmap_edges import cleanup_cases, tri_cases
from tests.test_gpu_depthmap_ops import CLEANUP_THRES, TRI_CASES, depth_case, tri_inputs
from tests.util import golden_ref


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def check_floats(r, ref, key, color):
    pick = ref[key + "_pick"]
    vmax = float(ref[key + "_verts_absmax"])
    assert np.abs(r["vertices"][pick] - ref[key + "_verts"]).max(initial=0) <= 1e-6 * vmax
    assert np.abs(r["vertices64"][pick] - ref[key + "_verts"]).max(initial=0) <= 4 * np.finfo(np.float32).eps * vmax
    if len(pick) == 0:
        return
    dn = np.abs(r["normals"][pick] - ref[key + "_normals"]).max(-1)
    assert np.percentile(dn, 99.9) <= 1e-4, np.percentile(dn, 99.9)
    smax = max(float(ref[key + "_scales_absmax"]), 1e-30)
    assert np.abs(r["scales"][pick] - ref[key + "_scales"]).max() <= 3e-5 * smax
    if color:
        assert np.abs(r["colors"][pick] - ref[key + "_colors"]).max() <= 1e-6


@pytest.mark.parametrize("kind", ["golden", "ragged", "large"])
def test_ops_fixture_cleanup(kind):
    ref = golden_ref("depthmap_ops")
    dm, cm = depth_case(kind)
    assert sha(R.confidence_clean(dm, cm)) == str(ref["confclean_%s" % kind])
    for t in CLEANUP_THRES:
        assert sha(R.cleanup(dm, t)) == str(ref["cleanup_%s_%d" % (kind, t)]), t


@pytest.mark.parametrize("kind,dd,color", TRI_CASES)
def test_ops_fixture_pointset(kind, dd, color):
    ref = golden_ref("depthmap_ops")
    key = "tri_%s_%g_%d" % (kind, dd, int(color))
    dm, ip, ci = tri_inputs(kind, color)
    r = R.pointset(dm, ip, dd, ci, conf_iterations=4, scale_factor=2.5)
    nv, nf = (int(x) for x in ref[key + "_n"])
    assert (len(r["vertices"]), len(r["faces"])) == (nv, nf)
    sv, sf, sc = (str(x) for x in ref[key + "_sha"])
    assert sha(r["vertex_ids"]) == sv and sha(r["faces"]) == sf and sha(r["confidences"]) == sc
    check_floats(r, ref, key, color)


@pytest.mark.parametrize("name", list(cleanup_cases()))
def test_edges_fixture_cleanup(name):
    ref = golden_ref("depthmap_edges")
    dm, cm, thres = cleanup_cases()[name]
    assert list(ref["cleanup_%s_thres" % name]) == thres
    assert sha(R.confidence_clean(dm, cm)) == str(ref["confclean_%s" % name])
    for t in thres:
        assert sha(R.cleanup(dm, t)) == str(ref["cleanup_%s_%d" % (name, t)]), t


@pytest.mark.parametrize("name", list(tri_cases()))
def test_edges_fixture_pointset(name):
    ref = golden_ref("depthmap_edges")
    c = tri_cases()[name]
    key = "tri_%s" % name
    r = R.pointset(c["dm"], c["invproj"], c["dd"], c["color"], conf_iterations=4, scale_factor=c["scale"])
    nv, nf = (int(x) for x in ref[key + "_n"])
    assert (len(r["vertices"]), len(r["faces"])) == (nv, nf)
    sv, sf = (str(x) for x in ref[key + "_sha"])
    assert sha(r["vertex_ids"]) == sv and sha(r["faces"]) == sf
    for it in c["ref_iters"]:
        assert sha(R.confidences(nv, r["faces"], it, r["rings"])) == str(ref["%s_confs_%d" % (key, it)]), it
    check_floats(r, ref, key, c["color"] is not None)


def test_fma32_is_correctly_rounded():
    """fma32 against exact rational arithmetic.  The first rows are double-rounding traps: (1 + 2^-20)(1 - 2^-20) + c is
    2^-40 below a float32 half-way point, which a plain float64 sum would round onto before rounding to float32."""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    a = rng.standard_normal(3000).astype(np.float32)
    b = rng.standard_normal(3000).astype(np.float32)
    c = (rng.standard_normal(3000) * 10.0 ** rng.integers(-3, 4, 3000)).astype(np.float32)
    traps = np.float32([2.0 ** 24 + 2, -(2.0 ** 24 + 2), 2.0 ** 25 + 4, 2.0 ** 23 + 1])
    a[:4], b[:4], c[:4] = np.float32(1 + 2.0 ** -20), np.float32(1 - 2.0 ** -20), traps
    a[4:8], b[4:8], c[4:8] = np.float32(1 + 2.0 ** -20), np.float32(-(1 - 2.0 ** -20)), -traps
    got = R.fma32(a, b, c)
    assert got[0] == np.float32(2.0 ** 24 + 2) and got[1] == np.float32(-(2.0 ** 24 + 2))
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        near = np.float32(float(exact))
        cands = [np.nextafter(near, np.float32(-np.inf)), near, np.nextafter(near, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.uint32)) & 1))
        assert g == best, (x, y, z, g, best)
