"""Depth-map consumers on the device (-m gpu) against the REFERENCE's own functions (libs/mve/depthmap.cc) run through
oracle/_ref/ref_harness dmops on the same buffers (golden fixture tests/golden/depthmap_ops_ref.npz, minted by
tests/golden/make_golden.py): depthmap_confidence_clean, depthmap_cleanup (bit-exact, compared by SHA-256) and
depthmap_triangulate - vertex ids, faces and vertex count exact, vertices / colours exact up to the reference binary's own
-funsafe-math contraction (<= 1e-6 relative), compared at up to 256 seeded vertices per case."""
import hashlib

import numpy as np
import pytest

from tests.util import golden_ref

pytestmark = pytest.mark.gpu
CLEANUP_THRES = (1, 7, 50, 2000)
TRI_CASES = [("golden", 5.0, True), ("ragged", 5.0, False), ("large", 0.0, True), ("large", 2.0, False)]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def depth_case(kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "golden":
        ref = golden_ref("T0")
        return np.ascontiguousarray(ref["depth_0"], np.float32), np.ascontiguousarray(ref["conf_0"], np.float32)
    h, w = (97, 131) if kind == "ragged" else (270, 480)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    d = (5.0 + 0.4 * np.sin(xx / 17.0) + 0.3 * np.cos(yy / 11.0)).astype(np.float32)
    d[(xx > w * 0.6) & (yy > h * 0.3)] += 1.5                      # a depth discontinuity
    hole = rng.random((h, w)) < (0.45 if kind == "ragged" else 0.08)   # ragged: many small islands
    d[hole] = 0.0
    d[:, :3] = 0.0
    conf = rng.random((h, w)).astype(np.float32) - 0.2
    return d, conf


def tri_inputs(kind, color):
    dm, _ = depth_case(kind, seed=3)
    h, w = dm.shape
    ax = float(max(w, h))
    invproj = np.array([1 / ax, 0, -0.5 * w / ax, 0, 1 / ax, -0.5 * h / ax, 0, 0, 1], np.float32)
    ci = np.random.default_rng(1).integers(0, 255, size=(h, w, 3), dtype=np.uint8) if color else None
    return dm, invproj, ci


@pytest.mark.parametrize("kind", ["golden", "ragged", "large"])
def test_confidence_clean_and_cleanup_bit_exact(kind):
    from mve_b200 import depthmap as D
    ref = golden_ref("depthmap_ops")
    dm, cm = depth_case(kind)
    got = dm.copy()
    D.depthmap_confidence_clean(got, cm)
    assert _sha(got) == str(ref["confclean_%s" % kind])
    for thres in CLEANUP_THRES:
        got = D.depthmap_cleanup(dm, thres)
        assert got.dtype == np.float32 and got.shape == dm.shape
        assert _sha(got) == str(ref["cleanup_%s_%d" % (kind, thres)]), thres
    # empty and full maps
    z = np.zeros((5, 7), np.float32)
    assert (D.depthmap_cleanup(z, 3) == 0).all()
    o = np.ones((5, 7), np.float32)
    assert (D.depthmap_cleanup(o, 35) == 1).all() and (D.depthmap_cleanup(o, 36) == 0).all()


@pytest.mark.parametrize("kind,dd,color", TRI_CASES)
def test_triangulate_matches_reference(kind, dd, color):
    from mve_b200 import depthmap as D
    ref = golden_ref("depthmap_ops")
    key = "tri_%s_%g_%d" % (kind, dd, int(color))
    dm, invproj, ci = tri_inputs(kind, color)
    nv, nf = (int(x) for x in ref[key + "_n"])
    sha_vids, sha_faces, sha_confs = (str(x) for x in ref[key + "_sha"])
    pick = ref[key + "_pick"]
    verts = ref[key + "_verts"]
    got = D.depthmap_triangulate(dm, invproj, dd_factor=dd, color=ci)
    assert nv > 100 and nf > 100
    # the rest of scene2pset's per-view work: vertex normals (angle-weighted), boundary confidences (exact: ring / 4), scale values
    ps = D.depthmap_pointset(dm, invproj, dd_factor=dd, color=ci, with_normals=True, conf_iterations=4, scale_factor=2.5)
    assert _sha(ps["faces"].astype(np.uint32)) == sha_faces and _sha(ps["vertex_ids"].astype(np.uint32)) == sha_vids
    cfs = ps["confidences"].astype(np.float32)
    assert _sha(cfs) == sha_confs
    assert set(np.unique(cfs)).issubset({0.0, 0.25, 0.5, 0.75, 1.0}) and (cfs == 0).any()
    assert kind == "ragged" or (cfs == 1).any()        # a ragged map may have no vertex further than 4 rings from a boundary
    dn = np.abs(ps["normals"][pick] - ref[key + "_normals"]).max(-1)
    # angle weights are acos() of float dot products (device acosf vs the host's libm): measured p99.9 3.4e-5, max 6.7e-5
    assert np.percentile(dn, 99.9) <= 1e-4 and dn.max() <= 2e-3, (np.percentile(dn, 99.9), dn.max())
    ds = np.abs(ps["scales"][pick] - ref[key + "_scales"]) / float(ref[key + "_scales_absmax"])
    assert ds.max() <= 3e-5, ds.max()          # float sums over <= 9 neighbours, the reference binary contracts to FMAs
    assert _sha(got["vertex_ids"].astype(np.uint32)) == sha_vids
    assert got["faces"].shape == (nf, 3) and _sha(got["faces"].astype(np.uint32)) == sha_faces
    assert got["vertices"].shape == (nv, 3)
    vmax = float(ref[key + "_verts_absmax"])
    assert np.abs(got["vertices"][pick] - verts).max() <= 1e-6 * vmax
    if color:
        assert np.abs(got["colors"][pick] - ref[key + "_colors"]).max() <= 1e-6
    # world transform = the reference's mesh_transform of the same vertices
    ctw = np.eye(4, dtype=np.float32)
    ctw[:3, :3] = np.array([[0.36, 0.48, -0.8], [-0.8, 0.6, 0.0], [0.48, 0.64, 0.6]], np.float32)
    ctw[:3, 3] = [1.5, -2.0, 0.25]
    gw = D.depthmap_triangulate(dm, invproj, dd_factor=dd, cam_to_world=ctw)
    want = verts @ ctw[:3, :3].T + ctw[:3, 3]
    assert np.abs(gw["vertices"][pick] - want).max() <= 2e-6 * np.abs(want).max()
    assert _sha(gw["faces"].astype(np.uint32)) == sha_faces
