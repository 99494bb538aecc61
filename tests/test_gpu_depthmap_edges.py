"""Depth-map consumers on the device (-m gpu) at their decision boundaries and edge shapes, against the NumPy restatement
tests/dm_reference.py and, for the same inputs, against the reference binary's results (golden fixture
tests/golden/depthmap_edges_ref.npz, minted by tests/golden/make_golden.py depthmap_edges; tests/test_depthmap_reference.py
pins the restatement to it without a GPU).

Exact: cleanup / confidence_clean results, vertex ids, faces, counts, boundary confidences.  Vertices and colours within
1e-6 relative to the restatement's float32 path and within a few ulps of its float64 path, normals p99.9 <= 1e-4 and
max <= 2e-3, scale values within 3e-5 relative."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import scipy.ndimage

from tests import dm_reference as R

pytestmark = pytest.mark.gpu
F32 = np.float32
DD_EDGE = (5.0, 12.7428637, 16.3189125)        # the last two: float(dd * sqrt2) != dd * (float)sqrt2
CONF_ITERS = (1, 2, 4, 7, 255, 256, 300)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---------------------------------------------------------------- inputs
def smooth_map(h, w, seed, holes=0.1):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(F32)
    d = (5.0 + 0.4 * np.sin(xx / 7.0) + 0.3 * np.cos(yy / 5.0)).astype(F32)
    d[rng.random((h, w)) < holes] = 0.0
    return d


def spiral(h, w):
    """One serpentine component through the whole map: every other row filled, joined alternately at the right and left."""
    d = np.zeros((h, w), F32)
    d[0::2] = 3.0
    d[1::4, -1] = 3.0
    d[3::4, 0] = 3.0
    return d


def comb(h, w):
    """A spine along the top with teeth of growing length hanging off it, and loose teeth of the same lengths below."""
    d = np.zeros((h, w), F32)
    d[0] = 2.0
    for i, x in enumerate(range(0, w, 2)):
        d[1:1 + (i % (h // 2 - 1)) + 1, x] = 2.0
        d[h // 2 + 1:h // 2 + 1 + (i % (h // 2 - 2)) + 1, x] = 4.0
    return d


def checker(h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.where((xx + yy) % 2 == 0, F32(1.5), F32(0.0)).astype(F32)


def diagonal(h, w):
    """2x2 squares that touch only at their corners: separate components under 4-connectivity."""
    yy, xx = np.mgrid[0:h, 0:w]
    return np.where(((xx // 2) + (yy // 2)) % 2 == 0, F32(2.5), F32(0.0)).astype(F32)


def special(h, w, seed):
    """Depths of -0.0, NaN, +-inf and negative values among ordinary ones and zeros."""
    rng = np.random.default_rng(seed)
    d = (1.0 + rng.random((h, w))).astype(F32)
    pick = rng.integers(0, 7, size=(h, w))
    for k, v in enumerate((0.0, -0.0, np.nan, np.inf, -np.inf, -2.0)):
        d[pick == k + 1] = v
    return d


def cleanup_cases():
    """name -> (depth, conf, thresholds).  Thresholds: 0, -1 and every component size of interest and its neighbours."""
    out = {}
    rng = np.random.default_rng(5)
    shapes = {"1x1": (1, 1), "1xN": (1, 77), "Nx1": (63, 1), "2x2": (2, 2), "33x9": (9, 33), "31x7": (7, 31)}
    for name, (h, w) in shapes.items():
        out[name] = smooth_map(h, w, seed=h * 1000 + w, holes=0.3)
    out["spiral"] = spiral(131, 257)
    out["comb"] = comb(40, 97)
    out["checker"] = checker(33, 65)
    out["diagonal"] = diagonal(36, 70)
    out["special"] = special(47, 53, seed=2)
    cases = {}
    for name, d in out.items():
        lab, n = scipy.ndimage.label(d != 0, structure=R.FOUR)
        sizes = sorted(set(np.bincount(lab.ravel())[1:].tolist()))
        sizes = sizes[:3] + sizes[-3:]
        thres = sorted({-1, 0, 1, 2} | {s + k for s in sizes for k in (-1, 0, 1)})
        conf = rng.random(d.shape).astype(F32) - 0.3
        conf.reshape(-1)[rng.integers(0, conf.size, size=max(1, conf.size // 7))] = np.nan
        conf.reshape(-1)[rng.integers(0, conf.size, size=max(1, conf.size // 7))] = -0.0
        conf.reshape(-1)[rng.integers(0, conf.size, size=max(1, conf.size // 9))] = 0.0
        cases[name] = (d, conf, thres)
    return cases


def invproj_for(h, w, m0=None):
    ax = float(max(w, h))
    f = 1.0 / ax if m0 is None else m0
    return np.array([f, 0, -0.5 * w * f, 0, f, -0.5 * h * f, 0, 0, 1], F32)


def boundary_map(dd, seed, h=96, w=192):
    """Isolated 2x2 blocks (one empty row and column between them) whose tested edge has d_max - d_min exactly on
    width * dd_factor (width from the reference build's footprint arithmetic, the diagonal factor rounded through double)
    or one ulp of d_max either side.  The other corners sit half-way, far from their own thresholds.  3-of-4 masks test
    axis and diagonal edges; 4-of-4 blocks use the mirrored tie |d0 - d3| == |d1 - d2| with an axis edge on the threshold."""
    rng = np.random.default_rng(seed)
    ip = invproj_for(h, w, m0=0.02)
    d = np.zeros((h, w), F32)
    by, bx = np.mgrid[0:h - 1:3, 0:w - 1:3]
    by, bx = by.ravel(), bx.ravel()
    nb = len(by)
    masks = rng.choice([7, 11, 13, 14, 15], size=nb)
    # tested edge (i_min, i_max) per mask: one axis and one diagonal edge of the mask's triangle
    edges = {7: [(0, 1), (1, 2)], 11: [(1, 3), (0, 3)], 13: [(2, 3), (3, 0)], 14: [(3, 1), (2, 1)], 15: [(0, 1)]}
    e = np.array([edges[m][rng.integers(0, len(edges[m]))] for m in masks])
    a, b = e[:, 0], e[:, 1]
    ax_, ay_ = bx + a % 2, by + a // 2
    _, _, _, sq = R.pixel_rays(ip, ax_, ay_)
    norm = np.sqrt(sq)
    ddf = np.where((a + b) == 3, R.diagonal_factor(dd), F32(dd)).astype(F32)
    lo = (F32(2.0) + rng.random(nb).astype(F32)).astype(F32)
    found = np.zeros(nb, bool)
    d_lo, d_hi = lo.copy(), lo.copy()
    for _ in range(256):
        thr = ((ip[0] * lo) / norm) * ddf
        hi = lo + thr
        ok = ~found & ((hi - lo) == thr)
        d_lo[ok], d_hi[ok] = lo[ok], hi[ok]
        found |= ok
        lo = np.nextafter(lo, F32(np.inf))
    assert found.all()
    side = rng.integers(-1, 2, size=nb)                  # -1, 0, +1 ulp of d_max
    d_hi = np.where(side > 0, np.nextafter(d_hi, F32(np.inf)), np.where(side < 0, np.nextafter(d_hi, F32(0)), d_hi))
    mid = ((d_lo + d_hi) * F32(0.5)).astype(F32)
    for k in range(nb):
        blk = np.full(4, mid[k], F32)
        for j in range(4):
            if not (masks[k] >> j) & 1:
                blk[j] = 0.0
        blk[a[k]], blk[b[k]] = d_lo[k], d_hi[k]
        if masks[k] == 15:                               # mirrored tie: d0 = d2 = lo, d1 = d3 = hi
            blk[:] = (d_lo[k], d_hi[k], d_lo[k], d_hi[k])
        d[by[k]:by[k] + 2, bx[k]:bx[k] + 2] = blk.reshape(2, 2)
    return d, ip


def ties_map(seed, h=60, w=90):
    """Full 2x2 blocks whose diagonals differ by exactly as much, or by one ulp more or less, all below the threshold."""
    rng = np.random.default_rng(seed)
    d = np.zeros((h, w), F32)
    for y in range(0, h - 1, 3):
        for x in range(0, w - 1, 3):
            base = F32(3.0 + rng.random())
            step = F32(0.01 * rng.random())
            d0, d3 = base, F32(base + step)
            diff = F32(d3 - d0)
            d1 = F32(base + F32(0.02))
            d2 = F32(d1 + diff)
            d2 = [d2, np.nextafter(d2, F32(np.inf)), np.nextafter(d2, F32(0))][rng.integers(0, 3)]
            blk = np.array([d0, d1, d2, d3], F32)
            if rng.random() < 0.5:
                blk = blk[[1, 0, 3, 2]]                 # the tie the other way round
            d[y:y + 2, x:x + 2] = blk.reshape(2, 2)
    return d


def special_blocks(seed, h=64, w=96):
    """A smooth map with NaN, +-inf, -0.0 and negative depths inside blocks (the mask takes > 0, the widths != 0).  +inf
    only at even (x, y), so no block has two: its edges to finite depths are discontinuities, no face keeps it."""
    rng = np.random.default_rng(seed)
    d = smooth_map(h, w, seed, holes=0.05)
    pick = rng.integers(0, 14, size=(h, w))
    yy, xx = np.mgrid[0:h, 0:w]
    for k, v in enumerate((np.nan, np.inf, -np.inf, -0.0, -3.0)):
        d[(pick == k + 1) & ((v != np.inf) | ((xx % 2 == 0) & (yy % 2 == 0)))] = v
    return d


def complex_map(h=64, w=96):
    """Fans that meet at single pixels: a checkerboard of 2x2 holes in one half, mask-7 / mask-14 staircases in the other."""
    d = np.full((h, w), 4.0, F32)
    yy, xx = np.mgrid[0:h, 0:w]
    left = xx < w // 2
    d[left & ((xx // 2) % 2 == 0) & ((yy // 2) % 2 == 0) & ((xx // 4 + yy // 4) % 2 == 0)] = 0.0
    stair = ~left & ((xx - yy) % 4 == 0) & ((yy % 6) < 4)
    d[stair] = 0.0
    d[~left & ((xx + yy) % 5 == 0) & ((yy % 7) == 3)] = 0.0
    return d


def tri_cases():
    """name -> dict(dm, invproj, dd, color, conf_iters, ref_iters, scale).  ref_iters: the conf_iterations the fixture has
    reference results for.  The reference's ring loop queues a vertex once for every queued neighbour, duplicates included
    (depthmap.cc:537-543), so its work grows exponentially with the ring depth: it cannot run the deep rings of the
    hole-free 600x600 map, which only the restatement checks."""
    rng = np.random.default_rng(11)
    cases = {}

    def add(name, dm, dd=5.0, color=3, conf_iters=(4,), scale=2.5, ip=None, ref_iters=None):
        h, w = dm.shape
        ci = None
        if color == 1:
            ci = rng.integers(0, 256, size=(h, w), dtype=np.uint8)
        elif color:
            ci = rng.integers(0, 256, size=(h, w, color), dtype=np.uint8)
        cases[name] = dict(dm=dm, invproj=invproj_for(h, w) if ip is None else ip, dd=float(F32(dd)), color=ci,
                           conf_iters=tuple(conf_iters), ref_iters=tuple(conf_iters if ref_iters is None else ref_iters),
                           scale=scale)

    for name, (h, w) in {"2x2": (2, 2), "2xN": (2, 37), "Nx2": (41, 2), "33x9": (9, 33), "31x7": (7, 31),
                         "257x131": (131, 257)}.items():
        add(name, smooth_map(h, w, seed=h + 7 * w, holes=0.15))
    for k, (dd, ch) in enumerate(zip(DD_EDGE, (1, 2, 4))):
        dm, ip = boundary_map(dd, seed=20 + k)
        add("bound_%d" % k, dm, dd=dd, color=ch, ip=ip)
    add("ties", ties_map(seed=3), color=0)
    add("special", special_blocks(seed=4), color=3)
    add("complex", complex_map(), color=1)
    plate = (6.0 + 0.3 * np.sin(np.mgrid[0:600, 0:600][1] / 50.0)).astype(F32)     # hole-free: ~300 rings deep
    add("plate600", plate, color=0, conf_iters=CONF_ITERS, ref_iters=(1, 2, 4, 7))
    add("ragged", smooth_map(97, 131, seed=9, holes=0.45), color=0, conf_iters=CONF_ITERS)
    add("scale0", smooth_map(50, 70, seed=12, holes=0.2), color=0, scale=0.0)
    add("scale1", smooth_map(50, 70, seed=13, holes=0.2), color=0, scale=1.0)
    return cases


# ---------------------------------------------------------------- device vs restatement (and fixture)
def _ref():
    from tests.util import golden_ref
    return golden_ref("depthmap_edges")


@pytest.fixture(scope="module")
def edges_ref():
    return _ref()


@pytest.fixture(scope="module")
def tcases():
    return tri_cases()


@pytest.mark.parametrize("name", list(cleanup_cases()))
def test_cleanup_and_confclean_edges(name, edges_ref):
    from mve_b200 import depthmap as D
    dm, cm, thres = cleanup_cases()[name]
    assert list(edges_ref["cleanup_%s_thres" % name]) == thres
    got = dm.copy()
    D.depthmap_confidence_clean(got, cm)
    want = R.confidence_clean(dm, cm)
    assert got.tobytes() == want.tobytes()
    assert sha(got) == str(edges_ref["confclean_%s" % name])
    for t in thres:
        got = D.depthmap_cleanup(dm, t)
        want = R.cleanup(dm, t)
        assert got.tobytes() == want.tobytes(), (name, t, int((got.view(np.uint32) != want.view(np.uint32)).sum()))
        assert sha(got) == str(edges_ref["cleanup_%s_%d" % (name, t)]), (name, t)


def _check_vertices(got, want32, want64, absmax):
    ok = np.isfinite(want32)
    assert (np.isfinite(got) == ok).all()
    scale = max(float(absmax), 1e-30)
    assert np.abs(got[ok] - want32[ok]).max(initial=0) <= 1e-6 * scale
    # a different operation order than the reference's shows up as more than a few ulps from the exact value
    assert np.abs(got[ok].astype(np.float64) - want64[ok]).max(initial=0) <= 4 * np.finfo(F32).eps * scale


def _compare(ps, ref, case, fixture, key):
    nv, nf = len(ref["vertices"]), len(ref["faces"])
    assert (len(ps["vertices"]), len(ps["faces"])) == (nv, nf), "vertex / face counts differ"
    assert ps["vertex_ids"].tobytes() == ref["vertex_ids"].tobytes()
    assert ps["faces"].astype(np.uint32).tobytes() == ref["faces"].tobytes()
    if fixture is not None:
        n = fixture[key + "_n"]
        assert (int(n[0]), int(n[1])) == (nv, nf)
        sv, sf = (str(x) for x in fixture[key + "_sha"])
        assert sha(ps["vertex_ids"].astype(np.uint32)) == sv and sha(ps["faces"].astype(np.uint32)) == sf
    if nv == 0:
        return
    absmax = np.abs(ref["vertices64"][np.isfinite(ref["vertices64"])]).max(initial=1.0)
    _check_vertices(ps["vertices"], ref["vertices"], ref["vertices64"], absmax)
    if case["color"] is not None:
        assert np.abs(ps["colors"] - ref["colors"]).max() <= 1e-6


@pytest.mark.parametrize("name", list(tri_cases()))
def test_pointset_edges(name, tcases, edges_ref):
    from mve_b200 import depthmap as D
    case = tcases[name]
    dm, ip, dd, ci = case["dm"], case["invproj"], case["dd"], case["color"]
    ref = R.pointset(dm, ip, dd, ci, scale_factor=case["scale"], conf_iterations=max(case["conf_iters"]))
    key = "tri_%s" % name
    wrong_confs = {}                                    # conf_iterations -> vertices whose confidence differs
    for it in case["conf_iters"]:
        ps = D.depthmap_pointset(dm, ip, dd_factor=dd, color=ci, with_normals=True, conf_iterations=it,
                                 scale_factor=case["scale"])
        _compare(ps, ref, case, edges_ref, key)
        want = R.confidences(len(ref["vertices"]), ref["faces"], it, ref["rings"])
        if ps["confidences"].tobytes() != want.tobytes():
            wrong_confs[it] = int((ps["confidences"] != want).sum())
        elif it in case["ref_iters"]:
            assert sha(ps["confidences"].astype(F32)) == str(edges_ref["%s_confs_%d" % (key, it)]), (name, it)
    assert not wrong_confs, wrong_confs
    if len(ref["vertices"]) == 0:
        return
    dn = np.abs(ps["normals"] - ref["normals"]).max(-1)
    assert np.percentile(dn, 99.9) <= 1e-4 and dn.max() <= 2e-3, (np.percentile(dn, 99.9), dn.max())
    # from the device's own vertices: on a flat map the distances to the neighbours are differences of nearly equal
    # coordinates, and the vertices' last-ulp differences alone would move them by more than the scale arithmetic does
    want = R.scales(ps["vertices"], ref["faces"], case["scale"])
    smax = max(float(np.abs(want).max()), 1e-30)
    assert np.abs(ps["scales"] - want).max() <= 3e-5 * smax, np.abs(ps["scales"] - want).max() / smax
    if case["scale"] == 0.0:
        assert (ps["scales"] == 0).all()
    # the plain triangulation entry point gives the same mesh
    tr = D.depthmap_triangulate(dm, ip, dd_factor=dd, color=ci)
    _compare(tr, ref, case, edges_ref, key)


def test_boundary_cases_sit_on_the_threshold(tcases):
    """The boundary maps do what they claim: every kind of block, and faces both kept and dropped at the threshold."""
    for k, dd in enumerate(DD_EDGE):
        case = tcases["bound_%d" % k]
        tri = R.block_triangles(case["dm"], case["invproj"], dd)
        tri0 = R.block_triangles(case["dm"], case["invproj"], 0.0)
        kept, total = (tri > 0).sum(), (tri0 > 0).sum()
        assert 0.2 * total < kept < 0.9 * total, (kept, total)
    assert R.diagonal_factor(DD_EDGE[1]) != F32(F32(DD_EDGE[1]) * F32(R.MATH_SQRT2))
    assert R.diagonal_factor(DD_EDGE[2]) != F32(F32(DD_EDGE[2]) * F32(R.MATH_SQRT2))
    mesh = R.triangulate(tcases["complex"]["dm"], tcases["complex"]["invproj"])
    cls = R.mesh_info(len(mesh["vertices"]), mesh["faces"])[0]
    assert (cls == 1).sum() >= 10 and (cls == 2).sum() >= 100


def test_cam_to_world_and_large_map():
    """cam_to_world on depthmap_pointset, and a 4096x2304 map (> 2^23 pixels, many CTA tiles) for cleanup and triangulate."""
    from mve_b200 import depthmap as D
    dm = smooth_map(131, 257, seed=31, holes=0.1)
    ip = invproj_for(131, 257)
    ctw = np.eye(4, dtype=F32)
    ctw[:3, :3] = np.array([[0.36, 0.48, -0.8], [-0.8, 0.6, 0.0], [0.48, 0.64, 0.6]], F32)
    ctw[:3, 3] = [1.5, -2.0, 0.25]
    ref = R.pointset(dm, ip, 5.0, cam_to_world=ctw)
    ps = D.depthmap_pointset(dm, ip, dd_factor=5.0, cam_to_world=ctw)
    assert ps["faces"].astype(np.uint32).tobytes() == ref["faces"].tobytes()
    assert np.abs(ps["vertices"] - ref["vertices"]).max() <= 2e-6 * np.abs(ref["vertices64"]).max()
    assert np.abs(ps["vertices"] - ref["vertices64"]).max() <= 8 * np.finfo(F32).eps * np.abs(ref["vertices64"]).max()
    big = spiral(2304, 4096)
    big[1::4, 2000:2100] = 5.0                          # bridges between the rows: cycles in one long component
    big[:, ::7] = np.where(big[:, ::7] != 0, F32(5.125), F32(0.0))
    for t in (0, 1000, int((big != 0).sum()), int((big != 0).sum()) + 1):
        assert D.depthmap_cleanup(big, t).tobytes() == R.cleanup(big, t).tobytes(), t
    hb = smooth_map(2304, 4096, seed=32, holes=0.2)
    ipb = invproj_for(2304, 4096)
    tr = D.depthmap_triangulate(hb, ipb, dd_factor=5.0)
    rt = R.triangulate(hb, ipb, 5.0)
    assert tr["vertex_ids"].tobytes() == rt["vertex_ids"].tobytes()
    assert tr["faces"].astype(np.uint32).tobytes() == rt["faces"].tobytes()
    assert np.abs(tr["vertices"] - rt["vertices"]).max() <= 1e-6 * np.abs(rt["vertices64"]).max()


# ---------------------------------------------------------------- the C ABI: capacities and argument checks
def _abi_call(dm, ip, cap_v, cap_f, w=None, h=None, conf_iterations=4, color=None, cch=0):
    from mve_b200 import depthmap as D
    L = D._lib()
    hh, ww = dm.shape
    w = ww if w is None else w
    h = hh if h is None else h
    vids = np.empty(dm.size, np.uint32)
    verts = np.empty((max(cap_v, 1), 3), F32)
    faces = np.empty((max(cap_f, 1), 3), np.uint32)
    nrm = np.empty((max(cap_v, 1), 3), F32)
    cf = np.empty(max(cap_v, 1), F32)
    sc = np.empty(max(cap_v, 1), F32)
    nv, nf = C.c_uint64(0), C.c_uint64(0)
    p = D._p
    rc = L.b200mvs_depthmap_pointset(0, p(dm), w, h, p(ip), 5.0, None, p(color), cch, p(vids), p(verts), None, p(faces),
                                     p(nrm), p(cf), conf_iterations, p(sc), 2.5, cap_v, cap_f, C.byref(nv), C.byref(nf), None)
    return rc, nv.value, nf.value, vids, verts, faces


def test_abi_capacities_and_errors():
    dm = smooth_map(33, 47, seed=40, holes=0.2)
    ip = invproj_for(33, 47)
    ref = R.triangulate(dm, ip, 5.0)
    nv, nf = len(ref["vertices"]), len(ref["faces"])
    rc, gv, gf, vids, verts, faces = _abi_call(dm, ip, nv, nf)
    assert rc == 0 and (gv, gf) == (nv, nf)
    assert faces[:nf].tobytes() == ref["faces"].tobytes() and vids.tobytes() == ref["vertex_ids"].tobytes()
    for cv, cf in ((nv - 1, nf), (nv, nf - 1)):
        rc, gv, gf, *_ = _abi_call(dm, ip, cv, cf)
        assert rc == -5 and (gv, gf) == (nv, nf), (rc, gv, gf)          # B200MVS_ERR_OVERFLOW, true counts reported
    assert _abi_call(dm, ip, nv, nf, w=1)[0] == -1                       # B200MVS_ERR_INVALID_ARG
    assert _abi_call(dm, ip, nv, nf, h=1)[0] == -1
    assert _abi_call(dm, ip, nv, nf, conf_iterations=-1)[0] == -1
    col = np.zeros(dm.size * 5, np.uint8)
    assert _abi_call(dm, ip, nv, nf, color=col, cch=0)[0] == -1
    assert _abi_call(dm, ip, nv, nf, color=col, cch=5)[0] == -1
    assert _abi_call(dm, ip, nv, nf, color=col, cch=4)[0] == 0
