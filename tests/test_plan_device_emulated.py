"""The device planner (mve_b200/csrc/plan_device.cuh: analyzeFeatures + GlobalViewSelection + the seed list of
processFeatures, one CTA per reference view) compiled by g++ and run on the CPU with several threads per "CTA".  Its
selections must equal the planning context's global_view_selection exactly, its seeds a float32 NumPy restatement of
collect_seeds exactly, and its look-up of the parallax factor must equal the host's plx_factor for every float it can
meet."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import camera_reference as CR
from tests.util import golden_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")

PLAN_VIEW = np.dtype([("campos", "<f4", 3), ("w2c", "<f4", 12), ("proj0", "<f4", 9), ("inv0", "<f4"), ("proj_s", "<f4", 9),
                      ("inv_s", "<f4"), ("w0", "<i4"), ("h0", "<i4"), ("valid", "<i4"), ("pad", "<i4")])
SEED = np.dtype([("x", "<i4"), ("y", "<i4"), ("depth", "<f4")])
BIG = np.float32(3.0e38)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("plan_emu") / "libplan_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I" + EMU,
                           os.path.join(EMU, "plan_emu.cc"), "-o", lib])
    L = C.CDLL(lib)
    assert L.emu_plan_view_size() == PLAN_VIEW.itemsize
    L.emu_plan_view.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.emu_check_lookup.restype = C.c_longlong
    L.emu_check_lookup.argtypes = [C.c_float, C.c_uint, C.c_uint, C.POINTER(C.c_longlong)]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Inputs:
    """What the device planner reads, built from a scene as the library builds it from its registered cameras."""

    def __init__(self, s, scale, n_views=None, feat_pos=None, feat_refs=None):
        nv = n_views or s.n_views
        self.nv = nv
        self.views = np.zeros(nv, PLAN_VIEW)
        self.levels = {}
        for v in range(s.n_views):
            r = np.asarray(s.rot[v], np.float32).reshape(9)
            t = np.asarray(s.trans[v], np.float32).reshape(3)
            o = self.views[v]
            o["campos"] = [(-r[c] * t[0] - r[3 + c] * t[1]) - r[6 + c] * t[2] for c in range(3)]
            o["w2c"] = np.concatenate([np.r_[r[3 * i:3 * i + 3], t[i]] for i in range(3)])
            lv = CR.view_levels(s, v, np.float32)
            self.levels[v] = lv
            o["proj0"] = np.asarray(lv[0][2], np.float32).reshape(9)
            o["inv0"] = np.float32(lv[0][3][0, 0])
            if scale < len(lv):
                o["proj_s"] = np.asarray(lv[scale][2], np.float32).reshape(9)
                o["inv_s"] = np.float32(lv[scale][3][0, 0])
            o["w0"], o["h0"] = lv[0][0], lv[0][1]
            o["valid"] = 1
        self.pos = np.ascontiguousarray(s.feat_pos if feat_pos is None else feat_pos, np.float32).reshape(-1, 3)
        refs = s.feat_refs if feat_refs is None else feat_refs
        self.nf = len(refs)
        self.foff = np.zeros(self.nf + 1, np.int32)
        self.foff[1:] = np.cumsum([len(r) for r in refs])
        self.frefs = np.ascontiguousarray(np.concatenate([np.asarray(r, np.int32) for r in refs]) if self.nf else np.zeros(0, np.int32))
        vf = [[] for _ in range(nv)]
        for i, r in enumerate(refs):
            for v in r:
                if 0 <= v < nv and (not vf[v] or vf[v][-1] != i):
                    vf[v].append(i)
        self.vf = vf
        self.vfoff = np.zeros(nv + 1, np.int32)
        self.vfoff[1:] = np.cumsum([len(x) for x in vf])
        self.vfids = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32) for x in vf]) if self.vfoff[-1] else np.zeros(1, np.int32))

    def plan(self, L, ref, min_parallax, aabb, gvs_max, nt=8):
        sel = np.zeros(32, np.int32)
        n_sel = C.c_int()
        seeds = np.zeros(max(self.nf, 1), SEED)
        box = np.asarray(aabb, np.float32).reshape(6)
        n = L.emu_plan_view(_p(self.views), self.nv, _p(self.pos), _p(self.foff), _p(self.frefs), self.nf, _p(self.vfoff),
                            _p(self.vfids), float(min_parallax), _p(box), gvs_max, ref, nt, _p(sel), C.byref(n_sel),
                            _p(seeds), len(seeds))
        assert n >= 0 or n == -1, n
        return (None, None) if n == -1 else (sel[:n_sel.value].tolist(), seeds[:n])


def _dot3(a, b):
    f = np.float32
    return ((f(0) + a[..., 0] * b[..., 0]) + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def np_seeds(I, ref, gsel, scale, aabb):
    """collect_seeds (b200mvs.cu) in float32: the features of the reference view or a selected view, in feature order, that
    lie in its frustum and the box, at the rounded pixel of level `scale` with the distance to the camera centre."""
    ids = sorted(set(I.vf[ref]).union(*[I.vf[g] for g in gsel]))
    if not ids:
        return np.zeros(0, SEED)
    p = I.pos[ids]
    v = I.views[ref]
    w2c = v["w2c"].reshape(3, 4)
    cp = np.stack([_dot3(np.broadcast_to(w2c[i, :3], p.shape), p) + w2c[i, 3] for i in range(3)], -1)
    P0, Ps = v["proj0"].reshape(3, 3), v["proj_s"].reshape(3, 3)
    sp = np.stack([_dot3(np.broadcast_to(P0[i], p.shape), cp) for i in range(3)], -1)
    with np.errstate(all="ignore"):
        x = sp[:, 0] / sp[:, 2] - np.float32(0.5)
        y = sp[:, 1] / sp[:, 2] - np.float32(0.5)
        ok = (cp[:, 2] > 0) & (x >= 0) & (x <= np.float32(v["w0"] - 1)) & (y >= 0) & (y <= np.float32(v["h0"] - 1))
    lo, hi = np.asarray(aabb[:3], np.float32), np.asarray(aabb[3:], np.float32)
    ok &= ((p >= lo) & (p <= hi)).all(-1)
    p, cp = p[ok], cp[ok]
    ss = np.stack([_dot3(np.broadcast_to(Ps[i], p.shape), cp) for i in range(3)], -1)
    px = ss[:, 0] / ss[:, 2] - np.float32(0.5)
    py = ss[:, 1] / ss[:, 2] - np.float32(0.5)

    def round_mve(a):
        return np.where(a > 0, np.floor(a + np.float32(0.5)), np.ceil(a - np.float32(0.5))).astype(np.float32)

    dv = p - v["campos"]
    out = np.zeros(len(p), SEED)
    out["x"], out["y"] = round_mve(px).astype(np.int32), round_mve(py).astype(np.int32)
    out["depth"] = np.sqrt(_dot3(dv, dv))
    return out


def _planning_scene(s, n_views=None, feat_pos=None, feat_refs=None):
    from mve_b200 import dmrecon
    g = dmrecon.Scene(n_views or s.n_views, device=-1)
    for v in range(s.n_views):
        g.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    g.set_features(s.feat_pos if feat_pos is None else feat_pos, s.feat_refs if feat_refs is None else feat_refs)
    return g


def _cutting_box(s):
    lo, hi = np.percentile(np.asarray(s.feat_pos, np.float64).reshape(-1, 3), [20, 80], axis=0)
    return np.r_[lo, hi].astype(np.float32)


def _check(L, s, g, views, cases, **kw):
    from mve_b200 import dmrecon
    for scale, mp, gmax, box in cases:
        I = Inputs(s, scale, **kw)
        st = dmrecon.Settings(scale=scale, global_vs_max=gmax, min_parallax=mp)
        st.aabb_min[:] = box[:3].tolist()
        st.aabb_max[:] = box[3:].tolist()
        for v in views:
            if scale >= len(I.levels[v]):
                continue
            sel, seeds = I.plan(L, v, mp, box, gmax)
            want = g.global_view_selection(st, v)
            assert sel == want, (scale, mp, gmax, v)
            want_seeds = np_seeds(I, v, sel, scale, box)
            assert seeds.tobytes() == want_seeds.tobytes(), (scale, mp, gmax, v, len(seeds), len(want_seeds))


def _cases(s):
    full = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    cut = _cutting_box(s)
    out = [(s.scale, mp, gmax, full) for gmax in (1, 3, 20, 32) for mp in (5.0, 10.0, 30.0)]
    out += [(scale, 10.0, 20, box) for scale in (0, 1, 2) for box in (full, cut)]
    return out


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T3", "T4", "T5", "T6"])
def test_golden_scenes(emu, name):
    s = golden_scene(name)
    _check(emu, s, _planning_scene(s), range(s.n_views), _cases(s))


@pytest.fixture(scope="module")
def tiled():
    from mve_b200 import synth
    cfg = dict(synth.CONFIGS["C2"])
    cfg.update(views=48, grid=(12, 4), blocks=3, features=6000, width=96, height=54, name="C2x3")
    return synth.make_scene(cfg)


def test_tiled_c2x3(emu, tiled):
    """The tiled C2x3 scene of test_host_view_selection: 48 views, every selection saturates at globalVSMax."""
    s = tiled
    full = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    cases = [(0, mp, gmax, full) for gmax in (1, 3, 20, 32) for mp in (5.0, 10.0, 30.0)] + [(0, 10.0, 20, _cutting_box(s))]
    _check(emu, s, _planning_scene(s), (0, 7, 16, 23, 31, 47), cases)


@pytest.mark.parametrize("name", ["C3", "C5"])
def test_cameras_only_bench_scenes(emu, name):
    """The bench scenes' cameras and features (no images): many candidates and refs per feature."""
    from mve_b200 import synth
    s = synth.make_scene(name, only_views=[])
    full = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    cases = [(s.scale, 10.0, 20, full), (s.scale, 5.0, 32, full), (s.scale, 30.0, 3, _cutting_box(s))]
    _check(emu, s, _planning_scene(s), (0, s.n_views // 2 + 1, s.n_views - 1), cases)


@pytest.mark.parametrize("min_parallax", [5.0, 10.0, 30.0, 40.0])
def test_factor_lookup_is_the_host_factor(emu, min_parallax):
    """Every float in [dot_skip, 1], 2^20 floats below dot_skip and 2^20 above 1 (clamped): the look-up equals the host's
    plx_factor bit for bit.  This checks the indexing and both edges; the table is the host's function by construction."""
    n = C.c_longlong()
    bad = emu.emu_check_lookup(min_parallax, 1 << 20, 1 << 20, C.byref(n))
    assert bad == 0 and n.value > (1 << 21), (bad, n.value)


def test_table_cap(emu):
    """Above about 41 degrees of minParallax the table would exceed 2^22 entries: the device declines and the host plans."""
    s = golden_scene("T0")
    I = Inputs(s, s.scale)
    full = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    assert I.plan(emu, 0, 40.0, full, 20)[0] is not None
    assert I.plan(emu, 0, 45.0, full, 20) == (None, None)
    n = C.c_longlong()
    assert emu.emu_check_lookup(45.0, 0, 0, C.byref(n)) == -1
    assert emu.emu_check_lookup(95.0, 0, 0, C.byref(n)) == -1


def test_edge_cases(emu):
    """Duplicate and out-of-range refs, a view without a camera, ties between identical cameras, a view without features."""
    s = golden_scene("T0")
    nv = s.n_views + 2               # view nv - 2: a copy of view 1's camera (ties with it); nv - 1: no camera
    rng = np.random.default_rng(7)
    refs = []
    for r in s.feat_refs:
        r = list(r)
        if 1 in r:
            r.append(nv - 2)
        k = rng.integers(0, 6)
        if k == 0 and r:
            r.append(r[0])           # duplicate
        elif k == 1:
            r += [-1, 99]            # out of range
        elif k == 2:
            r.append(nv - 1)         # a view without a camera
        refs.append(np.asarray(r, np.int32))

    class S2:
        pass
    s2 = S2()
    for k in ("rot", "trans", "flen", "paspect", "ppoint"):
        a = list(getattr(s, k))
        setattr(s2, k, a + [a[1]])
    s2.n_views = s.n_views + 1
    s2.size = lambda v: s.size(min(v, 1) if v >= s.n_views else v)
    s2.feat_pos, s2.feat_refs, s2.scale = s.feat_pos, refs, s.scale
    g = _planning_scene(s2, n_views=nv)
    full = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    cases = [(s.scale, 10.0, gmax, full) for gmax in (1, 3, 20)]
    _check(emu, s2, g, range(s2.n_views), cases, n_views=nv)
    # the twin cameras tie wherever both are candidates: the lower id wins
    I = Inputs(s2, s.scale, n_views=nv)
    sel, _ = I.plan(emu, 0, 10.0, full, 1)
    assert sel != [nv - 2]
    # a view that no feature references: empty selection, no seeds
    I = Inputs(s2, s.scale, n_views=nv, feat_refs=[np.asarray([v for v in r if v != 0], np.int32) for r in refs])
    sel, seeds = I.plan(emu, 0, 10.0, full, 20)
    assert sel == [] and len(seeds) == 0
