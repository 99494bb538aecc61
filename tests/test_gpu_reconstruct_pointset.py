"""b200mvs_pset_add_reconstruction (-m gpu): dmrecon and scene2pset in one call, the maps staying on the device.

The result must be byte for byte what the host route gives: Scene.reconstruct with host maps, then scene_pointset of those
maps with each view's level-`scale` image (Scene.level) and the camera the view was registered with, in ref_views order.
Covered: the -F option set, -p, a bounding box that cuts the scene, -f skipping a view, -C, masks applied afterwards, on
T0, T5 and T6 (odd level sizes and clamped levels: a calibration taken from the pyramid level would move the points);
a budgeted context whose planner makes several groups out of ref_views order; 1- and 4-channel `undistorted` images at
scale 0; rejected handles, a failing view selection, one view and every view cancelled."""
import ctypes as C

import numpy as np
import pytest

from tests import pset_reference as S
from tests.util import golden_scene

pytestmark = pytest.mark.gpu

ARRAYS = ("vertices", "normals", "colors", "values", "confidences")
F_SET = dict(with_normals=True, with_conf=True, with_scale=True)


def _settings(s):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)


def _refs(s, seed=0):
    return np.random.default_rng(seed).permutation(s.n_views).tolist()


def host_route(sc, s, st, refs, options=None, masks=None, images=None):
    """The sequence the call replaces: reconstruct with host maps, the level images, scene_pointset."""
    from mve_b200 import depthmap as D
    maps, _ = sc.reconstruct(st, refs, want=("depth",))
    views = [dict(id=v, depth=maps[j]["depth"], camera=S.camera_of(s, v),
                  color=sc.level(v, st.scale) if images is None else images[v]) for j, v in enumerate(refs)]
    return D.scene_pointset(views, options, masks), maps


def same(a, b):
    for k in ARRAYS:
        assert (a[k] is None) == (b[k] is None), k
        if a[k] is not None:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
    assert a["views"] == b["views"]
    assert a["num_filtered"] == b["num_filtered"]
    assert (a["correspondence"] is None) == (b["correspondence"] is None)
    if a["correspondence"] is not None:
        assert a["correspondence"]["pixels"].tobytes() == b["correspondence"]["pixels"].tobytes()
        assert a["correspondence"]["views"] == b["correspondence"]["views"]


def _masks(s, views):
    return [dict(mask=S.make_mask(s.size(v)[1], s.size(v)[0], seed=v), camera=S.camera_of(s, v)) for v in views]


@pytest.fixture(scope="module")
def scenes():
    from mve_b200 import dmrecon
    cache = {}

    def get(name):
        if name not in cache:
            s = golden_scene(name)
            cache[name] = (s, dmrecon.Scene.from_synth(s), _settings(s))
        return cache[name]
    yield get
    for _, sc, _ in cache.values():
        sc.close()


@pytest.mark.parametrize("name", S.SCENES)
def test_equals_host_route(scenes, name):
    s, sc, st = scenes(name)
    refs = _refs(s)
    full, maps = host_route(sc, s, st, refs, F_SET)
    got, stats = sc.reconstruct_pointset(st, refs, F_SET)
    same(got, full)
    assert stats.n_filled > 0 and len(got["vertices"]) > 0
    assert all(v["added"] for v in got["views"]) and len(got["colors"]) == len(got["vertices"])

    V = full["vertices"]
    lo = np.array([np.percentile(V[:, k], 20, method="nearest") for k in range(3)], np.float32)
    hi = np.array([np.percentile(V[:, k], 85, method="nearest") for k in range(3)], np.float32)
    fr = sorted(S.fill_fraction(m["depth"]) for m in maps)
    assert fr[0] < fr[-1]
    cases = [dict(with_normals=True, with_conf=True, poisson_normals=True),
             dict(F_SET, aabb=(lo, hi)),
             dict(F_SET, min_valid_fraction=float(np.nextafter(fr[0], np.float32(1)))),
             dict(correspondence=True)]
    for opts in cases:
        want, _ = host_route(sc, s, st, refs, opts)
        got, _ = sc.reconstruct_pointset(st, refs, opts)
        same(got, want)
        if "aabb" in opts:
            assert 0 < len(got["vertices"]) < len(V)
        if "min_valid_fraction" in opts:
            skipped = [v for v in got["views"] if not v["added"]]
            assert skipped and len(skipped) < len(refs) and all(v["n_points"] == 0 for v in skipped)
    masks = _masks(s, refs[:3])
    want, _ = host_route(sc, s, st, refs, F_SET, masks)
    got, _ = sc.reconstruct_pointset(st, refs, F_SET, masks)
    same(got, want)
    assert got["num_filtered"] > 0


def test_groups_out_of_order(scenes):
    """A budget that makes the planner build several groups, not in ref_views order: the same point set as one launch,
    the peak within the budget.  T6: its views do not all select each other, so groups interleave (in T0 every view
    selects every other one and groups follow the given order)."""
    from mve_b200 import dmrecon
    s, whole, st = scenes("T6")
    refs = _refs(s, seed=3)
    want, _ = whole.reconstruct_pointset(st, refs, F_SET)
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    single = max(sc.working_set(st, [r]) for r in refs)
    total = sc.working_set(st, refs)
    # the call keeps the point-set workspace of the largest map free in every plan: far below 256 bytes per pixel
    px = max(int(np.prod(whole.level(r, st.scale).shape[:2])) for r in refs)
    slack = 256 * px + (1 << 20)
    chosen = None
    for avail in np.linspace(single + slack, total, 40).astype(np.int64).tolist():
        # every plan the call may make in [avail - slack, avail] has the same number of groups and runs a view before one
        # that comes earlier in ref_views
        plans = [sc.plan_batches(st, refs, int(a)) for a in np.linspace(avail - slack, avail, 9).astype(np.int64)]
        n = plans[0][0]
        if n >= 2 and all(p[0] == n and (np.diff(p[1]) < 0).any() for p in plans):
            chosen = (avail, n)
            break
    assert chosen, "no budget gives an out-of-order grouping"
    budget = fixed + chosen[0]
    sc.set_image_source(lambda v: s.images[v], budget)
    got, stats = sc.reconstruct_pointset(st, refs, F_SET)
    m = sc.memory_stats()
    same(got, want)
    assert m.n_groups == chosen[1] >= 2 and stats.n_patch_launches == m.n_groups
    assert m.peak <= m.budget == budget, m.as_dict()
    sc.close()


@pytest.mark.parametrize("channels", [1, 4])
def test_colours_at_scale_0(channels):
    """At scale 0 the level is the `undistorted` image; for 1 and 4 channels the point colours are what scene2pset makes of
    the raw image: grey expanded to r = g = b, alpha never read."""
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    assert s.scale == 0
    rng = np.random.default_rng(channels)
    raw = {}
    for v in range(s.n_views):
        img = s.images[v]
        if channels == 1:
            raw[v] = np.ascontiguousarray(img[:, :, 1])
        else:
            raw[v] = np.ascontiguousarray(np.concatenate([img, rng.integers(0, 256, img.shape[:2] + (1,), dtype=np.uint8)], 2))
    sc = dmrecon.Scene(s.n_views)
    for v in range(s.n_views):
        sc.set_view(v, raw[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    sc.set_features(s.feat_pos, s.feat_refs)
    st = _settings(s)
    refs = _refs(s, seed=2)
    want, _ = host_route(sc, s, st, refs, F_SET, images=raw)
    got, _ = sc.reconstruct_pointset(st, refs, F_SET)
    same(got, want)
    c = got["colors"]
    if channels == 1:
        assert (c[:, 0] == c[:, 1]).all() and (c[:, 0] == c[:, 2]).all()
    assert (c[:, 3] == 1.0).all()
    sc.close()


def _handle(options=None, device=0):
    from mve_b200 import depthmap as D
    o, opt = D._options(options)
    L = D._pset_lib()
    h = C.c_void_p()
    D._check(L.b200mvs_pset_create(device, C.byref(opt), C.byref(h)))
    return L, h, o


def _add(L, h, sc, st, refs, progress=None):
    from mve_b200 import depthmap as D
    r = (C.c_int32 * len(refs))(*refs)
    recs = (D._PsetView * len(refs))()
    failed = C.c_int32(-1)
    rc = L.b200mvs_pset_add_reconstruction(h, sc._h, C.byref(st), len(refs), r, progress, None, C.byref(failed), recs)
    return rc, failed.value, L.b200mvs_last_error(None).decode(), recs


def _state(L, h, o):
    from mve_b200 import depthmap as D
    return D._finish(L, h, o, None, [])


def test_rejected_handles(scenes):
    from mve_b200 import dmrecon
    s, sc, st = scenes("T0")
    L, h, o = _handle(F_SET)
    try:
        rc, _, msg, _ = _add(L, None, sc, st, [0])
        assert rc == dmrecon.ERR_INVALID_ARG and "null handle" in msg
        assert L.b200mvs_pset_clip_masks(h, 0, None, None, None, None, None) == 0
        rc, _, msg, _ = _add(L, h, sc, st, [0])
        assert rc == dmrecon.ERR_INVALID_ARG and "masks have been applied" in msg, msg
    finally:
        L.b200mvs_pset_destroy(h)


def test_handle_on_another_device(scenes):
    import torch
    from mve_b200 import dmrecon
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    s, sc, st = scenes("T0")
    L, h, o = _handle(F_SET, device=1)
    try:
        rc, _, msg, _ = _add(L, h, sc, st, [0])
        assert rc == dmrecon.ERR_INVALID_ARG and "the handle is on device 1, the context on device 0" in msg, msg
    finally:
        L.b200mvs_pset_destroy(h)


def test_failure_and_cancellation_leave_the_handle_alone(scenes):
    from mve_b200 import dmrecon
    s, sc, st = scenes("T0")
    refs = _refs(s, seed=3)
    full, _ = sc.reconstruct_pointset(st, refs, F_SET)
    L, h, o = _handle(F_SET)
    try:
        # one earlier call's points are in the handle; the failing calls below must leave them as they are
        rc, _, _, _ = _add(L, h, sc, st, refs[:2])
        assert rc == 0
        before = _state(L, h, o)
        # a view no feature sees: its global view selection is empty
        lonely = refs[2]
        g = dmrecon.Scene.from_synth(s)
        g.set_features(s.feat_pos, [r[r != lonely] for r in s.feat_refs])
        rc, failed, msg, _ = _add(L, h, g, st, refs)
        g.close()
        assert rc == dmrecon.ERR_GLOBAL_VS and failed == lonely and "Global View Selection failed" in msg
        same(_state(L, h, o), before)
        # every view cancelled
        prog = (dmrecon.Progress * len(refs))()
        for p in prog:
            p.cancelled = 1
        rc, _, _, _ = _add(L, h, sc, st, refs, prog)
        assert rc == dmrecon.ERR_CANCELLED
        same(_state(L, h, o), before)
    finally:
        L.b200mvs_pset_destroy(h)
    # one view cancelled: it adds nothing, the others are in, in order
    victim = 2
    prog = (dmrecon.Progress * len(refs))()
    prog[victim].cancelled = 1
    got, _ = sc.reconstruct_pointset(st, refs, F_SET, progress=prog)
    assert prog[victim].status == 5 and not got["views"][victim]["added"] and got["views"][victim]["n_points"] == 0
    keep = np.ones(len(full["vertices"]), bool)
    fv = full["views"][victim]
    keep[fv["first_index"]:fv["first_index"] + fv["n_points"]] = False
    for k in ARRAYS:
        assert got[k].tobytes() == full[k][keep].tobytes(), k
    assert all(v["added"] for j, v in enumerate(got["views"]) if j != victim)
