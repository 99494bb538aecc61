"""The device-resident point set (-m gpu): b200mvs_pset_create_on_device handles and b200mvs_pset_read_device, through
scene_pointset(on_device=True) and reconstruct_pointset(on_device=True).

The oracle of every case is a b200mvs_pset_create handle fed the same inputs; the device set must be byte for byte the
same: every array (float bits), n_points / n_colors / n_views, the per-view records, num_filtered and the correspondence.
Covered on T0, T5 and T6 through all three add routes (host maps, CUDA-tensor maps, add_reconstruction): the default
options, -n -c -s, -p, -S, a bounding box whose faces lie on vertex coordinates, -f skipping a view, -C, masks larger,
smaller and of the size of their map plus a view without one, and a colourless last view that its mask deletes (short
colour list).  Also: one handle fed by all three routes, add_reconstruction under a budget that runs groups out of order
(with the context's b200mvs_memory the same for both kinds of handle), growth over several reallocations, failure and
cancellation, rejected read buffers, read_device on a host-resident handle, and a read ordered after a caller's stream."""
import ctypes as C

import numpy as np
import pytest

from tests import pset_reference as S
from tests.test_gpu_reconstruct_pointset import ARRAYS, F_SET, _add, _refs, _state, same, scenes  # noqa: F401
from tests.util import golden_scene

pytestmark = pytest.mark.gpu
SENTINEL = -7.0


def host(r):
    """The result of an on_device call with its tensors copied to numpy (checked to be CUDA tensors of the right dtype)."""
    import torch
    out = dict(r)
    for k in ARRAYS:
        if r[k] is not None:
            assert isinstance(r[k], torch.Tensor) and r[k].is_cuda and r[k].dtype == torch.float32, k
            out[k] = r[k].cpu().numpy()
    if r["correspondence"] is not None:
        pix = r["correspondence"]["pixels"]
        assert pix.is_cuda and pix.dtype == getattr(torch, "uint32", torch.int32)
        out["correspondence"] = dict(r["correspondence"], pixels=pix.cpu().numpy().view(np.uint32))
    return out


def _handle(options, on_device):
    from mve_b200 import depthmap as D
    o, opt = D._options(options)
    L = D._pset_lib()
    return L, D._create(L, 0, opt, on_device), o


@pytest.fixture(scope="module")
def maps(scenes):
    cache = {}

    def get(name):
        if name not in cache:
            s, sc, st = scenes(name)
            refs = _refs(s)
            m, _ = sc.reconstruct(st, refs, want=("depth",))
            cache[name] = (s, sc, st, refs, [x["depth"] for x in m])
        return cache[name]
    return get


def _cases(s, sc, st, refs, depths):
    """(name, options, masks, colourless last view) of every option case."""
    from mve_b200 import depthmap as D
    V = D.scene_pointset([dict(id=v, depth=depths[j], camera=S.camera_of(s, v)) for j, v in enumerate(refs)])["vertices"]
    lo = np.array([np.percentile(V[:, k], 20, method="nearest") for k in range(3)], np.float32)
    hi = np.array([np.percentile(V[:, k], 85, method="nearest") for k in range(3)], np.float32)
    fr = sorted(S.fill_fraction(d) for d in depths)
    sized = []
    for j, (fx, fy) in enumerate([(2, 2), (0.5, 0.5), (1, 1)]):
        h, w = depths[j].shape
        mh, mw = max(2, int(h * fy)), max(2, int(w * fx))
        sized.append(dict(mask=S.make_mask(mh, mw, seed=refs[j]), camera=S.camera_of(s, refs[j])))
    last = refs[-1]
    h, w = depths[-1].shape
    wipe = [dict(mask=S.make_mask(*depths[0].shape, seed=1), camera=S.camera_of(s, refs[0])),
            dict(mask=np.zeros((h, w), np.uint8), camera=S.camera_of(s, last))]
    return [("defaults", {}, None, False), ("nsc", F_SET, None, False),
            ("poisson", dict(with_normals=True, with_conf=True, poisson_normals=True), None, False),
            ("scale", dict(with_normals=True, with_scale=True, scale_factor=1.75), None, False),
            ("box", dict(F_SET, aabb=(lo, hi)), None, False),
            ("fill", dict(F_SET, min_valid_fraction=float(np.nextafter(fr[0], np.float32(1)))), None, False),
            ("corr", dict(correspondence=True), None, False),
            ("masks", F_SET, sized, False),
            ("colourless", F_SET, wipe, True)]


@pytest.mark.parametrize("name", S.SCENES)
def test_routes_equal_host_handle(maps, name):
    import torch
    from mve_b200 import depthmap as D
    s, sc, st, refs, depths = maps(name)
    dev = "cuda:%d" % sc.device
    for case, opts, masks, colourless in _cases(s, sc, st, refs, depths):
        views = [dict(id=v, depth=depths[j], camera=S.camera_of(s, v),
                      color=None if colourless and j == len(refs) - 1 else sc.level(v, st.scale)) for j, v in enumerate(refs)]
        views_d = [dict(x, depth=torch.from_numpy(x["depth"]).to(dev),
                        color=None if x["color"] is None else torch.from_numpy(x["color"]).to(dev)) for x in views]
        want = D.scene_pointset(views, opts, masks)
        assert len(want["vertices"]) > 0, case
        for route in (views, views_d):
            got = D.scene_pointset(route, opts, masks, on_device=True)
            same(host(got), want)
        if case == "box":
            # the faces are vertex coordinates: points lie on them and are kept
            assert ((want["vertices"] == opts["aabb"][0]) | (want["vertices"] == opts["aabb"][1])).any()
        if case == "fill":
            assert any(not v["added"] for v in want["views"])
        if case == "colourless":
            assert want["num_filtered"] >= want["views"][-1]["n_points"] > 0
            assert len(want["colors"]) > len(want["vertices"])
        if masks and not colourless:
            assert want["num_filtered"] > 0
        if not colourless:
            want_r, _ = sc.reconstruct_pointset(st, refs, opts, masks)
            got_r, _ = sc.reconstruct_pointset(st, refs, opts, masks, on_device=True)
            same(host(got_r), want_r)


def _feed(L, h, sc, st, refs, depths, s):
    """One handle fed by all three routes: host maps, CUDA-tensor maps, add_reconstruction."""
    import torch
    from mve_b200 import depthmap as D
    recs = []
    for j in (0, 1):
        v = refs[j]
        dm = np.ascontiguousarray(depths[j])
        col = np.ascontiguousarray(sc.level(v, st.scale))
        cam = D._camera(S.camera_of(s, v))
        r = D._PsetView()
        if j == 0:
            rc = L.b200mvs_pset_add_view(h, v, D._p(dm), dm.shape[1], dm.shape[0], D._p(col), 3, C.byref(cam), C.byref(r))
        else:
            td, tc = torch.from_numpy(dm).cuda(), torch.from_numpy(col).cuda()
            rc = L.b200mvs_pset_add_view_device(h, v, C.c_void_p(td.data_ptr()), dm.shape[1], dm.shape[0], C.c_void_p(tc.data_ptr()),
                                                3, C.byref(cam), C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(r))
        assert rc == 0
        recs.append(D._view_record(v, r))
    rc, _, msg, rr = _add(L, h, sc, st, refs[2:])
    assert rc == 0, msg
    return recs + [D._view_record(v, rr[j]) for j, v in enumerate(refs[2:])]


@pytest.mark.parametrize("options", [F_SET, dict(correspondence=True)], ids=["nsc", "corr"])
def test_mixed_routes(maps, options):
    from mve_b200 import depthmap as D
    s, sc, st, refs, depths = maps("T6")
    out = []
    for on_device in (False, True):
        L, h, o = _handle(options, on_device)
        try:
            recs = _feed(L, h, sc, st, refs, depths, s)
            out.append(D._finish(L, h, o, None, recs, 0 if on_device else None))
        finally:
            L.b200mvs_pset_destroy(h)
    same(host(out[1]), out[0])
    assert len(out[0]["vertices"]) > 0


def test_groups_out_of_order_and_memory(scenes):
    """A budget that makes the planner run several groups, not in ref_views order: the same set from both kinds of handle,
    and the context's b200mvs_memory identical (the device set is not in the budget)."""
    from mve_b200 import dmrecon
    s, whole, st = scenes("T6")
    refs = _refs(s, seed=3)
    probe = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = probe.memory_stats().fixed
    single = max(probe.working_set(st, [r]) for r in refs)
    total = probe.working_set(st, refs)
    px = max(int(np.prod(whole.level(r, st.scale).shape[:2])) for r in refs)
    slack = 256 * px + (1 << 20)
    chosen = None
    for avail in np.linspace(single + slack, total, 40).astype(np.int64).tolist():
        plans = [probe.plan_batches(st, refs, int(a)) for a in np.linspace(avail - slack, avail, 9).astype(np.int64)]
        if plans[0][0] >= 2 and all(p[0] == plans[0][0] and (np.diff(p[1]) < 0).any() for p in plans):
            chosen = avail
            break
    probe.close()
    assert chosen, "no budget gives an out-of-order grouping"
    res, mem = [], []
    for on_device in (False, True):
        sc = dmrecon.Scene.from_synth(s, lazy=True)
        sc.set_image_source(lambda v: s.images[v], fixed + chosen)
        got, _ = sc.reconstruct_pointset(st, refs, F_SET, on_device=on_device)
        res.append(got)
        mem.append(sc.memory_stats().as_dict())
        sc.close()
    same(host(res[1]), res[0])
    assert mem[0] == mem[1] and mem[0]["n_groups"] >= 2, mem


def test_growth_over_reallocations(maps):
    """Lists start at 2^14 entries, at least double, and jump to what a view needs when that is more: small views of more
    than 2^15 points (a doubling), a 1500 x 1500 map of more than three times their points (a jump to exactly the points
    so far), then small views again (a doubling) reallocate at least three times."""
    from mve_b200 import depthmap as D
    s, sc, st, refs, depths = maps("T0")
    big = S.hand_map(1500, 1500, float(np.median(depths[0][depths[0] > 0])), seed=5)
    cam = S.camera_of(s, refs[0])
    small = [dict(id=v, depth=depths[j], camera=S.camera_of(s, v), color=sc.level(v, st.scale)) for j, v in enumerate(refs)]
    views = small + [dict(id=99, depth=big, camera=cam)] + small + small
    want = D.scene_pointset(views, F_SET)
    got = D.scene_pointset(views, F_SET, on_device=True)
    same(host(got), want)
    pre = sum(v["n_points"] for v in want["views"][:len(small)])
    assert pre > 2 * (1 << 14) and want["views"][len(small)]["n_points"] > 3 * pre, want["views"]
    n = len(want["vertices"])
    assert got["info"]["device_bytes"] >= n * 4 * (3 + 3 + 1 + 1)


def test_failure_and_cancellation_leave_the_set_alone(scenes):
    from mve_b200 import dmrecon
    s, sc, st = scenes("T0")
    refs = _refs(s, seed=3)
    L, h, o = _handle(F_SET, True)
    try:
        rc, _, _, _ = _add(L, h, sc, st, refs[:2])
        assert rc == 0
        before = host(_state_dev(L, h, o))
        assert len(before["vertices"]) > 0
        lonely = refs[2]
        g = dmrecon.Scene.from_synth(s)
        g.set_features(s.feat_pos, [r[r != lonely] for r in s.feat_refs])
        rc, failed, msg, _ = _add(L, h, g, st, refs)
        g.close()
        assert rc == dmrecon.ERR_GLOBAL_VS and failed == lonely, msg
        same(host(_state_dev(L, h, o)), before)
        same(_state(L, h, o), before)
        prog = (dmrecon.Progress * len(refs))()
        for p in prog:
            p.cancelled = 1
        rc, _, _, _ = _add(L, h, sc, st, refs, prog)
        assert rc == dmrecon.ERR_CANCELLED
        same(host(_state_dev(L, h, o)), before)
        # the handle goes on: a later call appends after the same points
        rc, _, _, _ = _add(L, h, sc, st, refs[2:])
        assert rc == 0
        after = host(_state_dev(L, h, o))
        assert after["vertices"][:len(before["vertices"])].tobytes() == before["vertices"].tobytes()
    finally:
        L.b200mvs_pset_destroy(h)


def _state_dev(L, h, o):
    from mve_b200 import depthmap as D
    return D._finish(L, h, o, None, [], 0)


def test_read_device_rejects_and_orders():
    import torch
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    depth = S.hand_map(120, 160, 3.0, seed=1)
    view = dict(id=0, depth=depth, camera=S.camera_of(s, 0), color=s.images[0][:120, :160].copy())
    for on_device in (False, True):
        L, h, o = _handle(F_SET, on_device)
        try:
            v = view
            dm, col = np.ascontiguousarray(v["depth"]), np.ascontiguousarray(v["color"])
            cam = D._camera(v["camera"])
            assert L.b200mvs_pset_add_view(h, 0, D._p(dm), dm.shape[1], dm.shape[0], D._p(col), 3, C.byref(cam), None) == 0
            want = D._finish(L, h, o, None, [])
            n = len(want["vertices"])
            assert n > 0
            # read_device on either kind of handle equals read
            same(host(D._finish(L, h, o, None, [], 0)), want)
            good = torch.empty((n, 3), dtype=torch.float32, device="cuda:0")
            pageable = np.zeros((n, 3), np.float32)
            pinned = torch.zeros((n, 3), dtype=torch.float32, pin_memory=True)
            spare = torch.zeros(3 * n + 4, dtype=torch.float32, device="cuda:0")
            pix = torch.zeros((n, 2), dtype=torch.int32, device="cuda:0")
            cases = [(dict(vertices=pageable.ctypes.data), "vertices", "pageable host memory"),
                     (dict(normals=pinned.data_ptr()), "normals", "pinned host memory"),
                     (dict(vertices=good.data_ptr(), normals=spare.data_ptr() + 2), "normals", "not 4-byte aligned"),
                     (dict(pixels=pix.data_ptr()), "pixels_xy", "without correspondence")]
            if torch.cuda.device_count() > 1:
                other = torch.zeros((n, 3), dtype=torch.float32, device="cuda:1")
                cases.append((dict(normals=other.data_ptr()), "normals", "memory of device"))
            for bufs, field, words in cases:
                args = [bufs.get(k) for k in ("vertices", "normals", "colors", "values", "confidences", "pixels")]
                rc = L.b200mvs_pset_read_device(h, *[None if a is None else C.c_void_p(a) for a in args], None)
                msg = L.b200mvs_depthmap_last_error().decode()
                assert rc == dmrecon.ERR_INVALID_ARG and field in msg and words in msg, msg
            torch.cuda.synchronize()
            assert not pageable.any() and not pinned.any().item() and not spare.any().item() and not pix.any().item()
            # a read on a side stream after a delayed sentinel fill of the same buffer returns the points
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(200_000_000)
                good.fill_(SENTINEL)
            rc = L.b200mvs_pset_read_device(h, C.c_void_p(good.data_ptr()), None, None, None, None, None, C.c_void_p(side.cuda_stream))
            assert rc == 0
            assert good.cpu().numpy().tobytes() == want["vertices"].tobytes()
        finally:
            L.b200mvs_pset_destroy(h)
