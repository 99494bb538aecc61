"""Masks from device memory (-m gpu): b200mvs_set_view_mask_device gives every map, counter and point of
b200mvs_set_view_mask with the same bytes, on every route, under a budget and across frontier resumes, and its block is
counted in b200mvs_memory.fixed; b200mvs_pset_clip_masks_device gives the point set of b200mvs_pset_clip_masks on both
kinds of handle."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from tests import pset_reference as S
from tests.test_gpu_recon_mask import COUNTERS, KEYS, MODES, _half_planes, _settings, _silhouettes
from tests.test_scene_pointset_reference import HAND, MASKS
from tests.util import golden_scene

pytestmark = pytest.mark.gpu


def _cuda(m, pitched=False):
    """The mask as a CUDA tensor; pitched: a column slice of a wider tensor (row stride > width)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    if not pitched:
        return t
    h, w = t.shape
    wide = torch.full((h, w + 13), 7, dtype=torch.uint8, device=t.device)
    wide[:, 5:5 + w] = t
    s = wide[:, 5:5 + w]
    assert s.stride() == (w + 13, 1)
    return s


def _set_masks(sc, refs, masks, on_device, pitched=False):
    for v in refs:
        m = None if masks is None else masks.get(v)
        if m is None or not on_device:
            sc.set_view_mask(v, m)
        else:
            sc.set_view_mask(v, _cuda(m, pitched), on_device=True)


def _run(sc, st, refs, masks, on_device, mode="default", route="host", pitched=False):
    """Maps (numpy) and counters of one reconstruction with host or device masks, by route."""
    import torch
    sc.set_patch_mode(0, MODES[mode])
    _set_masks(sc, refs, masks, on_device, pitched)
    if route == "device":
        maps, stats = sc.reconstruct(st, refs, on_device=True)
        torch.cuda.synchronize()
        maps = [{k: v.cpu().numpy() for k, v in m.items()} for m in maps]
    else:
        maps, stats = sc.reconstruct(st, refs)
    return maps, {k: getattr(stats, k) for k in COUNTERS}


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for k in KEYS:
            assert x[k].tobytes() == y[k].tobytes(), k


def _masks(s, refs, kind):
    if kind == "half":
        return _half_planes(s, refs)
    if kind in ("identity", "zero"):
        rng = np.random.default_rng(11)
        out = {}
        for v in refs:
            w, h = s.size(v)
            out[v] = rng.integers(1, 256, (h, w)).astype(np.uint8) if kind == "identity" else np.zeros((h, w), np.uint8)
        return out
    return _silhouettes(s, refs, kind)


@pytest.mark.parametrize("name", ["T0", "T2", "T5", "T6"])
@pytest.mark.parametrize("kind", ["photo", "map", (37, 29), (400, 300), "identity", "zero", "half"])
def test_maps_and_counters_equal_host_masks(name, kind):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    masks = _masks(s, refs, kind)
    sc = dmrecon.Scene.from_synth(s)
    want, wc = _run(sc, st, refs, masks, False)
    for route, pitched in (("host", False), ("host", True), ("device", False)):
        got, c = _run(sc, st, refs, masks, True, route=route, pitched=pitched)
        _same(got, want)
        assert c == wc, (route, pitched)
    sc.close()


@pytest.mark.parametrize("mode", ["warp", "thread"])
def test_patch_modes(mode):
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    masks = _silhouettes(s, refs)
    sc = dmrecon.Scene.from_synth(s)
    want, wc = _run(sc, st, refs, masks, False, mode)
    got, c = _run(sc, st, refs, masks, True, mode, pitched=True)
    _same(got, want)
    assert c == wc
    sc.close()


def test_reconstruct_pointset_equals_host_masks():
    import torch
    from mve_b200 import dmrecon
    from tests.test_gpu_reconstruct_pointset import F_SET, same
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    masks = _silhouettes(s, refs)
    sc = dmrecon.Scene.from_synth(s)
    _set_masks(sc, refs, masks, False)
    want, ws = sc.reconstruct_pointset(st, refs, F_SET)
    _set_masks(sc, refs, masks, True)
    got, gs = sc.reconstruct_pointset(st, refs, F_SET)
    same(got, want)
    assert {k: getattr(gs, k) for k in COUNTERS} == {k: getattr(ws, k) for k in COUNTERS}
    on_dev, _ = sc.reconstruct_pointset(st, refs, F_SET, on_device=True)
    torch.cuda.synchronize()
    for key in ("vertices", "normals", "confidences", "values", "colors"):
        assert on_dev[key].cpu().numpy().tobytes() == want[key].tobytes(), key
    sc.close()


def test_budget_groups_and_frontier_resume():
    """A lazy source whose budget splits the batch into groups out of order, then a frontier small enough to resume: device
    masks give the host masks' maps, with the groups and evictions planned with the mask bytes in `fixed`."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    masks = _silhouettes(s, refs)
    mask_bytes = sum(m.size for m in masks.values())
    plain = dmrecon.Scene.from_synth(s)
    want, wc = _run(plain, st, refs, masks, False)
    plain.close()

    results = []
    for on_device in (False, True):
        lazy = dmrecon.Scene.from_synth(s, lazy=True)
        fixed0 = lazy.memory_stats().fixed
        _set_masks(lazy, refs, masks, on_device)
        fixed = lazy.memory_stats().fixed
        assert fixed == fixed0 + (mask_bytes if on_device else 0)
        single = max(lazy.working_set(st, [r]) for r in refs)
        total = lazy.working_set(st, refs)
        chosen = None
        for avail in np.linspace(single, total, 40).astype(np.int64).tolist():
            n, groups = lazy.plan_batches(st, refs, int(avail))
            if n >= 2 and (np.diff(groups) < 0).any():
                chosen = (avail, n)
                break
        assert chosen, "no budget gives an out-of-order grouping"
        lazy.set_image_source(lambda v: s.images[v], fixed + chosen[0])
        got, c = _run(lazy, st, refs, masks, on_device)
        mem = lazy.memory_stats()
        assert mem.n_groups == chosen[1] and mem.fixed == fixed and mem.peak <= mem.budget
        _same(got, want)
        # the per-view counts are those of one launch; rounds, launches and barriers are the groups' (compared below)
        for k in ("n_filled", "n_seeds_processed"):
            assert c[k] == wc[k], k
        lazy.set_frontier_capacity(0.01, 1)
        again, c2 = _run(lazy, st, refs, masks, on_device)
        assert lazy.frontier_info()["resumes"] >= 1
        _same(again, want)
        results.append((chosen, mem.n_groups, mem.n_evictions, c, c2))
        lazy.close()
    assert results[0] == results[1]


def test_memory_accounting_and_replacement():
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    st = _settings(s)
    refs = [0, 3]
    sc = dmrecon.Scene.from_synth(s)
    masks = _silhouettes(s, refs)
    want, wc = _run(sc, st, refs, masks, False)
    sc.set_view_mask(0, None)
    sc.set_view_mask(3, None)
    m0 = sc.memory_stats()
    sc.set_view_mask(0, _cuda(masks[0]), on_device=True)
    m1 = sc.memory_stats()
    assert m1.fixed - m0.fixed == m1.resident - m0.resident == masks[0].size
    sc.set_view_mask(3, _cuda(masks[3], pitched=True), on_device=True)
    m2 = sc.memory_stats()
    assert m2.fixed - m1.fixed == m2.resident - m1.resident == masks[3].size
    small = np.ones((29, 37), np.uint8)
    sc.set_view_mask(3, _cuda(small), on_device=True)                   # a device mask replaces a device mask
    m3 = sc.memory_stats()
    assert m3.fixed - m1.fixed == m3.resident - m1.resident == small.size
    sc.set_view_mask(3, masks[3])                                       # a host mask replaces it and frees the block
    assert (sc.memory_stats().fixed, sc.memory_stats().resident) == (m1.fixed, m1.resident)
    maps, stats = sc.reconstruct(st, refs)                               # view 0 device, view 3 host
    _same(maps, want)
    assert {k: getattr(stats, k) for k in COUNTERS} == wc
    sc.set_view_mask(0, None)
    after = sc.memory_stats()
    assert after.fixed == m0.fixed
    sc.set_view_mask(0, _cuda(masks[0]), on_device=True)
    sc.set_view_mask(0, None, on_device=True)
    assert sc.memory_stats().fixed == m0.fixed

    # a mask beyond the budget: B200MVS_ERR_NO_MEMORY, and the previous mask keeps working
    sc.set_view_mask(0, _cuda(masks[0]), on_device=True)
    fixed = sc.memory_stats().fixed
    sc.set_image_source(lambda v: s.images[v], fixed + 4096)
    huge = torch.zeros((2048, 2048), dtype=torch.uint8, device="cuda")
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.set_view_mask(0, huge, on_device=True)
    assert e.value.code == dmrecon.ERR_NO_MEMORY and "b200mvs_set_view_mask_device" in str(e.value)
    assert sc.memory_stats().fixed == fixed
    sc.set_image_source(lambda v: s.images[v], 0)
    maps, stats = sc.reconstruct(st, refs)
    _same(maps, want)
    assert {k: getattr(stats, k) for k in COUNTERS} == wc
    sc.close()


def test_source_is_copied_and_ordered():
    """Overwriting the source right after the call changes nothing; a mask written on a side stream behind a delay and
    passed with that stream is read after the write."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = [0, 4, 7]
    masks = _silhouettes(s, refs)
    sc = dmrecon.Scene.from_synth(s)
    want, wc = _run(sc, st, refs, masks, False)
    for v in refs:
        t = _cuda(masks[v])
        sc.set_view_mask(v, t, on_device=True)
        t.fill_(0)
    maps, stats = sc.reconstruct(st, refs)
    _same(maps, want)
    assert {k: getattr(stats, k) for k in COUNTERS} == wc

    side = torch.cuda.Stream()
    srcs = {v: _cuda(masks[v]) for v in refs}
    dst = {v: torch.zeros_like(srcs[v]) for v in refs}
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for v in refs:
            torch.cuda._sleep(50_000_000)
            dst[v].copy_(srcs[v])
            sc.set_view_mask(v, dst[v], on_device=True)
    maps, stats = sc.reconstruct(st, refs)
    _same(maps, want)
    assert {k: getattr(stats, k) for k in COUNTERS} == wc
    sc.close()


# ---- silhouette clipping with CUDA masks ----
def _np(r):
    """The arrays of a scene_pointset result as numpy arrays."""
    out = dict(r)
    for k in ("vertices", "normals", "colors", "values", "confidences"):
        if out[k] is not None and not isinstance(out[k], np.ndarray):
            out[k] = out[k].cpu().numpy()
    return out


def _same_set(a, b):
    a, b = _np(a), _np(b)
    for k in ("vertices", "normals", "colors", "values", "confidences"):
        assert (a[k] is None) == (b[k] is None), k
        if a[k] is not None:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
    assert a["views"] == b["views"] and a["num_filtered"] == b["num_filtered"]


def _views_and_masks(tmp, name, **kw):
    from mve_b200 import synth
    sc = S.build_scene(tmp, name, **kw)
    s = sc["scene"]
    drop = kw.get("drop_color", ())
    views = []
    for v in sorted(sc["maps"]):
        vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
        col = None
        if v not in drop:
            f = "undist-L%d.mvei" % s.scale if s.scale else "undistorted.mvei"
            col = synth.read_mvei(os.path.join(vd, f)) if os.path.exists(os.path.join(vd, f)) else None
            if col is not None and col.shape[:2] != sc["maps"][v].shape:
                col = None
        views.append(dict(id=v, depth=sc["maps"][v], camera=S.camera_of(s, v), color=col))
    masks = [dict(mask=m, camera=S.camera_of(s, v)) for v, m in sorted(sc["masks"].items()) if m.ndim == 2]
    return views, masks


def _cuda_mask_dicts(masks, pitched):
    return [dict(m, mask=_cuda(m["mask"], pitched and k % 2 == 0)) for k, m in enumerate(masks)]


@pytest.mark.parametrize("name", S.SCENES)
def test_scene_pointset_clip_equals_numpy_masks(name):
    from mve_b200 import depthmap as D
    F = dict(with_normals=True, with_conf=True, with_scale=True)
    with tempfile.TemporaryDirectory() as tmp:
        views, masks = _views_and_masks(tmp, name, hand_views=HAND[name], mask_kinds=MASKS[name])
    assert masks
    for on_device in (False, True):
        want = D.scene_pointset(views, F, masks=masks, on_device=on_device)
        assert want["num_filtered"] > 0
        for pitched in (False, True):
            got = D.scene_pointset(views, F, masks=_cuda_mask_dicts(masks, pitched), on_device=on_device)
            _same_set(got, want)
            assert got["info"]["device_bytes"] == want["info"]["device_bytes"]


def test_short_colour_list_under_cuda_masks():
    from mve_b200 import depthmap as D
    with tempfile.TemporaryDirectory() as tmp:
        views, masks = _views_and_masks(tmp, "T0", hand_views=HAND["T0"], mask_kinds={0: "same", 3: "zero"}, drop_color=(3,))
    for on_device in (False, True):
        full = D.scene_pointset(views, on_device=on_device)
        want = D.scene_pointset(views, masks=masks, on_device=on_device)
        got = D.scene_pointset(views, masks=_cuda_mask_dicts(masks, True), on_device=on_device)
        _same_set(got, want)
        assert len(_np(got)["colors"]) == len(_np(full)["colors"]) > len(_np(got)["vertices"])


def test_reconstruct_pointset_with_cuda_masks():
    from mve_b200 import dmrecon
    from tests.test_gpu_reconstruct_pointset import F_SET, _masks as pset_masks
    s = golden_scene("T5")
    st = _settings(s)
    refs = np.random.default_rng(1).permutation(s.n_views).tolist()
    masks = pset_masks(s, refs[:3])
    sc = dmrecon.Scene.from_synth(s)
    for on_device in (False, True):
        want, _ = sc.reconstruct_pointset(st, refs, F_SET, masks, on_device=on_device)
        got, _ = sc.reconstruct_pointset(st, refs, F_SET, _cuda_mask_dicts(masks, True), on_device=on_device)
        assert want["num_filtered"] > 0
        _same_set(got, want)
    sc.close()


@pytest.mark.parametrize("on_device", [False, True])
def test_rejected_clip_leaves_the_set_alone(on_device):
    """Host memory, a short row pitch and a NULL pitch array are rejected before anything runs: the set reads back as it
    was, and a valid call afterwards clips it."""
    from mve_b200 import depthmap as D
    with tempfile.TemporaryDirectory() as tmp:
        views, masks = _views_and_masks(tmp, "T0", hand_views=HAND["T0"], mask_kinds=MASKS["T0"])
    want = D.scene_pointset(views, masks=masks, on_device=on_device)
    L = D._pset_lib()
    _, opt = D._options(None)
    h = D._create(L, 0, opt, on_device)
    try:
        for v in views:
            dm = np.ascontiguousarray(v["depth"], np.float32)
            col = v["color"]
            cam = D._camera(v["camera"])
            r = D._PsetView()
            assert L.b200mvs_pset_add_view(h, v["id"], D._p(dm), dm.shape[1], dm.shape[0], D._p(col),
                                           0 if col is None else (1 if col.ndim == 2 else col.shape[2]), C.byref(cam), C.byref(r)) == 0

        def state():
            info = D._PsetInfo()
            assert L.b200mvs_pset_get_info(h, C.byref(info)) == 0
            n = int(info.n_points)
            verts = np.empty((n, 3), np.float32)
            assert L.b200mvs_pset_read(h, D._p(verts), None, None, None, None) == 0
            return n, int(info.n_colors), verts.tobytes()

        before = state()
        ts = [_cuda(m["mask"]) for m in masks]
        n = len(ts)
        ws = np.array([t.shape[1] for t in ts], np.int32)
        hs = np.array([t.shape[0] for t in ts], np.int32)
        good = ws.astype(np.int64)
        cams = (D._PsetCamera * n)(*[D._camera(m["camera"]) for m in masks])
        dev_ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        host = [np.ascontiguousarray(m["mask"]) for m in masks]
        host_ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in host])
        short = good.copy()
        short[-1] -= 1
        nf = C.c_uint64(0)
        fn = "b200mvs_pset_clip_masks_device"
        for ptrs, pitches, msg in ((host_ptrs, D._p(good), "%s: masks_dev[0] is pageable host memory, not device memory" % fn),
                                   (dev_ptrs, D._p(short), "%s: row_pitches[%d] is %d, less than widths[%d] (%d)"
                                    % (fn, n - 1, short[-1], n - 1, ws[-1])),
                                   (dev_ptrs, None, "%s: null argument" % fn)):
            rc = L.b200mvs_pset_clip_masks_device(h, n, ptrs, D._p(ws), D._p(hs), pitches, cams, None, C.byref(nf))
            assert rc == -1 and L.b200mvs_depthmap_last_error().decode() == msg
            assert state() == before
        assert L.b200mvs_pset_clip_masks_device(h, n, dev_ptrs, D._p(ws), D._p(hs), D._p(good), cams, None, C.byref(nf)) == 0
        assert nf.value == want["num_filtered"] > 0
        after = state()
        assert after[0] == len(want["vertices"]) and after[2] == _np(want)["vertices"].tobytes()
        rc = L.b200mvs_pset_clip_masks_device(h, n, dev_ptrs, D._p(ws), D._p(hs), D._p(good), cams, None, C.byref(nf))
        assert rc == -1 and "applied already" in L.b200mvs_depthmap_last_error().decode()
    finally:
        L.b200mvs_pset_destroy(h)
