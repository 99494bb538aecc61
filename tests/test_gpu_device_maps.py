"""Results in device memory (-m gpu): b200mvs_reconstruct_device, b200mvs_get_level_device and b200mvs_pset_add_view_device
through Scene.reconstruct(on_device=True), Scene.level(on_device=True) and scene_pointset with CUDA tensors.

Every result must be byte for byte what the host route gives on T0, T5 and T6: the maps of Scene.reconstruct (in a
permuted ref_views order, all maps and depth alone), every level of every view (also after eviction under a budget), and
the point sets of scene_pointset from numpy maps.  Also covered: a budget whose plan makes several groups out of ref_views
order, the caller's stream ordering the call after a delayed sentinel fill, a view cancelled before the call, and buffers
rejected before anything is written (host memory, pinned or pageable; a misaligned pointer; NULL depth; another device)."""
import ctypes as C

import numpy as np
import pytest

from tests import pset_reference as S
from tests.util import golden_scene

pytestmark = pytest.mark.gpu

MAPS = ("depth", "conf", "dz", "normal", "view_ids")
F_SET = dict(with_normals=True, with_conf=True, with_scale=True)
SENTINEL = -7


def _settings(s):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)


def _refs(s, seed=0):
    return np.random.default_rng(seed).permutation(s.n_views).tolist()


@pytest.fixture(scope="module")
def scenes():
    from mve_b200 import dmrecon
    cache = {}

    def get(name):
        if name not in cache:
            s = golden_scene(name)
            sc = dmrecon.Scene.from_synth(s)
            st = _settings(s)
            refs = _refs(s)
            host, _ = sc.reconstruct(st, refs)
            cache[name] = (s, sc, st, refs, host)
        return cache[name]
    yield get
    for v in cache.values():
        v[1].close()


def _equal(dev, host, keys=MAPS):
    assert sorted(dev) == sorted(keys)
    for k in keys:
        d = dev[k].cpu().numpy()
        assert d.dtype == host[k].dtype and d.shape == host[k].shape, k
        assert d.tobytes() == host[k].tobytes(), k


def _sentinel_out(host_maps, device):
    import torch
    dt = dict(depth=torch.float32, conf=torch.float32, dz=torch.float32, normal=torch.float32, view_ids=torch.int32)
    return [{k: torch.full(m[k].shape, SENTINEL, dtype=dt[k], device=device) for k in MAPS} for m in host_maps]


@pytest.mark.parametrize("name", S.SCENES)
def test_maps_and_levels_equal_host_route(scenes, name):
    import torch
    s, sc, st, refs, host = scenes(name)
    dev, stats = sc.reconstruct(st, refs, on_device=True)
    assert stats.n_filled > 0 and len(dev) == len(refs)
    for d, h in zip(dev, host):
        _equal(d, h)
        assert all(t.device == torch.device("cuda:%d" % sc.device) and t.is_contiguous() for t in d.values())
    only, _ = sc.reconstruct(st, refs, on_device=True, want=("depth",))
    for d, h in zip(only, host):
        _equal(d, h, ("depth",))
    for v in range(s.n_views):
        for level in range(sc.num_levels(v)):
            got = sc.level(v, level, on_device=True)
            assert got.dtype == torch.uint8 and got.is_cuda
            assert got.cpu().numpy().tobytes() == sc.level(v, level).tobytes(), (v, level)


def test_budget_splits_the_batch(scenes):
    """A budget that makes the planner build several groups, not in ref_views order (as in
    test_gpu_reconstruct_pointset.test_groups_out_of_order): the maps of the unbudgeted host route, the peak within the
    budget; afterwards the levels of evicted views are fetched again and equal the resident ones."""
    from mve_b200 import dmrecon
    s, whole, st, _, _ = scenes("T6")
    refs = _refs(s, seed=3)
    host, _ = whole.reconstruct(st, refs)
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    single = max(sc.working_set(st, [r]) for r in refs)
    total = sc.working_set(st, refs)
    chosen = None
    for avail in np.linspace(single, total, 40).astype(np.int64).tolist():
        n, groups = sc.plan_batches(st, refs, int(avail))
        if n >= 2 and (np.diff(groups) < 0).any():
            chosen = (int(avail), n)
            break
    assert chosen, "no budget gives an out-of-order grouping"
    budget = fixed + chosen[0]
    sc.set_image_source(lambda v: s.images[v], budget)
    dev, stats = sc.reconstruct(st, refs, on_device=True)
    m = sc.memory_stats()
    for d, h in zip(dev, host):
        _equal(d, h)
    assert m.n_groups == chosen[1] >= 2 and stats.n_patch_launches == m.n_groups
    assert m.peak <= m.budget == budget, m.as_dict()
    # room for two pyramids (20 bytes per texel at a row pitch of 4 texels): reading every view's
    # levels in turn evicts
    pyr = max(sum(20 * ((w + 3) & ~3) * h for h, w in (whole.level(v, k).shape[:2] for k in range(whole.num_levels(v))))
              for v in range(s.n_views))
    small = m.fixed + 2 * pyr + 4096
    sc.set_image_source(lambda v: s.images[v], small)
    evictions = sc.memory_stats().n_evictions
    for v in range(s.n_views):
        for level in range(sc.num_levels(v)):
            assert sc.level(v, level, on_device=True).cpu().numpy().tobytes() == whole.level(v, level).tobytes(), (v, level)
    m = sc.memory_stats()
    assert m.n_evictions > evictions and m.peak <= small, m.as_dict()
    sc.close()


def test_stream_orders_the_call(scenes):
    """The output tensors are filled with a sentinel on a side stream behind a long sleep; the call on that stream must
    write after the fill."""
    import torch
    s, sc, st, refs, host = scenes("T5")
    dev = torch.device("cuda:%d" % sc.device)
    out = [{k: torch.empty(m[k].shape, dtype=torch.float32 if k != "view_ids" else torch.int32, device=dev) for k in MAPS}
           for m in host]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        for d in out:
            for t in d.values():
                t.fill_(SENTINEL)
    got, _ = sc.reconstruct(st, refs, on_device=True, out=out, stream=side)
    assert got is not None and all(g is o for g, o in zip(got, out))
    for d, h in zip(out, host):
        _equal(d, h)


def test_cancelled_view_left_untouched(scenes):
    from mve_b200 import dmrecon
    s, sc, st, refs, host = scenes("T0")
    out = _sentinel_out(host, "cuda:%d" % sc.device)
    progress = (dmrecon.Progress * len(refs))()
    progress[1].cancelled = 1
    got, _ = sc.reconstruct(st, refs, on_device=True, out=out, progress=progress)
    for j, (d, h) in enumerate(zip(got, host)):
        if j == 1:
            assert progress[j].status == 5
            assert all((t == SENTINEL).all().item() for t in d.values())
        else:
            assert progress[j].status == 0
            _equal(d, h)


def test_rejected_buffers(scenes):
    """Host memory (pageable and pinned), a pointer 2 bytes off, NULL depth and memory of another device: each is
    B200MVS_ERR_INVALID_ARG naming the field, and nothing is written."""
    import torch
    from mve_b200 import dmrecon
    s, sc, st, refs, host = scenes("T0")
    L = dmrecon.lib()
    out = _sentinel_out(host, "cuda:%d" % sc.device)
    refs_c = (C.c_int32 * len(refs))(*refs)
    pageable = np.zeros(host[0]["conf"].size + 16, np.float32)
    pinned = torch.zeros(host[0]["conf"].size + 16, dtype=torch.float32, pin_memory=True)
    spare = torch.zeros(host[0]["conf"].size + 16, dtype=torch.float32, device="cuda:%d" % sc.device)
    cases = [("conf", pageable.ctypes.data, "pageable host memory"), ("conf", pinned.data_ptr(), "pinned host memory"),
             ("normal", spare.data_ptr() + 2, "not 4-byte aligned"), ("depth", None, "depth (view %d) is NULL" % refs[1])]
    if torch.cuda.device_count() > 1:
        other = torch.zeros(host[0]["conf"].size, dtype=torch.float32, device="cuda:%d" % ((sc.device + 1) % torch.cuda.device_count()))
        cases.append(("dz", other.data_ptr(), "memory of device"))
    for field, ptr, words in cases:
        maps = (dmrecon._Maps * len(refs))()
        for j, d in enumerate(out):
            for k in MAPS:
                setattr(maps[j], k, d[k].data_ptr())
        setattr(maps[1], field, ptr)
        rc = L.b200mvs_reconstruct_device(sc._h, C.byref(st), len(refs), refs_c, maps, None, None, None, None)
        msg = L.b200mvs_last_error(None).decode()
        assert rc == dmrecon.ERR_INVALID_ARG, (field, rc, msg)
        assert "maps_dev[1].%s" % field in msg and words in msg, msg
        assert maps[0].width == 0
        torch.cuda.synchronize()
        assert all((t == SENTINEL).all().item() for d in out for t in d.values())
        assert not pageable.any() and not pinned.any().item() and not spare.any().item()
    rc = L.b200mvs_get_level_device(sc._h, 0, 0, None, None, C.c_void_p(pageable.ctypes.data), None)
    assert rc == dmrecon.ERR_INVALID_ARG and "rgb_dev" in L.b200mvs_last_error(None).decode()
    assert not pageable.any()


def _colour(level, channels, seed):
    if channels == 3:
        return level
    if channels == 1:
        return np.ascontiguousarray(level[:, :, 1])
    alpha = np.random.default_rng(seed).integers(0, 256, level.shape[:2], dtype=np.uint8)
    return np.ascontiguousarray(np.concatenate([level, alpha[:, :, None]], -1))


@pytest.mark.parametrize("name", S.SCENES)
def test_pointset_from_device_maps(scenes, name):
    import torch
    from mve_b200 import depthmap as D
    from tests.test_gpu_reconstruct_pointset import same
    s, sc, st, refs, host = scenes(name)
    dev = "cuda:%d" % sc.device
    fr = sorted(S.fill_fraction(m["depth"]) for m in host)
    V = D.scene_pointset([dict(id=v, depth=host[j]["depth"], camera=S.camera_of(s, v)) for j, v in enumerate(refs)])["vertices"]
    lo = np.array([np.percentile(V[:, k], 20, method="nearest") for k in range(3)], np.float32)
    hi = np.array([np.percentile(V[:, k], 85, method="nearest") for k in range(3)], np.float32)
    cases = [(F_SET, 3), (F_SET, 1), (F_SET, 4), (dict(with_normals=True, with_conf=True, poisson_normals=True), 3),
             (dict(correspondence=True), 4), (dict(F_SET, aabb=(lo, hi)), 3),
             (dict(F_SET, min_valid_fraction=float(np.nextafter(fr[0], np.float32(1)))), 1)]
    masks = [dict(mask=S.make_mask(s.size(v)[1], s.size(v)[0], seed=v), camera=S.camera_of(s, v)) for v in refs[:3]]
    for k, (opts, channels) in enumerate(cases + [(F_SET, 3)]):
        mk = masks if k == len(cases) else None
        views_h = [dict(id=v, depth=host[j]["depth"], camera=S.camera_of(s, v),
                        color=_colour(sc.level(v, st.scale), channels, v)) for j, v in enumerate(refs)]
        views_d = [dict(id=x["id"], camera=x["camera"], depth=torch.from_numpy(x["depth"]).to(dev),
                        color=torch.from_numpy(x["color"]).to(dev)) for x in views_h]
        want = D.scene_pointset(views_h, opts, mk)
        got = D.scene_pointset(views_d, opts, mk)
        same(got, want)
        assert len(got["vertices"]) > 0
        if "aabb" in opts:
            assert 0 < len(got["vertices"]) < len(V)
        if "min_valid_fraction" in opts:
            assert any(not v["added"] for v in got["views"])
        if mk:
            assert got["num_filtered"] > 0
