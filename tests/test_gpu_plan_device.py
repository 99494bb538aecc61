"""Planning on the device (-m gpu): a reconstruction whose views have no b200mvs_plan_views plan selects their views and
collects their seeds on the device.  Its maps and counters must be byte-identical to the same reconstruction from plans
made on host threads, b200mvs_plan_info must say which route ran, and the planning allocations must stay within the
budget."""
import numpy as np
import pytest

from tests.test_gpu_reconstruct_pointset import same as _same_pointset
from tests.util import golden_scene

pytestmark = pytest.mark.gpu

KEYS = ("depth", "conf", "dz", "normal", "view_ids")
COUNTERS = ("n_seeds_processed", "n_seeds_success", "n_opt", "n_sample_sets", "n_rounds")
F_SET = dict(with_normals=True, with_conf=True, with_scale=True)


def _settings(s, **kw):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, **kw)


def _same_maps(a, b):
    assert len(a) == len(b)
    for j in range(len(a)):
        for k in KEYS:
            x, y = a[j][k], b[j][k]
            if hasattr(x, "cpu"):
                x, y = x.cpu().numpy(), y.cpu().numpy()
            assert x.tobytes() == y.tobytes(), (j, k)


def _same_counters(a, b, keys=COUNTERS):
    for k in keys:
        assert getattr(a, k) == getattr(b, k), k


def _both_routes(sc, st, refs, run):
    """run() after plans from host threads, then run() planning on the device: both results with their plan_info."""
    sc.plan_views(st, refs)
    host = run()
    ih = sc.plan_info()
    dev = run()
    idev = sc.plan_info()
    assert ih["n_prepared"] == len(refs) and ih["n_device"] == 0 and ih["n_host"] == 0, ih
    return host, dev, idev


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T3", "T4", "T5", "T6"])
def test_golden_scenes(name):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = list(range(s.n_views))
    (mh, sh), (md, sd), info = _both_routes(sc, st, refs, lambda: sc.reconstruct(st, refs))
    assert info["n_device"] == len(refs) and info["n_prepared"] == 0 and info["n_host"] == 0, info
    assert info["ms_device"] > 0 and info["ms_plan"] >= info["ms_device"] * 0.5 and info["peak_bytes"] > 0, info
    _same_maps(mh, md)
    _same_counters(sh, sd)
    # other settings: fewer global views, a larger minimum parallax
    st3 = _settings(s, global_vs_max=3, min_parallax=30.0)
    (mh, sh), (md, sd), info = _both_routes(sc, st3, refs, lambda: sc.reconstruct(st3, refs))
    assert info["n_device"] == len(refs)
    _same_maps(mh, md)
    _same_counters(sh, sd)
    # a minimum parallax above the table's cap plans on host threads
    st45 = _settings(s, min_parallax=45.0)
    (mh, sh), (md, sd), info = _both_routes(sc, st45, refs, lambda: sc.reconstruct(st45, refs))
    assert info["n_host"] == len(refs) and info["n_device"] == 0
    _same_maps(mh, md)
    sc.close()


def test_c2_full_size():
    from mve_b200 import dmrecon, synth
    s = synth.make_scene("C2", device="cuda")
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = list(range(s.n_views))
    (mh, sh), (md, sd), info = _both_routes(sc, st, refs, lambda: sc.reconstruct(st, refs))
    assert info["n_device"] == len(refs)
    _same_maps(mh, md)
    _same_counters(sh, sd)
    sc.close()


def test_reconstruct_device_and_pointset():
    from mve_b200 import dmrecon
    s = golden_scene("T5")
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = list(range(s.n_views))
    (mh, sh), (md, sd), info = _both_routes(sc, st, refs, lambda: sc.reconstruct(st, refs, on_device=True))
    assert info["n_device"] == len(refs)
    _same_maps(mh, md)
    _same_counters(sh, sd)
    (ph, sh), (pd, sd), info = _both_routes(sc, st, refs, lambda: sc.reconstruct_pointset(st, refs, F_SET))
    assert info["n_device"] == len(refs)
    _same_pointset(ph, pd)
    _same_counters(sh, sd)
    sc.close()


def _many_refs(s, times):
    """The scene's features with every ref repeated `times` times (a duplicate ref is a valid input): a planning workspace
    larger than a view's frontier workspace."""
    return [np.repeat(np.sort(np.asarray(r, np.int32)), times) for r in s.feat_refs]


def _lazy(s, budget, many, fetch=None):
    """Scene `s` with the features `many` and a small frontier workspace, its images loaded on demand within `budget`
    (through `fetch` when given)."""
    from mve_b200 import dmrecon
    sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget)
    if fetch is not None:
        sc.set_image_source(fetch, budget)
    sc.set_features(s.feat_pos, many)
    sc.set_frontier_capacity(0.25, 4096)          # maps do not depend on it
    return sc


def test_budget_groups_chunks_and_host_fallback():
    """Under a budget: groups out of ref order, planning chunks of one view, and views whose planning workspace does not
    fit on its own planned on host threads; the maps equal those of the whole batch in one call, and the peak stays
    within the budget."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    refs = list(range(s.n_views))[::-1]
    st = _settings(s)
    many = _many_refs(s, 512)
    whole = dmrecon.Scene.from_synth(s)
    whole.set_features(s.feat_pos, many)
    whole.set_frontier_capacity(0.25, 4096)          # a small frontier workspace; maps do not depend on it
    want, wst = whole.reconstruct(st, refs)
    single_plan = max(0, *[(whole.reconstruct(st, [r]), whole.plan_info()["peak_bytes"])[1] for r in refs])
    all_plan = (whole.reconstruct(st, refs), whole.plan_info()["peak_bytes"])[1]
    assert all_plan > single_plan
    fixed = whole.memory_stats().fixed
    single_ws = max(whole.working_set(st, [r]) for r in refs)
    total_ws = whole.working_set(st, refs)
    whole.close()
    budgets = {"few_groups": fixed + max(single_ws, total_ws // 2, single_plan),
               "one_view_chunks": fixed + max(single_ws, single_plan + 4096)}
    if single_ws < single_plan - (1 << 20):
        budgets["host"] = fixed + single_ws
    for tag, budget in budgets.items():
        sc = _lazy(s, budget, many)
        got, gst = sc.reconstruct(st, refs)
        info = sc.plan_info()
        mem = sc.memory_stats()
        assert mem.peak <= budget, (tag, mem.peak, budget)
        if tag == "host":
            assert info["n_host"] == len(refs) and info["n_device"] == 0, (tag, info)
        else:
            assert info["n_device"] == len(refs) and info["peak_bytes"] <= budget, (tag, info)
        if tag == "one_view_chunks":
            assert info["peak_bytes"] <= budget - fixed and info["peak_bytes"] < all_plan, (tag, info)
        _same_maps(want, got)
        _same_counters(wst, gst, [k for k in COUNTERS if k != "n_rounds"])   # rounds add up over groups
        sc.close()
    assert "host" in budgets, (single_ws, single_plan)


@pytest.mark.parametrize("before", ["level", "optimize_patches", "failed_reconstruction"])
def test_pins_last_one_call(before):
    """The views a call pins are unpinned when it returns, also after a level read, a patch optimisation and a failed
    reconstruction.  The budget fits the planning workspace of the next reconstruction only when a resident pyramid is
    evicted, so it plans as on a context that skipped the earlier call: every view on the device, with the same maps."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    refs = list(range(s.n_views))[::-1]
    st = _settings(s)
    many = _many_refs(s, 512)
    whole = dmrecon.Scene.from_synth(s)
    whole.set_features(s.feat_pos, many)
    whole.set_frontier_capacity(0.25, 4096)
    single_plan = max(0, *[(whole.reconstruct(st, [r]), whole.plan_info()["peak_bytes"])[1] for r in refs])
    fixed = whole.memory_stats().fixed
    single_ws = max(whole.working_set(st, [r]) for r in refs)
    whole.close()
    assert single_ws < single_plan, (single_ws, single_plan)
    budget = fixed + single_plan + 4096

    def routes(sc):
        maps, stats = sc.reconstruct(st, refs)
        info = sc.plan_info()
        return maps, stats, (info["n_prepared"], info["n_device"], info["n_host"])

    sc = _lazy(s, budget, many)
    want, wst, want_routes = routes(sc)
    sc.close()
    assert want_routes == (0, len(refs), 0), want_routes
    failing = {"view": -1}

    def fetch(view):
        if view == failing["view"]:
            raise RuntimeError("view %d is not available" % view)
        return s.images[view]

    sc = _lazy(s, budget, many, fetch)
    v = 0
    if before == "level":
        sc.level(v, 0)
    elif before == "optimize_patches":
        m = want[refs.index(v)]
        y, x = np.nonzero(m["conf"] > 0)
        y, x = y[:64], x[:64]
        pin = np.zeros(len(y), dmrecon.PATCH_IN)
        pin["x"], pin["y"], pin["depth"] = x, y, m["depth"][y, x]
        pin["dz_i"], pin["dz_j"] = m["dz"][y, x, 0], m["dz"][y, x, 1]
        pin["n_local"] = 4
        pin["local_ids"] = m["view_ids"][y, x]
        assert (sc.optimize_patches(st, v, sc.global_view_selection(st, v), pin)["conf"] > 0).any()
    else:
        failing["view"] = refs[0]                   # the first group's reference view, loaded after its neighbours
        with pytest.raises(dmrecon.B200MVSError):
            sc.reconstruct(st, refs)
        failing["view"] = -1
    got, gst, got_routes = routes(sc)
    assert got_routes == want_routes, got_routes
    _same_maps(want, got)
    _same_counters(wst, gst, [k for k in COUNTERS if k != "n_rounds"])   # rounds add up over groups
    assert sc.memory_stats().peak <= budget
    sc.close()


def test_empty_selection_fails_the_same_way():
    """A view that no feature references has an empty selection: both routes fail with B200MVS_ERR_GLOBAL_VS naming it."""
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s)
    sc.set_features(s.feat_pos, [np.asarray([v for v in r if v != 2], np.int32) for r in s.feat_refs])
    st = _settings(s)
    errs = []
    for prepared in (True, False):
        if prepared:
            sc.plan_views(st, [0, 2, 1])
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.reconstruct(st, [0, 2, 1])
        errs.append((e.value.code, e.value.failed_view, str(e.value)))
    assert errs[0] == errs[1] and errs[0][0] == -3 and errs[0][1] == 2, errs
    assert sc.plan_info()["n_device"] == 3
    sc.close()
