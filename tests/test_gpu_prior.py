"""Prior depth maps (b200mvs_set_view_prior[_device], Scene.set_view_prior): a prior that seeds nothing changes no byte
and no counter; the seeds it adds are those of tests/prior_reference.py; an isolated prior seed holds exactly what
b200mvs_optimize_patches gives for it; host and device priors, levels, budgets, resumes and the point set agree; the seed
limit is checked before any image is fetched; a prior from the analytic depth grows maps at least as full and as accurate
in fewer rounds; and the drop-in CLI runs coarse to fine."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests.prior_reference import prior_cells, prior_seeds
from tests.test_gpu_mask_device import _cuda
from tests.test_gpu_recon_mask import CLI, COUNTERS, KEYS, MODES, _map_size, _settings, _silhouettes
from tests.util import golden_scene

pytestmark = pytest.mark.gpu


def _dev(d, pitched=False):
    """The prior as a float32 CUDA tensor; pitched: a column slice of a wider tensor (row stride > width)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda()
    if not pitched:
        return t
    h, w = t.shape
    wide = torch.full((h, w + 9), -7.0, dtype=torch.float32, device=t.device)
    wide[:, 3:3 + w] = t
    return wide[:, 3:3 + w]


def _set_priors(sc, refs, priors, stride, on_device=False, pitched=False):
    for v in refs:
        d = None if priors is None else priors.get(v)
        if d is None or not on_device:
            sc.set_view_prior(v, d, stride)
        else:
            sc.set_view_prior(v, _dev(d, pitched), stride, on_device=True)


def _run(sc, st, refs, route="host", mode="default", **kw):
    import torch
    sc.set_patch_mode(0, MODES[mode])
    if route == "pset":
        from tests.test_gpu_reconstruct_pointset import F_SET
        ps, stats = sc.reconstruct_pointset(st, refs, F_SET)
        return ps, {k: getattr(stats, k) for k in COUNTERS}
    if route == "device":
        maps, stats = sc.reconstruct(st, refs, on_device=True, **kw)
        torch.cuda.synchronize()
        maps = [{k: v.cpu().numpy() for k, v in m.items()} for m in maps]
    else:
        maps, stats = sc.reconstruct(st, refs, **kw)
    return maps, {k: getattr(stats, k) for k in COUNTERS}


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for k in KEYS:
            assert x[k].tobytes() == y[k].tobytes(), k


def _same_route(a, b, route):
    if route == "pset":
        from tests.test_gpu_reconstruct_pointset import same
        same(a, b)
    else:
        _same(a, b)


def _depth_priors(s, refs, size="photo"):
    from mve_b200 import synth
    out = {}
    for v in refs:
        w, h = s.size(v) if size == "photo" else _map_size(s, v) if size == "map" else size
        out[v] = synth.depth(s, v, w, h)
    return out


@pytest.mark.parametrize("mode", ["warp", "thread"])
@pytest.mark.parametrize("route", ["host", "device", "pset"])
def test_no_op_priors(route, mode):
    """A prior set and cleared again, or one of only 0, negative, NaN and +-inf values, changes no byte and no counter."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    want, wc = _run(sc, st, refs, route, mode)
    _set_priors(sc, refs, _depth_priors(s, refs), 2)
    _set_priors(sc, refs, None, 2)
    got, c = _run(sc, st, refs, route, mode)
    _same_route(got, want, route)
    assert c == wc
    rng = np.random.default_rng(7)
    vals = np.array([0.0, -1.0, -0.0, np.nan, np.inf, -np.inf], np.float32)
    junk = {v: rng.choice(vals, (s.size(v)[1], s.size(v)[0])).astype(np.float32) for v in refs}
    for on_device in (False, True):
        _set_priors(sc, refs, junk, 1, on_device)
        got, c = _run(sc, st, refs, route, mode)
        _same_route(got, want, route)
        assert c == wc, on_device
    sc.close()


def _expected_seeds(s, refs, priors, stride, masks, level_of=None):
    n = 0
    for v in refs:
        W, H = _map_size(s, v) if level_of is None else level_of[v]
        n += len(prior_seeds(W, H, priors[v], stride, None if masks is None else masks.get(v)))
    return n


@pytest.mark.parametrize("name", ["T0", "T5", "T6"])
@pytest.mark.parametrize("size", ["photo", "map", (37, 29), (400, 300)])
@pytest.mark.parametrize("stride", [1, 3, 8])
def test_seed_count(name, size, stride):
    """n_seeds_processed with the prior minus without it is the reference count, without a mask and with host and
    device silhouette masks."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    priors = _depth_priors(s, refs, size)
    rng = np.random.default_rng(stride)
    for d in priors.values():                       # some invalid values among the valid ones
        d[rng.random(d.shape) < 0.2] = np.nan
    masks = _silhouettes(s, refs)
    for mask_kind in (None, "host", "device"):
        for v in refs:
            if mask_kind is None:
                sc.set_view_mask(v, None)
            else:
                sc.set_view_mask(v, masks[v] if mask_kind == "host" else _cuda(masks[v]), on_device=mask_kind == "device")
        _set_priors(sc, refs, None, stride)
        _, without = _run(sc, st, refs)
        _set_priors(sc, refs, priors, stride)
        _, with_ = _run(sc, st, refs)
        want = _expected_seeds(s, refs, priors, stride, None if mask_kind is None else masks)
        assert with_["n_seeds_processed"] - without["n_seeds_processed"] == want, mask_kind
        assert with_["n_seeds_success"] >= without["n_seeds_success"] or want == 0
    sc.close()


def test_seed_round_exactness():
    """A mask whose foreground is exactly the candidate grid keeps every seed where it is.  Each seeded pixel the run
    without the prior left unfilled holds what b200mvs_optimize_patches (one warp per patch) gives: first r1 for
    (x, y, prior depth, no local views) with the view's global selection, as the seed round does.  A committed seed is
    queued again at its own pixel with r1's depth, dz and local views (processFeatures pushes it, dmrecon.cc:325), so
    the next round optimises it once more, to r2, and commits r2 when r2.conf != 0 and r1.conf < r2.conf (dmrecon.cc:
    377-398).  The map therefore holds r2 or r1, never r1 alone by rule; a pixel with r1.conf <= 0 stays unfilled."""
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    st = _settings(s)
    refs = list(range(s.n_views))
    stride = 3
    sc = dmrecon.Scene.from_synth(s)
    priors = _depth_priors(s, refs, "map")
    grid = {}
    for v in refs:
        W, H = _map_size(s, v)
        m = np.zeros((H, W), np.uint8)
        m[2:H - 2:stride, 2:W - 2:stride] = 255
        m[:, prior_cells(W, stride) * stride + 2:] = 0
        m[prior_cells(H, stride) * stride + 2:, :] = 0
        grid[v] = m
        sc.set_view_mask(v, m)
    plain, _ = _run(sc, st, refs, mode="warp")
    _set_priors(sc, refs, priors, stride)
    seeded, _ = _run(sc, st, refs, mode="warp")
    sc.set_patch_mode(1)
    n_checked = n_failed = n_second = 0
    for j, v in enumerate(refs):
        W, H = _map_size(s, v)
        seeds = [q for q in prior_seeds(W, H, priors[v], stride, grid[v]) if plain[j]["conf"][q[1], q[0]] == 0]
        assert seeds
        patches = np.zeros(len(seeds), dmrecon.PATCH_IN)
        patches["x"] = [q[0] for q in seeds]
        patches["y"] = [q[1] for q in seeds]
        patches["depth"] = [q[2] for q in seeds]
        patches["local_ids"] = -1
        gsel = sc.global_view_selection(st, v)
        r1 = sc.optimize_patches(st, v, gsel, patches)
        again = patches.copy()
        for k in ("depth", "dz_i", "dz_j", "n_local", "local_ids"):
            again[k] = r1[k]
        r2 = sc.optimize_patches(st, v, gsel, again)
        m = seeded[j]
        for q, a, b in zip(seeds, r1, r2):
            x, y = q[0], q[1]
            if not a["conf"] > 0:
                assert m["conf"][y, x] == 0, (v, x, y)
                n_failed += 1
                continue
            second = b["conf"] != 0 and a["conf"] < b["conf"]
            n_second += int(second)
            o = b if second else a
            assert m["conf"][y, x] == o["conf"] and m["depth"][y, x] == o["depth"], (v, x, y)
            assert (m["dz"][y, x] == np.array([o["dz_i"], o["dz_j"]], np.float32)).all(), (v, x, y)
            assert m["normal"][y, x].tobytes() == o["normal"].tobytes(), (v, x, y)
            assert list(m["view_ids"][y, x]) == list(o["local_ids"]), (v, x, y)
            n_checked += 1
    assert n_checked > 50 and n_second > 0
    sc.close()


@pytest.mark.parametrize("pitched", [False, True])
def test_host_and_device_priors_agree(pitched):
    """The device form gives the host form's maps, counters and memory_stats; the source is written on a side stream
    right before the call and overwritten right after it returns."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    priors = _depth_priors(s, refs, (57, 41))
    results = []
    for on_device in (False, True):
        sc = dmrecon.Scene.from_synth(s)
        if on_device:
            side = torch.cuda.Stream()
            for v in refs:
                with torch.cuda.stream(side):
                    torch.cuda._sleep(2_000_000)
                    t = _dev(np.zeros_like(priors[v]), pitched)
                    t.copy_(torch.from_numpy(priors[v]).cuda(non_blocking=True))
                    sc.set_view_prior(v, t, 4, on_device=True)
                    t.fill_(5.0)
            torch.cuda.synchronize()
        else:
            _set_priors(sc, refs, priors, 4)
        m = sc.memory_stats()
        maps, c = _run(sc, st, refs, "device" if on_device else "host")
        results.append((maps, c, (m.fixed, m.resident)))
        sc.close()
    _same(results[0][0], results[1][0])
    assert results[0][1:] == results[1][1:]


def test_levels_equal_single_level_calls():
    """One view at two levels in one call: each entry equals the single-level call with the same prior."""
    from mve_b200 import dmrecon
    s = golden_scene("T6")
    refs = [0, 0, 1]
    levels = [1, 2, 0]                              # view 0: 179 x 180, view 1: 118 x 58
    sc = dmrecon.Scene.from_synth(s)
    priors = _depth_priors(s, [0, 1], "photo")
    _set_priors(sc, [0, 1], priors, 2)
    got, _ = _run(sc, dmrecon.Settings(scale=-3, nr_recon_neighbors=s.nr_recon_neighbors), refs, scales=levels)
    for j, (v, lv) in enumerate(zip(refs, levels)):
        one, _ = _run(sc, dmrecon.Settings(scale=lv, nr_recon_neighbors=s.nr_recon_neighbors), [v])
        _same([got[j]], one)
    sc.close()


def test_budget_groups_resumes_and_memory():
    """A lazy source whose budget splits the batch into groups out of order, then a frontier small enough to resume: the
    maps of the unbudgeted call, peak <= budget; fixed and working sets grow by exactly the prior's bytes and bounds; a
    prior that does not fit gives NO_MEMORY and keeps the old one."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    priors = _depth_priors(s, refs)
    stride = 4
    plain = dmrecon.Scene.from_synth(s)
    _set_priors(plain, refs, priors, stride)
    want, wc = _run(plain, st, refs)
    plain.close()

    lazy = dmrecon.Scene.from_synth(s, lazy=True)
    f0 = lazy.memory_stats().fixed
    ws0 = {v: lazy.working_set(st, [v]) for v in refs}
    lazy.set_view_prior(refs[0], priors[refs[0]], stride)
    assert lazy.memory_stats().fixed == f0 + priors[refs[0]].nbytes
    lazy.set_view_prior(refs[0], None, stride)
    assert lazy.memory_stats().fixed == f0
    _set_priors(lazy, refs, priors, stride)
    fixed = lazy.memory_stats().fixed
    assert fixed == f0 + sum(4 * d.size for d in priors.values())
    # with a capacity of max(seeds, 1) entries the frontier arrays (169 bytes per entry) grow by the candidate bound
    lazy.set_frontier_capacity(0.0, 1)
    for v in refs:
        lazy.set_view_prior(v, None, stride)
    base = {v: lazy.working_set(st, [v]) for v in refs}
    _set_priors(lazy, refs, priors, stride)
    for v in refs:
        W, H = _map_size(s, v)
        assert lazy.working_set(st, [v]) - base[v] == 169 * prior_cells(W, stride) * prior_cells(H, stride), v
    lazy.set_frontier_capacity()
    assert all(lazy.working_set(st, [v]) == ws0[v] for v in refs)    # 2 x pixels still bounds the capacity
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
    got, c = _run(lazy, st, refs)
    mem = lazy.memory_stats()
    assert mem.n_groups == chosen[1] and mem.fixed == fixed and mem.peak <= mem.budget
    _same(got, want)
    for k in ("n_filled", "n_seeds_processed", "n_seeds_success"):
        assert c[k] == wc[k], k
    # a frontier small enough to resume, under a budget that holds the batch's working set at the default capacity
    lazy.set_image_source(lambda v: s.images[v], fixed + total)
    lazy.set_frontier_capacity(0.01, 1)
    again, c = _run(lazy, st, refs)
    assert lazy.frontier_info()["resumes"] >= 1 and lazy.memory_stats().peak <= lazy.memory_stats().budget
    _same(again, want)
    assert c["n_seeds_processed"] == wc["n_seeds_processed"]
    lazy.set_frontier_capacity()

    # a prior beyond the budget: NO_MEMORY, and the previous prior stays
    lazy.set_image_source(lambda v: s.images[v], fixed + 4096)
    for huge in (np.ones((1024, 1024), np.float32), torch.ones((1024, 1024), device="cuda")):
        with pytest.raises(dmrecon.B200MVSError) as e:
            lazy.set_view_prior(refs[0], huge, stride, on_device=not isinstance(huge, np.ndarray))
        assert e.value.code == dmrecon.ERR_NO_MEMORY and "b200mvs_set_view_prior" in str(e.value)
        assert lazy.memory_stats().fixed == fixed
    lazy.set_image_source(lambda v: s.images[v], 0)
    got, c = _run(lazy, st, refs)
    _same(got, want)
    lazy.close()


def test_pointset_equals_reconstruct_and_scene_pointset():
    from mve_b200 import dmrecon
    from tests.test_gpu_reconstruct_pointset import F_SET, host_route, same
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    sc = dmrecon.Scene.from_synth(s)
    _set_priors(sc, refs, _depth_priors(s, refs, "map"), 3)
    got, gs = sc.reconstruct_pointset(st, refs, F_SET)
    want, _ = host_route(sc, s, st, refs, F_SET)
    same(got, want)
    _, ms = sc.reconstruct(st, refs)
    assert {k: getattr(gs, k) for k in COUNTERS} == {k: getattr(ms, k) for k in COUNTERS}
    sc.close()


def test_seed_limit_before_any_fetch():
    """A 1 x 1 prior at stride 1 on a view registered at 50000 x 50000 (a candidate bound of 49996^2 > 2^31 - 1 at level
    0): INVALID_ARG naming the view, before any image is fetched."""
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    st = dmrecon.Settings(scale=0, nr_recon_neighbors=s.nr_recon_neighbors)
    sc.set_view_camera(0, 50000, 50000, s.flen[0], s.paspect[0], s.ppoint[0], s.rot[0], s.trans[0])
    sc.set_view_prior(0, np.ones((1, 1), np.float32), 1)
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, [0])
    assert e.value.code == dmrecon.ERR_INVALID_ARG and e.value.failed_view == 0
    assert "prior candidates" in str(e.value)
    assert sc.memory_stats().n_loads == 0
    sc.close()


def _fill_and_error(s, maps, refs):
    from mve_b200 import synth
    fill, err = [], []
    for j, v in enumerate(refs):
        W, H = _map_size(s, v)
        truth = synth.depth(s, v, W, H)
        d = maps[j]["depth"]
        ok = (d > 0) & (truth > 0)
        fill.append((d > 0).mean())
        err.append(np.abs(d[ok] - truth[ok]) / truth[ok])
    e = np.concatenate(err)
    return float(np.mean(fill)), float(np.median(e)), float(np.percentile(e, 95))


@pytest.mark.parametrize("name", ["T1", "T2"])
def test_quality(name):
    """synth.depth as the prior at stride 4: fill not below the plain run, median and p95 relative depth error within
    5 % of its own, fewer rounds."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    plain, pc = _run(sc, st, refs)
    _set_priors(sc, refs, _depth_priors(s, refs, "map"), 4)
    seeded, sc_ = _run(sc, st, refs)
    f0, m0, p0 = _fill_and_error(s, plain, refs)
    f1, m1, p1 = _fill_and_error(s, seeded, refs)
    print("%s plain: fill %.4f median %.3e p95 %.3e rounds %d | prior: fill %.4f median %.3e p95 %.3e rounds %d"
          % (name, f0, m0, p0, pc["n_rounds"], f1, m1, p1, sc_["n_rounds"]))
    assert f1 >= f0
    assert m1 <= 1.05 * m0 and p1 <= 1.05 * p0
    assert sc_["n_rounds"] < pc["n_rounds"]
    sc.close()


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_coarse_to_fine():
    """-s<L+1>, then B200MVS_PRIOR=depth-L<L+1>,4 -s<L>: the level-L depth and conf of the Python route with those maps as
    priors; a view without the embedding runs without a prior and says so."""
    from mve_b200 import dmrecon, synth
    s = golden_scene("T1")
    views = [0, 4, 7]
    lo, hi = 0, 1
    base = ["--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--progress=silent", "--force"]
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        out = subprocess.run([CLI, "-s%d" % hi] + base + ["-l" + ",".join(str(v) for v in views), tmp],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        coarse = {v: synth.read_mvei(os.path.join(tmp, "views", "view_%04d.mve" % v, "depth-L%d.mvei" % hi))[:, :, 0]
                  for v in views}
        os.remove(os.path.join(tmp, "views", "view_0007.mve", "depth-L%d.mvei" % hi))
        out = subprocess.run([CLI, "-s%d" % lo] + base + ["-l" + ",".join(str(v) for v in views), tmp],
                             capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200MVS_PRIOR="depth-L%d,4" % hi))
        assert out.returncode == 0, out.stdout + out.stderr
        assert 'Prior not found for image "0007", skipping.' in out.stdout, out.stdout
        sc = dmrecon.Scene.from_synth(s)
        st = dmrecon.Settings(scale=lo, nr_recon_neighbors=s.nr_recon_neighbors)
        for v in views:
            sc.set_view_prior(v, coarse[v] if v != 7 else None, 4)
            want, _ = sc.reconstruct(st, [v])
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            depth = synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % lo))[:, :, 0]
            conf = synth.read_mvei(os.path.join(vd, "conf-L%d.mvei" % lo))[:, :, 0]
            assert depth.tobytes() == want[0]["depth"].tobytes(), v
            assert conf.tobytes() == want[0]["conf"].tobytes(), v
        sc.close()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        out = subprocess.run([CLI, "-s%d" % lo] + base + ["-l0", tmp], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200MVS_PRIOR="depth-L1"))
        assert "B200MVS_PRIOR: expected <embedding>,<stride>" in out.stderr, out.stderr
