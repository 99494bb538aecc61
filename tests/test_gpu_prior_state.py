"""Priors with state (b200mvs_set_view_prior_state[_device], Scene.set_view_prior(dz=, view_ids=)): a prior without dz
and ids, or with a dz of zeros and ids of -1, gives the depth-only prior's bytes and counters; an isolated prior seed
holds exactly what b200mvs_optimize_patches gives for the depth, scaled dz and local views of tests/prior_state_reference
.py; host and device forms, levels, budgets and resumes agree; the blocks are counted in memory_stats; state priors keep
the depth-only prior's quality; and the drop-in CLI carries a dz embedding."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests.prior_reference import prior_cells
from tests.prior_state_reference import prior_state_seeds
from tests.test_gpu_prior import _run, _same, _same_route
from tests.test_gpu_recon_mask import CLI, _map_size, _settings
from tests.util import golden_scene

pytestmark = pytest.mark.gpu


def _earlier(sc, s, refs, level):
    """The maps of an earlier reconstruction of the scene at `level`, on the host."""
    from mve_b200 import dmrecon
    maps, _ = sc.reconstruct(dmrecon.Settings(scale=level, nr_recon_neighbors=s.nr_recon_neighbors), refs)
    return {v: maps[j] for j, v in enumerate(refs)}


def _cuda(a, pitched=False):
    """A CUDA tensor of `a` (H x W or H x W x C); pitched: a column slice of a wider tensor (row stride > width)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if not pitched:
        return t
    wide = torch.full((t.shape[0], t.shape[1] + 9) + tuple(t.shape[2:]), -7, dtype=t.dtype, device=t.device)
    wide[:, 3:3 + t.shape[1]] = t
    return wide[:, 3:3 + t.shape[1]]


def _set_state(sc, refs, prior, stride, planes=("dz", "view_ids"), on_device=False, pitched=False):
    for v in refs:
        m = prior[v]
        kw = {k: (_cuda(m[k], pitched) if on_device else m[k]) for k in planes}
        sc.set_view_prior(v, _cuda(m["depth"], pitched) if on_device else m["depth"], stride, on_device=on_device, **kw)


@pytest.mark.parametrize("mode", ["warp", "thread"])
@pytest.mark.parametrize("route", ["host", "device", "pset"])
def test_no_op_state(route, mode):
    """set_view_prior(d) == set_view_prior_state(d, NULL, NULL) in maps, counters and memory_stats; a dz of zeros and
    ids of -1 give the same maps and counters, and memory_stats larger by exactly their blocks."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    prior = _earlier(sc, s, refs, s.scale + 1)
    L = dmrecon.lib()
    for v in refs:
        sc.set_view_prior(v, prior[v]["depth"], 3)
    want, wc = _run(sc, st, refs, route, mode)
    m0 = sc.memory_stats()
    for v in refs:
        d = np.ascontiguousarray(prior[v]["depth"])
        h, w = d.shape
        assert L.b200mvs_set_view_prior_state(sc._h, v, d.ctypes.data, None, None, w, h, 3) == 0
    got, c = _run(sc, st, refs, route, mode)
    m1 = sc.memory_stats()
    _same_route(got, want, route)
    assert c == wc and (m1.fixed, m1.resident, m1.budget) == (m0.fixed, m0.resident, m0.budget)
    blank = {v: dict(depth=prior[v]["depth"], dz=np.zeros_like(prior[v]["dz"]),
                     view_ids=np.full_like(prior[v]["view_ids"], -1)) for v in refs}
    extra = sum(24 * prior[v]["depth"].size for v in refs)
    for on_device in (False, True):
        _set_state(sc, refs, blank, 3, on_device=on_device)
        got, c = _run(sc, st, refs, route, mode)
        _same_route(got, want, route)
        assert c == wc, on_device
        assert sc.memory_stats().fixed == m0.fixed + extra
    sc.close()


def _grid_masks(s, refs, stride):
    grid = {}
    for v in refs:
        W, H = _map_size(s, v)
        m = np.zeros((H, W), np.uint8)
        m[2:H - 2:stride, 2:W - 2:stride] = 255
        m[:, prior_cells(W, stride) * stride + 2:] = 0
        m[prior_cells(H, stride) * stride + 2:, :] = 0
        grid[v] = m
    return grid


def _edit_ids(prior, gsel, N, rng):
    """Rewrites the prior's id maps so that the candidates meet every branch of the id rule, in a random order of the
    four ids: exactly N valid ids; N with a duplicate; N with an id outside the global selection; N - 1; more than N
    (N < 4); none (all -1)."""
    for v, m in prior.items():
        g = np.asarray(gsel[v])
        outside = np.setdiff1d(np.arange(64), g)
        h, w = m["depth"].shape
        ids = np.full((h, w, 4), -1, np.int32)
        for y in range(h):
            for x in range(w):
                kind = (x + 3 * y) % 6
                n_valid = {0: N, 1: N, 2: N, 3: N - 1, 4: N + 1, 5: 0}[kind]
                pick = [int(i) for i in rng.choice(g, min(n_valid, len(g), 4), replace=False)]
                if kind == 1 and pick:
                    pick.append(pick[0])
                if kind == 2:
                    pick.append(int(outside[(x + y) % len(outside)]))
                ids[y, x] = rng.permutation((pick + [-1] * 4)[:4])
        m["view_ids"] = ids


@pytest.mark.parametrize("source", ["same", "coarser", "edited"])
def test_seed_round_exactness(source):
    """A mask whose foreground is exactly the candidate grid keeps every seed where it is.  Each seeded pixel the run
    without the prior left unfilled holds what b200mvs_optimize_patches (one warp per patch) gives: r1 for (x, y,
    depth, scaled dz, the rule's local ids or none) with the view's global selection, then r2 for r1's state, committed
    when r2.conf != 0 and r1.conf < r2.conf (tests/test_gpu_prior.py::test_seed_round_exactness).  The priors are the
    maps of an earlier reconstruction at the same level (dz ratio 1) or the next coarser one (dz scaled), or those of
    the same level with id maps edited to meet every branch of the id rule."""
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    st = _settings(s)
    refs = list(range(s.n_views))
    stride = 3
    N = s.nr_recon_neighbors
    sc = dmrecon.Scene.from_synth(s)
    prior = _earlier(sc, s, refs, s.scale + (1 if source == "coarser" else 0))
    gsel = {v: sc.global_view_selection(st, v) for v in refs}
    if source == "edited":
        _edit_ids(prior, gsel, N, np.random.default_rng(4))
    grid = _grid_masks(s, refs, stride)
    for v in refs:
        sc.set_view_mask(v, grid[v])
    plain, _ = _run(sc, st, refs, mode="warp")
    _set_state(sc, refs, prior, stride)
    seeded, _ = _run(sc, st, refs, mode="warp")
    sc.set_patch_mode(1)
    n_checked = n_local = n_none = n_scaled = 0
    for j, v in enumerate(refs):
        W, H = _map_size(s, v)
        seeds = [q for q in prior_state_seeds(W, H, prior[v]["depth"], stride, gsel[v], N, prior[v]["dz"],
                                              prior[v]["view_ids"], grid[v]) if plain[j]["conf"][q[1], q[0]] == 0]
        assert seeds
        patches = np.zeros(len(seeds), dmrecon.PATCH_IN)
        patches["x"] = [q[0] for q in seeds]
        patches["y"] = [q[1] for q in seeds]
        patches["depth"] = [q[2] for q in seeds]
        patches["dz_i"] = [q[3] for q in seeds]
        patches["dz_j"] = [q[4] for q in seeds]
        patches["n_local"] = [0 if q[5] is None else N for q in seeds]
        patches["local_ids"] = [([-1] * 4 if q[5] is None else (q[5] + [-1] * 4)[:4]) for q in seeds]
        n_local += sum(q[5] is not None for q in seeds)
        n_none += sum(q[5] is None for q in seeds)
        h = prior[v]["depth"].shape[0]
        n_scaled += int(h != H) * len(seeds)
        r1 = sc.optimize_patches(st, v, gsel[v], patches)
        again = patches.copy()
        for k in ("depth", "dz_i", "dz_j", "n_local", "local_ids"):
            again[k] = r1[k]
        r2 = sc.optimize_patches(st, v, gsel[v], again)
        m = seeded[j]
        for q, a, b in zip(seeds, r1, r2):
            x, y = q[0], q[1]
            if not a["conf"] > 0:
                assert m["conf"][y, x] == 0, (v, x, y)
                continue
            o = b if (b["conf"] != 0 and a["conf"] < b["conf"]) else a
            assert m["conf"][y, x] == o["conf"] and m["depth"][y, x] == o["depth"], (v, x, y)
            assert (m["dz"][y, x] == np.array([o["dz_i"], o["dz_j"]], np.float32)).all(), (v, x, y)
            assert m["normal"][y, x].tobytes() == o["normal"].tobytes(), (v, x, y)
            assert list(m["view_ids"][y, x]) == list(o["local_ids"]), (v, x, y)
            n_checked += 1
    print("%s: %d checked, %d seeds with local views, %d without" % (source, n_checked, n_local, n_none))
    assert n_checked > 50 and n_local > 0
    if source == "coarser":
        assert n_scaled > 0
    if source == "edited":
        assert n_none > 0
    sc.close()


@pytest.mark.parametrize("pitched", [False, True])
def test_host_and_device_forms_agree(pitched):
    """The device form gives the host form's maps, counters and memory_stats; each plane is written on a side stream
    right before the call and overwritten right after it returns."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    src = dmrecon.Scene.from_synth(s)                 # its own scene: both below start with nothing resident
    prior = _earlier(src, s, refs, s.scale + 1)
    src.close()
    results = []
    for on_device in (False, True):
        sc = dmrecon.Scene.from_synth(s)
        if on_device:
            side = torch.cuda.Stream()
            for v in refs:
                with torch.cuda.stream(side):
                    torch.cuda._sleep(2_000_000)
                    t = {k: _cuda(np.zeros_like(prior[v][k]), pitched) for k in ("depth", "dz", "view_ids")}
                    for k in t:
                        t[k].copy_(torch.from_numpy(prior[v][k]).cuda(non_blocking=True))
                    sc.set_view_prior(v, t["depth"], 4, on_device=True, dz=t["dz"], view_ids=t["view_ids"])
                    for k in t:
                        t[k].fill_(5)
            torch.cuda.synchronize()
        else:
            _set_state(sc, refs, prior, 4)
        m = sc.memory_stats()
        maps, c = _run(sc, st, refs, "device" if on_device else "host")
        results.append((maps, c, (m.fixed, m.resident)))
        sc.close()
    _same(results[0][0], results[1][0])
    assert results[0][1:] == results[1][1:]


def test_levels_equal_single_level_calls():
    """One view at two levels in one call, each with its own W x H and global selection: each entry equals the
    single-level call with the same state prior."""
    from mve_b200 import dmrecon
    s = golden_scene("T6")
    refs = [0, 0, 1]
    levels = [1, 2, 0]
    sc = dmrecon.Scene.from_synth(s)
    prior = _earlier(sc, s, [0, 1], 1)
    _set_state(sc, [0, 1], prior, 2)
    got, _ = _run(sc, dmrecon.Settings(scale=-3, nr_recon_neighbors=s.nr_recon_neighbors), refs, scales=levels)
    for j, (v, lv) in enumerate(zip(refs, levels)):
        one, _ = _run(sc, dmrecon.Settings(scale=lv, nr_recon_neighbors=s.nr_recon_neighbors), [v])
        _same([got[j]], one)
    sc.close()


def test_budget_groups_resumes_and_memory():
    """memory_stats.fixed grows by exactly 4 + 8 + 16 B per prior pixel for the planes given and returns on clear; a
    budget that splits the batch into groups, and a frontier small enough to resume, give the unbudgeted maps; a prior
    that does not fit gives NO_MEMORY and leaves the old one whole."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    stride = 4
    plain = dmrecon.Scene.from_synth(s)
    prior = _earlier(plain, s, refs, s.scale + 1)
    _set_state(plain, refs, prior, stride)
    want, wc = _run(plain, st, refs)
    plain.close()

    lazy = dmrecon.Scene.from_synth(s, lazy=True)
    f0 = lazy.memory_stats().fixed
    v0 = refs[0]
    npx = prior[v0]["depth"].size
    for planes, per_px in (((), 4), (("dz",), 12), (("view_ids",), 20), (("dz", "view_ids"), 28)):
        for on_device in (False, True):
            _set_state(lazy, [v0], prior, stride, planes, on_device)
            assert lazy.memory_stats().fixed == f0 + per_px * npx, (planes, on_device)
    lazy.set_view_prior(v0, None, stride)
    assert lazy.memory_stats().fixed == f0
    _set_state(lazy, refs, prior, stride)
    fixed = lazy.memory_stats().fixed
    assert fixed == f0 + sum(28 * prior[v]["depth"].size for v in refs)
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
    lazy.set_image_source(lambda v: s.images[v], fixed + total)
    lazy.set_frontier_capacity(0.01, 1)
    again, c = _run(lazy, st, refs)
    assert lazy.frontier_info()["resumes"] >= 1
    _same(again, want)
    lazy.set_frontier_capacity()

    # a prior beyond the budget: NO_MEMORY, and the previous prior (all three planes) stays
    lazy.set_image_source(lambda v: s.images[v], fixed + 4096)
    big = (1024, 1024)
    for on_device in (False, True):
        d, z, i = np.ones(big, np.float32), np.zeros(big + (2,), np.float32), np.full(big + (4,), -1, np.int32)
        if on_device:
            d, z, i = torch.from_numpy(d).cuda(), torch.from_numpy(z).cuda(), torch.from_numpy(i).cuda()
        with pytest.raises(dmrecon.B200MVSError) as e:
            lazy.set_view_prior(v0, d, stride, on_device=on_device, dz=z, view_ids=i)
        assert e.value.code == dmrecon.ERR_NO_MEMORY and "b200mvs_set_view_prior_state" in str(e.value)
        assert lazy.memory_stats().fixed == fixed
    lazy.set_image_source(lambda v: s.images[v], 0)
    got, c = _run(lazy, st, refs)
    _same(got, want)
    lazy.close()


def test_device_checks_name_the_field():
    """The device form's pitch and buffer checks, before anything is copied: the message names the function and field."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s)
    L = dmrecon.lib()
    fn = "b200mvs_set_view_prior_state_device"
    w, h = 6, 5
    d = torch.ones((h, w), device="cuda")
    z = torch.zeros((h, w, 2), device="cuda")
    i = torch.full((h, w, 4), -1, dtype=torch.int32, device="cuda")
    host = np.zeros((h, w, 4), np.int32)
    P = lambda t: C.c_void_p(t.data_ptr())                      # noqa: E731
    cases = [
        ((P(d), P(z), P(i), 4 * w - 4, 8 * w, 16 * w), "depth_pitch is %d, not a multiple of 4 of at least 4 w (%d)" % (4 * w - 4, 4 * w)),
        ((P(d), P(z), P(i), 4 * w, 8 * w - 4, 16 * w), "dz_pitch is %d, not a multiple of 4 of at least 8 w (%d)" % (8 * w - 4, 8 * w)),
        ((P(d), P(z), P(i), 4 * w, 8 * w, 16 * w + 2), "ids_pitch is %d, not a multiple of 4 of at least 16 w (%d)" % (16 * w + 2, 16 * w)),
        ((P(d), P(z), C.c_void_p(host.ctypes.data), 4 * w, 8 * w, 16 * w), "view_ids_dev"),
        ((P(d), C.c_void_p(z.data_ptr() + 2), None, 4 * w, 8 * w, 16 * w), "dz_dev"),
    ]
    for (dp, zp, ip, p0, p1, p2), msg in cases:
        rc = L.b200mvs_set_view_prior_state_device(sc._h, 0, dp, zp, ip, w, h, p0, p1, p2, 1, None)
        err = L.b200mvs_last_error(sc._h).decode()
        assert rc == dmrecon.ERR_INVALID_ARG and err.startswith(fn + ": ") and msg in err, err
    # the pitch of a plane that is not given is not looked at
    assert L.b200mvs_set_view_prior_state_device(sc._h, 0, P(d), None, P(i), w, h, 4 * w, 0, 16 * w, 1, None) == 0
    sc.close()


@pytest.mark.parametrize("name", ["T1", "T2"])
def test_quality(name):
    """Level-1 maps as state priors for level 0 at stride 4: fill within 1 % and median and p95 relative depth error
    within 5 % of the depth-only prior (SURVEY §8c).  n_opt and rounds are printed; no speed-up is asserted."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings(scale=0, nr_recon_neighbors=s.nr_recon_neighbors)
    prior = _earlier(sc, s, refs, 1)
    _set_state(sc, refs, prior, 4, planes=())
    depth_only, dc = _run(sc, st, refs)
    _set_state(sc, refs, prior, 4)
    state, sc_ = _run(sc, st, refs)
    sizes = {v: depth_only[j]["depth"].shape[::-1] for j, v in enumerate(refs)}

    def fe(maps):
        from mve_b200 import synth
        fill, err = [], []
        for j, v in enumerate(refs):
            W, H = sizes[v]
            truth = synth.depth(s, v, W, H)
            d = maps[j]["depth"]
            ok = (d > 0) & (truth > 0)
            fill.append((d > 0).mean())
            err.append(np.abs(d[ok] - truth[ok]) / truth[ok])
        e = np.concatenate(err)
        return float(np.mean(fill)), float(np.median(e)), float(np.percentile(e, 95))
    f0, m0, p0 = fe(depth_only)
    f1, m1, p1 = fe(state)
    print("%s depth-only: fill %.4f median %.3e p95 %.3e rounds %d n_opt %d | state: fill %.4f median %.3e p95 %.3e "
          "rounds %d n_opt %d" % (name, f0, m0, p0, dc["n_rounds"], dc["n_opt"], f1, m1, p1, sc_["n_rounds"], sc_["n_opt"]))
    assert abs(f1 - f0) <= 0.01
    assert m1 <= 1.05 * m0 and p1 <= 1.05 * p0
    sc.close()


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_prior_dz():
    """-s1 --keep-dz, then B200MVS_PRIOR=depth-L1,4 B200MVS_PRIOR_DZ=dz-L1 -s0: the depth and conf of the Python route
    with the same depth and dz; a view whose dz embedding is missing runs with its depth alone and says so."""
    from mve_b200 import dmrecon, synth
    s = golden_scene("T1")
    views = [0, 4, 7]
    lo, hi = 0, 1
    base = ["--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--progress=silent", "--force"]
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        out = subprocess.run([CLI, "-s%d" % hi, "--keep-dz"] + base + ["-l" + ",".join(str(v) for v in views), tmp],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        vd = {v: os.path.join(tmp, "views", "view_%04d.mve" % v) for v in views}
        depth = {v: synth.read_mvei(os.path.join(vd[v], "depth-L%d.mvei" % hi))[:, :, 0] for v in views}
        dz = {v: np.ascontiguousarray(synth.read_mvei(os.path.join(vd[v], "dz-L%d.mvei" % hi))) for v in views}
        assert all(d.shape == depth[v].shape + (2,) and d.dtype == np.float32 for v, d in dz.items())
        os.remove(os.path.join(vd[7], "dz-L%d.mvei" % hi))
        out = subprocess.run([CLI, "-s%d" % lo] + base + ["-l" + ",".join(str(v) for v in views), tmp],
                             capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200MVS_PRIOR="depth-L%d,4" % hi, B200MVS_PRIOR_DZ="dz-L%d" % hi))
        assert out.returncode == 0, out.stdout + out.stderr
        assert 'Prior dz not found for image "0007", using the depth alone.' in out.stdout, out.stdout
        sc = dmrecon.Scene.from_synth(s)
        st = dmrecon.Settings(scale=lo, nr_recon_neighbors=s.nr_recon_neighbors)
        for v in views:
            sc.set_view_prior(v, depth[v], 4, dz=dz[v] if v != 7 else None)
            want, _ = sc.reconstruct(st, [v])
            got_d = synth.read_mvei(os.path.join(vd[v], "depth-L%d.mvei" % lo))[:, :, 0]
            got_c = synth.read_mvei(os.path.join(vd[v], "conf-L%d.mvei" % lo))[:, :, 0]
            assert got_d.tobytes() == want[0]["depth"].tobytes(), v
            assert got_c.tobytes() == want[0]["conf"].tobytes(), v
        sc.close()
