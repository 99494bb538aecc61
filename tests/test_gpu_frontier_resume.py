"""Frontier grow-and-resume (-m gpu): a launch whose frontier outgrows its capacity stops before the pushes of a round,
grows its arrays and resumes.  With a capacity small enough to force several resumes the maps must be bit-identical to the
default capacity, which never resumes on these scenes, and so must the work counters."""
import os
import threading
import time

import numpy as np
import pytest

from tests.util import ROOT, golden_scene

pytestmark = pytest.mark.gpu

KEYS = ("depth", "conf", "dz", "normal", "view_ids")
COUNTERS = ("n_opt", "n_rounds", "n_filled", "n_seeds_processed", "n_seeds_success", "n_entries_peak")
SMALL = (0.01, 1)                       # entries per pixel, floor: far below the peak of every test scene


def _settings(s, **kw):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, **kw)


def _same(a, b, idx_a, idx_b):
    for i, j in zip(idx_a, idx_b):
        for k in KEYS:
            assert a[i][k].tobytes() == b[j][k].tobytes(), (i, k)


def _run(sc, st, refs, capacity=None, **kw):
    sc.set_frontier_capacity(*(capacity or ()))
    maps, stats = sc.reconstruct(st, refs, **kw)
    return maps, {k: getattr(stats, k) for k in COUNTERS}, sc.frontier_info()


def _check(sc, st, refs, min_resumes=2):
    want, wstats, winfo = _run(sc, st, refs)
    assert winfo["resumes"] == 0 and winfo["initial"] == winfo["final"], winfo
    got, gstats, ginfo = _run(sc, st, refs, SMALL)
    assert ginfo["resumes"] >= min_resumes and ginfo["final"] > ginfo["initial"], ginfo
    _same(got, want, range(len(refs)), range(len(refs)))
    assert gstats == wstats
    sc.set_frontier_capacity()
    return ginfo


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T3", "T4", "T5", "T6"])
def test_resume_bit_identical(name):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    _check(sc, st, list(range(s.n_views)))
    for v in (0, s.n_views - 1):
        _check(sc, st, [v], min_resumes=1)
    sc.close()


def test_resume_thresholded():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s)
    _check(sc, _settings(s, frontier_topk=64), list(range(s.n_views)))
    sc.close()


@pytest.mark.parametrize("thread_min", [0, 1 << 40])
def test_resume_one_patch_implementation(thread_min):
    """Every round one thread per patch (thread_min 0, the tile-grouped run list) or one warp per patch."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    sc = dmrecon.Scene.from_synth(s)
    sc.set_patch_mode(0, thread_min)
    _check(sc, _settings(s), list(range(s.n_views)))
    sc.close()


def test_resume_lazy_budgeted_groups():
    """A lazy scene within a budget, split into several launches that each resume.  The planner packs a group up to the
    budget at its initial capacity, so growing needs room left by the packing or by pyramids the group does not need:
    budgets are tried from the most room down; one that is too tight fails with B200MVS_ERR_OVERFLOW and the context goes
    on with the next."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s, global_vs_max=4)
    refs = list(range(s.n_views))
    full = dmrecon.Scene.from_synth(s)
    want, wstats, _ = _run(full, st, refs)
    full.close()
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    sc.set_frontier_capacity(*SMALL)
    total = sc.working_set(st, refs)
    single = max(sc.working_set(st, [r]) for r in refs)
    done = []
    for frac in (0.95, 0.9, 0.8, 0.7, 0.6, 0.5):
        avail = max(single, int(total * frac))
        n_plan, _ = sc.plan_batches(st, refs, avail)
        if n_plan < 2:
            continue
        sc.set_image_source(lambda v: s.images[v], fixed + avail)
        try:
            got, stats = sc.reconstruct(st, refs)
        except dmrecon.B200MVSError as e:
            assert e.code == dmrecon.ERR_OVERFLOW, e
            continue
        info, m = sc.frontier_info(), sc.memory_stats()
        assert info["resumes"] >= 1 and m.n_groups == n_plan and m.peak <= fixed + avail, (info, m.as_dict())
        _same(got, want, refs, refs)
        assert stats.n_opt == wstats["n_opt"] and stats.n_filled == wstats["n_filled"]
        done.append(n_plan)
    assert done, "no budget both split the batch and left room to grow"
    sc.close()


def test_resume_c2_view_at_baseline_size():
    from mve_b200 import dmrecon, synth
    s = synth.make_scene("C2", device="cuda")
    st = dmrecon.Settings(scale=s.scale)
    v = 5
    plan = dmrecon.Scene.from_synth(s, lazy=True)
    views = sorted(set(plan.global_view_selection(st, v)) | {v})
    plan.close()
    sc = dmrecon.Scene.from_synth(s, views=views)
    info = _check(sc, st, [v])
    sc.close()
    print("C2 view %d: %s" % (v, info))


def _watch(prog, n, stop, samples, cancel_view=None):
    """Records progress.filled of every view until `stop`; cancels `cancel_view` once it has filled pixels."""
    while not stop.is_set():
        samples.append([prog[k].filled for k in range(n)])
        if cancel_view is not None and prog[cancel_view].filled > 0:
            prog[cancel_view].cancelled = 1
        time.sleep(0.0002)


def test_cancel_and_progress_across_resumes():
    """frontier_topk = 64 makes many short rounds, so the run is long enough to watch: progress.filled never decreases
    across the resumes, and a view cancelled while the launch grows ends cancelled while the others keep their maps."""
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    st = _settings(s, frontier_topk=64)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    want, _, _ = _run(sc, st, refs)
    for victim in (None, 1):
        prog = (dmrecon.Progress * len(refs))()
        stop, samples = threading.Event(), []
        t = threading.Thread(target=_watch, args=(prog, len(refs), stop, samples, victim))
        t.start()
        try:
            got, _, info = _run(sc, st, refs, SMALL, progress=prog)
        finally:
            stop.set()
            t.join()
        assert info["resumes"] >= 2, info
        a = np.asarray(samples, np.int64)
        assert len(a) > 10 and (np.diff(a, axis=0) >= 0).all()
        others = [r for r in refs if r != victim]
        if victim is not None:
            assert prog[victim].status == 5
        assert all(prog[r].status == 0 for r in others)
        _same(got, want, others, others)
    sc.close()


def test_budget_too_small_to_grow():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    st = _settings(s)
    refs = list(range(s.n_views))
    full = dmrecon.Scene.from_synth(s)
    want, _, _ = _run(full, st, refs)
    full.close()
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    sc.set_frontier_capacity(*SMALL)
    sc.set_image_source(lambda v: s.images[v], fixed + sc.working_set(st, refs))
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, refs)
    assert e.value.code == dmrecon.ERR_OVERFLOW
    assert "needs" in str(e.value) and "allows" in str(e.value)
    assert sc.memory_stats().peak <= fixed + sc.working_set(st, refs)
    sc.set_image_source(lambda v: s.images[v], fixed + 4 * sc.working_set(st, refs))
    got, _ = sc.reconstruct(st, refs)
    assert sc.frontier_info()["resumes"] >= 1
    _same(got, want, refs, refs)
    sc.close()


CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_with_frontier_capacity():
    """The drop-in CLI with B200MVS_FRONTIER_CAPACITY writes the same maps as without it."""
    import shutil
    import subprocess
    import tempfile
    from mve_b200 import synth
    s = golden_scene("T0")
    views = list(range(s.n_views))
    names = ["%s-L%d.mvei" % (k, s.scale) for k in ("depth", "conf", "dz")]
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, os.path.join(tmp, "a"))
        shutil.copytree(os.path.join(tmp, "a"), os.path.join(tmp, "b"))
        for d, cap in (("a", None), ("b", "%g,%d" % SMALL)):
            env = dict(os.environ, OMP_NUM_THREADS="6")
            env.pop("B200MVS_DEVICE_BUDGET_MB", None)
            env.pop("B200MVS_FRONTIER_CAPACITY", None)
            if cap:
                env["B200MVS_FRONTIER_CAPACITY"] = cap
            cmd = [CLI, "-s%d" % s.scale, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--keep-dz",
                   "--progress=silent", "--force", "-l" + ",".join(str(v) for v in views), os.path.join(tmp, d)]
            r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)
            assert r.returncode == 0, r.stdout + r.stderr
        for v in views:
            for n in names:
                a = open(os.path.join(tmp, "a", "views", "view_%04d.mve" % v, n), "rb").read()
                b = open(os.path.join(tmp, "b", "views", "view_%04d.mve" % v, n), "rb").read()
                assert a == b, (v, n)
