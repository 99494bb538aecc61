"""Reconstruction within a device budget (-m gpu): images loaded on demand through an image source, batches split into
groups that fit, pyramids evicted least recently used first.  The maps of every view must be byte-identical to one launch
of the whole batch without a source: a view's maps do not depend on which views share its launch."""
import os

import pytest

from tests.util import ROOT, golden_scene

pytestmark = pytest.mark.gpu

KEYS = ("depth", "conf", "dz", "normal", "view_ids")


def _settings(s):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)


@pytest.fixture(scope="module")
def baseline():
    """Golden scene -> (scene, settings, maps of all views in one call without a source, level images of every view)."""
    from mve_b200 import dmrecon
    cache = {}

    def get(name):
        if name not in cache:
            s = golden_scene(name)
            g = dmrecon.Scene.from_synth(s)
            st = _settings(s)
            maps, _ = g.reconstruct(st, list(range(s.n_views)))
            levels = {v: [g.level(v, l) for l in range(g.num_levels(v))] for v in range(s.n_views)}
            g.close()
            cache[name] = (s, st, maps, levels)
        return cache[name]
    return get


def _budgets(sc, st, refs):
    """Budgets (fixed + available) for one group, two or three groups, one view per group."""
    fixed = sc.memory_stats().fixed
    total = sc.working_set(st, refs)
    single = max(sc.working_set(st, [r]) for r in refs)
    out = {"one": fixed + total, "per_view": fixed + single}
    for frac in (0.7, 0.6, 0.5, 0.8, 0.4, 0.9):
        avail = max(single, int(total * frac))
        n, _ = sc.plan_batches(st, refs, avail)
        if n in (2, 3):
            out["few"] = fixed + avail
            break
    return out


def _same(a, b, views):
    for v in views:
        for k in KEYS:
            assert a[v][k].tobytes() == b[v][k].tobytes(), (v, k)


@pytest.mark.parametrize("name", ["T0", "T1", "T2"])
def test_groups_bit_identical(baseline, name):
    from mve_b200 import dmrecon
    s, st, want, levels = baseline(name)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    budgets = _budgets(sc, st, refs)
    assert "few" in budgets
    for tag in ("one", "few", "per_view"):
        sc.set_image_source(lambda v: s.images[v], budgets[tag])
        fixed = sc.memory_stats().fixed
        n_plan, _ = sc.plan_batches(st, refs, budgets[tag] - fixed)
        before = sc.memory_stats()
        got, stats = sc.reconstruct(st, refs)
        m = sc.memory_stats()
        _same(got, want, refs)
        assert m.peak <= m.budget == budgets[tag], (tag, m.as_dict())
        assert m.n_groups == n_plan and stats.n_patch_launches == n_plan
        assert {"one": 1, "per_view": len(refs)}.get(tag, n_plan) == n_plan and (tag != "few" or n_plan in (2, 3))
        if tag == "per_view":
            # a group evicts only pyramids it does not need: in scenes where every view selects all others there are none
            if any(len(set(sc.global_view_selection(st, r)) | {r}) < len(refs) for r in refs):
                assert m.n_evictions > before.n_evictions
            # an evicted view is fetched again: its pyramid is bitwise what it was before the eviction
            for v in refs:
                for l, img in enumerate(levels[v]):
                    assert sc.level(v, l).tobytes() == img.tobytes(), (v, l)
            assert sc.memory_stats().peak <= budgets[tag]
    sc.close()


def test_lazy_loads_only_needed_views(baseline):
    """With room for everything, each needed image is loaded exactly once: references and their selections only
    (dmrecon.cc:238-240)."""
    from mve_b200 import dmrecon
    s, _, _, _ = baseline("T2")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, global_vs_max=4)
    refs = [0, 3]
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    needed = set(refs)
    for r in refs:
        needed |= set(sc.global_view_selection(st, r))
    assert len(needed) < s.n_views
    got, _ = sc.reconstruct(st, refs)
    m = sc.memory_stats()
    assert m.n_loads == len(needed) and m.n_evictions == 0 and m.n_groups == 1
    assert m.bytes_loaded == len(needed) * s.width * s.height * 3
    sc.reconstruct(st, refs)
    assert sc.memory_stats().n_loads == len(needed)
    sc.close()


def test_budget_below_one_view(baseline):
    from mve_b200 import dmrecon
    s, st, want, _ = baseline("T0")
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    smallest = min(sc.working_set(st, [r]) for r in refs)
    sc.set_image_source(lambda v: s.images[v], fixed + smallest - 1)
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, refs)
    assert e.value.code == dmrecon.ERR_NO_MEMORY and e.value.failed_view == refs[0]
    sc.set_image_source(lambda v: s.images[v], fixed + sc.working_set(st, refs))
    got, _ = sc.reconstruct(st, refs)
    _same(got, want, refs)
    sc.close()


def test_cancel_view_of_last_group(baseline):
    from mve_b200 import dmrecon
    s, st, want, _ = baseline("T1")
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    budget = _budgets(sc, st, refs)["few"]
    sc.set_image_source(lambda v: s.images[v], budget)
    n, groups = sc.plan_batches(st, refs, budget - sc.memory_stats().fixed)
    victim = [r for r, g in zip(refs, groups) if g == n - 1][0]
    prog = (dmrecon.Progress * len(refs))()
    prog[victim].cancelled = 1
    got, _ = sc.reconstruct(st, refs, progress=prog)
    assert prog[victim].status == 5
    others = [r for r in refs if r != victim]
    assert all(prog[r].status == 0 for r in others)
    _same(got, want, others)
    sc.close()


def test_maps_on_device_needs_one_group(baseline):
    from mve_b200 import dmrecon
    s, st, _, _ = baseline("T0")
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    sc.set_image_source(lambda v: s.images[v], _budgets(sc, st, refs)["per_view"])
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, refs, download=False)
    assert e.value.code == -1                            # B200MVS_ERR_INVALID_ARG
    sc.close()


def test_c4_all_views_in_16_gib():
    """C4 (32 views of 4096 x 3072) in one call within 16 GiB; without a budget the batch asks for far more."""
    import torch
    from mve_b200 import dmrecon, synth
    s = synth.make_scene("C4", device="cuda")
    torch.cuda.empty_cache()
    st = _settings(s)
    refs = list(range(s.n_views))
    budget = 16 << 30
    sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget)
    got, _ = sc.reconstruct(st, refs, want=("depth", "conf", "dz", "normal", "view_ids"))
    m = sc.memory_stats()
    assert m.peak <= budget and m.n_groups > 1
    assert sc.working_set(st, refs) > budget
    sel = {v: sc.global_view_selection(st, v) for v in (0, 13, 31)}
    sc.close()
    for v in (0, 13, 31):
        single = dmrecon.Scene.from_synth(s, views=sorted(set(sel[v]) | {v}))
        want, _ = single.reconstruct(st, [v])
        single.close()
        for k in KEYS:
            assert got[v][k].tobytes() == want[0][k].tobytes(), (v, k)


CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")


def _run_cli(s, tmp, views, budget_mb=None):
    import subprocess
    cmd = [CLI, "-s%d" % s.scale, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--keep-dz",
           "--progress=silent", "--force", "-l" + ",".join(str(v) for v in views), tmp]
    env = dict(os.environ, OMP_NUM_THREADS="6")
    env.pop("B200MVS_DEVICE_BUDGET_MB", None)
    if budget_mb is not None:
        env["B200MVS_DEVICE_BUDGET_MB"] = str(budget_mb)
    return subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_within_budget():
    """The drop-in CLI with B200MVS_DEVICE_BUDGET_MB: a budget that splits the batch writes the same bytes as a run without
    it; a budget below one view fails every view and writes no depth map."""
    import shutil
    import tempfile
    from mve_b200 import dmrecon, synth
    s = golden_scene("T0")
    st = _settings(s)
    views = list(range(s.n_views))
    plan = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = plan.memory_stats().fixed
    single = [plan.working_set(st, [v]) for v in views]
    mb = 1 << 20
    split_mb = -(-(fixed + max(single)) // mb)
    n_groups, _ = plan.plan_batches(st, views, split_mb * mb - fixed)
    assert n_groups >= 3
    low_mb = (fixed + min(single) - 1) // mb
    assert low_mb >= 1
    plan.close()
    names = ["%s-L%d.mvei" % (k, s.scale) for k in ("depth", "conf", "dz")]
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, os.path.join(tmp, "a"))
        shutil.copytree(os.path.join(tmp, "a"), os.path.join(tmp, "b"))
        shutil.copytree(os.path.join(tmp, "a"), os.path.join(tmp, "c"))
        r = _run_cli(s, os.path.join(tmp, "a"), views)
        assert r.returncode == 0, r.stdout + r.stderr
        r = _run_cli(s, os.path.join(tmp, "b"), views, split_mb)
        assert r.returncode == 0, r.stdout + r.stderr
        for v in views:
            for n in names:
                a = open(os.path.join(tmp, "a", "views", "view_%04d.mve" % v, n), "rb").read()
                b = open(os.path.join(tmp, "b", "views", "view_%04d.mve" % v, n), "rb").read()
                assert a == b, (v, n)
        r = _run_cli(s, os.path.join(tmp, "c"), views, low_mb)
        assert r.stderr.count("on its own") == len(views), r.stdout + r.stderr
        for v in views:
            assert not os.path.exists(os.path.join(tmp, "c", "views", "view_%04d.mve" % v, names[0]))
