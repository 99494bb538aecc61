"""One pyramid level per entry (-m gpu): b200mvs_reconstruct_levels, its device form, b200mvs_pset_add_reconstruction_levels
and the drop-in dmrecon batching views of different scales into one call.

Each entry's maps must be byte for byte those of a single-level reconstruct of its view at its level, on T6 at the levels
--max-pixels=10000 gives (1 for the 179x180 views, 0 for the 118x58 and 58x118 ones) and on T0 with every view at levels 0
and 1: host maps, on_device, a budget that splits the call into groups out of entry order, host and device masks, prepared
plans at one level, a cancelled entry, and the point set of the entries."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from tests import pset_reference as S
from tests.test_gpu_parity import CLI_CONF_P99
from tests.test_levels_abi import _max_pixels_level
from tests.util import ROOT, golden_scene, map_stats

pytestmark = pytest.mark.gpu

MAPS = ("depth", "conf", "dz", "normal", "view_ids")
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")
REF_CLI = os.path.join(ROOT, "oracle", "_ref", "dmrecon")


def _settings(s, scale=None):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale if scale is None else scale, nr_recon_neighbors=s.nr_recon_neighbors)


def _entries(name, s):
    if name == "T6":
        views = list(range(s.n_views))
        return views, [_max_pixels_level(*s.size(v), 10000) for v in views]
    views = [v for v in range(s.n_views) for _ in (0, 1)]
    return views, [k % 2 for k in range(len(views))]


@pytest.fixture(scope="module")
def scenes():
    from mve_b200 import dmrecon
    cache = {}

    def get(name):
        if name not in cache:
            s = golden_scene(name)
            cache[name] = (s, dmrecon.Scene.from_synth(s))
        return cache[name]
    yield get
    for _, sc in cache.values():
        sc.close()


def _host(m):
    return {k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in m.items()}


def per_level(sc, s, views, levels, **kw):
    """The maps of each entry from single-level calls (one per distinct level, over the entries at that level), and the
    summed counters of those calls."""
    out = [None] * len(views)
    sums = dict(n_seeds_processed=0, n_seeds_success=0, n_filled=0)
    for l in sorted(set(levels)):
        idx = [j for j in range(len(views)) if levels[j] == l]
        maps, st = sc.reconstruct(_settings(s, l), [views[j] for j in idx], **kw)
        for j, m in zip(idx, maps):
            out[j] = _host(m)
        for k in sums:
            sums[k] += getattr(st, k)
    return out, sums


def same_maps(got, want, views, levels, sc=None):
    assert len(got) == len(want)
    for j, (a, b) in enumerate(zip(got, want)):
        a = _host(a)
        if sc is not None:
            h, w = sc.level(views[j], levels[j]).shape[:2]
            assert a["depth"].shape == (h, w), (j, a["depth"].shape, (h, w))
        for k in MAPS:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (j, k)


@pytest.mark.parametrize("name", ["T6", "T0"])
@pytest.mark.parametrize("on_device", [False, True])
def test_maps_equal_single_level_calls(scenes, name, on_device):
    s, sc = scenes(name)
    views, levels = _entries(name, s)
    order = np.random.default_rng(1).permutation(len(views)).tolist()
    views, levels = [views[j] for j in order], [levels[j] for j in order]
    want, sums = per_level(sc, s, views, levels)
    got, st = sc.reconstruct(_settings(s, scale=-3), views, on_device=on_device, scales=levels)
    same_maps(got, want, views, levels, sc)
    assert len(set(levels)) == 2 and st.n_filled > 0
    for k, v in sums.items():
        assert getattr(st, k) == v, k
    # uniform levels: the call without levels, counters included
    lv = [s.scale] * s.n_views
    a, sa = sc.reconstruct(_settings(s), list(range(s.n_views)), on_device=on_device, scales=lv)
    b, sb = sc.reconstruct(_settings(s), list(range(s.n_views)), on_device=on_device)
    same_maps(a, [_host(m) for m in b], list(range(s.n_views)), lv)
    for k in ("n_opt", "n_sample_sets", "n_rounds", "n_filled", "n_seeds_processed", "n_seeds_success", "n_entries_peak"):
        assert getattr(sa, k) == getattr(sb, k), k


def test_budget_groups_out_of_order_and_loads(scenes):
    """A budget that splits the entries into groups, not in entry order, gives the same maps; with an image source a view
    needed at two levels is fetched once per call."""
    from mve_b200 import dmrecon
    s, whole = scenes("T0")
    views, levels = _entries("T0", s)
    order = np.random.default_rng(5).permutation(len(views)).tolist()
    views, levels = [views[j] for j in order], [levels[j] for j in order]
    want, _ = per_level(whole, s, views, levels)
    st = _settings(s)

    # unlimited budget: every needed view is fetched once, though most are needed at two levels
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    got, _ = sc.reconstruct(st, views, scales=levels)
    same_maps(got, want, views, levels)
    one_call = sc.memory_stats().n_loads
    assert one_call == s.n_views
    sc.close()
    two_calls = 0
    for l in (0, 1):
        sc = dmrecon.Scene.from_synth(s, lazy=True)
        sc.reconstruct(_settings(s, l), [views[j] for j in range(len(views)) if levels[j] == l])
        two_calls += sc.memory_stats().n_loads
        sc.close()
    assert one_call <= two_calls

    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    single = max(sc.working_set(st, [v], scales=[l]) for v, l in zip(views, levels))
    total = sc.working_set(st, views, scales=levels)
    chosen = None
    for avail in np.linspace(single, total, 60).astype(np.int64).tolist():
        n, groups = sc.plan_batches(st, views, avail, scales=levels)
        if n >= 2 and (np.diff(groups) < 0).any():
            chosen = (avail, n)
            break
    assert chosen, "no budget gives an out-of-order grouping"
    sc.set_image_source(lambda v: s.images[v], fixed + chosen[0])
    got, stats = sc.reconstruct(st, views, scales=levels)
    m = sc.memory_stats()
    same_maps(got, want, views, levels)
    assert m.n_groups == chosen[1] and stats.n_patch_launches >= m.n_groups and m.peak <= m.budget
    got, _ = sc.reconstruct(st, views, scales=levels, on_device=True)
    same_maps(got, want, views, levels)
    sc.close()


@pytest.mark.parametrize("on_device", [False, True])
def test_masks(scenes, on_device):
    """Host and device masks are per view; each entry resamples its view's mask to its own map size."""
    import torch
    s, sc = scenes("T0")
    views, levels = _entries("T0", s)
    masked = (0, 2, 3)
    try:
        for v in masked:
            w, h = s.size(v)
            m = S.make_mask(h, w, seed=v)
            sc.set_view_mask(v, torch.from_numpy(m).cuda() if on_device else m, on_device=on_device)
        want, sums = per_level(sc, s, views, levels)
        got, st = sc.reconstruct(_settings(s), views, scales=levels)
        same_maps(got, want, views, levels)
        assert st.n_seeds_processed == sums["n_seeds_processed"] and st.n_filled == sums["n_filled"]
        with_masks = got
    finally:
        for v in masked:
            sc.set_view_mask(v, None)
    clear, _ = sc.reconstruct(_settings(s), views, scales=levels)
    assert any((a["depth"] != b["depth"]).any() for a, b in zip(with_masks, clear))


def test_prepared_plans_at_one_level(scenes):
    s, sc = scenes("T0")
    views, levels = _entries("T0", s)
    want, _ = per_level(sc, s, views, levels)
    sc.plan_views(_settings(s, 1), list(range(s.n_views)))
    got, _ = sc.reconstruct(_settings(s), views, scales=levels)
    info = sc.plan_info()
    assert info["n_prepared"] == levels.count(1)
    assert info["n_prepared"] + info["n_device"] + info["n_host"] == len(views)
    same_maps(got, want, views, levels)


def test_cancelled_entry(scenes):
    from mve_b200 import dmrecon
    s, sc = scenes("T6")
    views, levels = _entries("T6", s)
    want, _ = per_level(sc, s, views, levels)
    prog = (dmrecon.Progress * len(views))()
    prog[3].cancelled = 1
    got, _ = sc.reconstruct(_settings(s), views, scales=levels, progress=prog)
    keep = [j for j in range(len(views)) if j != 3]
    same_maps([got[j] for j in keep], [want[j] for j in keep], [views[j] for j in keep], [levels[j] for j in keep])
    assert prog[3].status == 5 and all(prog[j].status == 0 for j in keep)


@pytest.mark.parametrize("on_device", [False, True])
def test_pointset(scenes, on_device):
    """reconstruct_pointset(scales=...) is scene_pointset over the entries' maps and level images, in entry order."""
    from mve_b200 import depthmap as D
    from tests.test_gpu_reconstruct_pointset import F_SET, same
    for name in ("T6", "T0"):
        s, sc = scenes(name)
        views, levels = _entries(name, s)
        maps, _ = per_level(sc, s, views, levels)
        host = [dict(id=v, depth=maps[j]["depth"], camera=S.camera_of(s, v), color=sc.level(v, levels[j]))
                for j, v in enumerate(views)]
        want = D.scene_pointset(host, F_SET)
        got, st = sc.reconstruct_pointset(_settings(s), views, F_SET, scales=levels, on_device=on_device)
        if on_device:
            got = dict(got, **{k: (got[k].cpu().numpy() if got[k] is not None else None)
                               for k in ("vertices", "normals", "colors", "values", "confidences")})
        same(got, want)
        assert len(got["views"]) == len(views) and len(want["vertices"]) > 0


def _mvei_bytes(scene_dir, v, prefix):
    vd = os.path.join(scene_dir, "views", "view_%04d.mve" % v)
    names = sorted(f for f in os.listdir(vd) if re.match(prefix + r"-L\d+\.mvei$", f))
    return {f: open(os.path.join(vd, f), "rb").read() for f in names}


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_batches_views_of_different_scales():
    """--max-pixels=10000 on T6 with 10 threads: one b200mvs_reconstruct_levels call (every 'Reconstructed view' line
    reports the same batch), and the files of -s0 over the small views plus -s1 over the large ones."""
    from mve_b200 import synth
    s = golden_scene("T6")
    small = [v for v in range(s.n_views) if _max_pixels_level(*s.size(v), 10000) == 0]
    large = [v for v in range(s.n_views) if v not in small]
    assert small and large
    base = ["--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--keep-dz", "--progress=simple", "--force"]
    env = dict(os.environ, OMP_NUM_THREADS="10")
    with tempfile.TemporaryDirectory() as tmp:
        mixed, split = os.path.join(tmp, "mixed"), os.path.join(tmp, "split")
        synth.write_mve_scene(s, mixed)
        synth.write_mve_scene(s, split)
        out = subprocess.run([CLI, "--max-pixels=10000"] + base + [mixed], capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        lines = re.findall(r"Reconstructed view (\d+) \(batch of all views in flight: (\d+) features processed, (\d+) "
                           r"succeeded optimization, (\d+) frontier rounds\)", out.stdout)
        assert sorted(int(l[0]) for l in lines) == list(range(s.n_views))
        assert len({l[1:] for l in lines}) == 1, lines                      # one batch
        for scale, vs in ((0, small), (1, large)):
            r = subprocess.run([CLI, "-s%d" % scale] + base + ["-l" + ",".join(map(str, vs)), split], capture_output=True,
                               text=True, timeout=600, env=env)
            assert r.returncode == 0, r.stdout + r.stderr
        for v in range(s.n_views):
            level = 0 if v in small else 1
            for prefix in ("depth", "conf", "dz"):
                a, b = _mvei_bytes(mixed, v, prefix), _mvei_bytes(split, v, prefix)
                assert list(a) == ["%s-L%d.mvei" % (prefix, level)] and a == b, (v, prefix)
        if not os.path.exists(REF_CLI):
            return
        r = subprocess.run([REF_CLI, "--max-pixels=10000"] + base + [split], capture_output=True, text=True, timeout=3000, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
        # the CLI tolerances over the whole scene; per view, a map of 6 844 pixels moves its IoU by 0.015 per hundred pixels
        ref, got = {k: [] for k in ("depth", "conf", "dz")}, {k: [] for k in ("depth", "conf", "dz")}
        per_view = {}
        for v in range(s.n_views):
            level = 0 if v in small else 1
            for k in ref:
                ref[k].append(synth.read_mvei(os.path.join(split, "views", "view_%04d.mve" % v, "%s-L%d.mvei" % (k, level))).reshape(-1, 1 if k != "dz" else 2))
                got[k].append(synth.read_mvei(os.path.join(mixed, "views", "view_%04d.mve" % v, "%s-L%d.mvei" % (k, level))).reshape(-1, 1 if k != "dz" else 2))
            per_view[v] = round(float(map_stats(ref["depth"][-1][:, 0], got["depth"][-1][:, 0])[0]), 4)
        print("per-view depth IoU against the reference CLI:", per_view)
        ref, got = {k: np.concatenate(a) for k, a in ref.items()}, {k: np.concatenate(a) for k, a in got.items()}
        iou, rel, both = map_stats(ref["depth"][:, 0], got["depth"][:, 0])
        assert iou > 0.99 and min(per_view.values()) > 0.95, (iou, per_view)
        assert np.percentile(rel, 50) < 5e-4 and np.percentile(rel, 99) < 5e-3, per_view
        assert np.percentile(np.abs(ref["conf"][:, 0] - got["conf"][:, 0])[both], 99) < CLI_CONF_P99.get("T6", 2e-2)
        assert np.percentile(np.abs(ref["dz"] - got["dz"])[both], 99) < 1e-2
