"""Reconstruction masks (-m gpu): b200mvs_set_view_mask / Scene.set_view_mask keep background pixels from being seeded,
queued or optimised.  Identity masks change no byte and no counter; an all-zero mask does no work; silhouettes and
half-planes fill nothing outside the mask and drop exactly the seeds on background pixels (the NumPy restatement of the
seed list); where the unmasked run filled no background pixel the foreground equals it bit for bit; every route (device
maps, point sets, budgets, frontier resumes, the drop-in CLI) gives the host route's masked maps."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests.test_plan_device_emulated import BIG, Inputs, np_seeds
from tests.test_recon_mask import background_map
from tests.util import ROOT, golden_scene

pytestmark = pytest.mark.gpu

KEYS = ("depth", "conf", "dz", "normal", "view_ids")
COUNTERS = ("n_opt", "n_sample_sets", "n_rounds", "n_filled", "n_seeds_processed", "n_seeds_success", "n_entries_peak",
            "n_patch_launches", "n_kernel_launches", "n_grid_barriers")
MODES = {"default": -1, "warp": 1 << 40, "thread": 0}          # thread_min of b200mvs_set_patch_mode
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")


def _settings(s, **kw):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, **kw)


def _map_size(s, v):
    w, h = s.size(v)
    for _ in range(s.scale):
        if min(w, h) < 30:
            break
        w, h = (w + 1) // 2, (h + 1) // 2
    return w, h


def _run(sc, st, refs, masks=None, mode="default", **kw):
    """Maps and counters of one reconstruction with these masks (view -> mask; None: every mask cleared)."""
    sc.set_patch_mode(0, MODES[mode])
    for v in refs:
        sc.set_view_mask(v, None if masks is None else masks.get(v))
    maps, stats = sc.reconstruct(st, refs, **kw)
    return maps, {k: getattr(stats, k) for k in COUNTERS}


def _same(a, b, ia, ib):
    for i, j in zip(ia, ib):
        for k in KEYS:
            assert a[i][k].tobytes() == b[j][k].tobytes(), (i, j, k)


def _silhouettes(s, refs, size="photo"):
    from mve_b200 import synth
    out = {}
    for v in refs:
        w, h = s.size(v) if size == "photo" else _map_size(s, v) if size == "map" else size
        out[v] = synth.silhouette(s, v, w, h)
    return out


def _half_planes(s, refs):
    out = {}
    for k, v in enumerate(refs):
        w, h = s.size(v)
        m = np.full((h, w), 255, np.uint8)
        if k % 2:
            m[: h // 2] = 0                          # upper half background
        else:
            m[:, : (2 * w) // 3] = 0                 # left two thirds background
        out[v] = m
    return out


def _check_outside(s, maps, refs, masks):
    """No filled pixel outside the mask; background pixels are exactly unfilled pixels."""
    n_fg_filled = 0
    for j, v in enumerate(refs):
        m = maps[j]
        H, W = m["depth"].shape
        bg = background_map(masks[v], W, H)
        assert bg.any() and (~bg).any(), v
        assert (m["depth"][bg] == 0).all() and (m["conf"][bg] == 0).all(), v
        assert (m["dz"][bg] == 0).all() and (m["normal"][bg] == 0).all() and (m["view_ids"][bg] == -1).all(), v
        n_fg_filled += int((m["depth"][~bg] > 0).sum())
    return n_fg_filled


def _seeds_on_foreground(s, st, sc, refs, masks):
    """The seeds of processFeatures (the NumPy restatement of the host's seed list), counted on foreground pixels; a seed
    outside the map is kept (it fails in the kernel as without a mask)."""
    box = np.r_[np.full(3, -BIG), np.full(3, BIG)].astype(np.float32)
    I = Inputs(s, st.scale)
    total = kept = 0
    for v in refs:
        seeds = np_seeds(I, v, sc.global_view_selection(st, v), st.scale, box)
        W, H = _map_size(s, v)
        inside = (seeds["x"] >= 0) & (seeds["x"] < W) & (seeds["y"] >= 0) & (seeds["y"] < H)
        bg = np.zeros(len(seeds), bool)
        bgm = background_map(masks[v], W, H)
        bg[inside] = bgm[seeds["y"][inside], seeds["x"][inside]]
        total += len(seeds)
        kept += int((~bg).sum())
    return total, kept


@pytest.mark.parametrize("name", ["T0", "T5", "T6"])
@pytest.mark.parametrize("mode", list(MODES))
def test_identity_masks_are_a_no_op(name, mode):
    """All-nonzero masks at the map's size and at the photo's size: every byte, counter and memory figure as without."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    results = []
    for kind in (None, "map", "photo"):
        sc = dmrecon.Scene.from_synth(s)
        masks = None
        if kind:
            rng = np.random.default_rng(7)
            masks = {}
            for v in refs:
                w, h = _map_size(s, v) if kind == "map" else s.size(v)
                masks[v] = rng.integers(1, 256, (h, w)).astype(np.uint8)
        maps, counters = _run(sc, st, refs, masks, mode)
        results.append((maps, counters, sc.memory_stats().as_dict()))
        sc.close()
    for maps, counters, mem in results[1:]:
        _same(maps, results[0][0], range(len(refs)), range(len(refs)))
        assert counters == results[0][1]
        assert mem == results[0][2]


def test_all_zero_mask_does_nothing():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = [0, 3]
    _, plain = _run(sc, st, refs)
    assert plain["n_filled"] > 0 and plain["n_seeds_processed"] > 0
    zeros = {v: np.zeros((s.size(v)[1], s.size(v)[0]), np.uint8) for v in refs}
    prog = (dmrecon.Progress * len(refs))()
    maps, c = _run(sc, st, refs, zeros, progress=prog)
    assert c["n_filled"] == c["n_seeds_processed"] == c["n_seeds_success"] == c["n_opt"] == c["n_sample_sets"] == 0, c
    assert all(p.filled == 0 for p in prog)
    for m in maps:
        assert not m["depth"].any() and not m["conf"].any() and not m["dz"].any() and not m["normal"].any()
        assert (m["view_ids"] == -1).all()
    sc.close()


@pytest.mark.parametrize("name,kind", [("T2", "photo"), ("T2", "map"), ("T2", (37, 29)), ("T2", (400, 300)), ("T0", "half")])
def test_silhouettes_and_half_planes(name, kind):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = list(range(s.n_views))
    masks = _half_planes(s, refs) if kind == "half" else _silhouettes(s, refs, kind)
    plain, pc = _run(sc, st, refs)
    total, kept = _seeds_on_foreground(s, st, sc, refs, masks)
    assert pc["n_seeds_processed"] == total
    maps, c = _run(sc, st, refs, masks)
    n_fg = _check_outside(s, maps, refs, masks)
    assert c["n_filled"] == n_fg > 0
    assert c["n_seeds_processed"] == kept < total
    assert c["n_seeds_success"] <= pc["n_seeds_success"] and c["n_opt"] < pc["n_opt"]
    again, c2 = _run(sc, st, refs, masks)
    _same(again, maps, range(len(refs)), range(len(refs)))
    assert c2 == c
    for j, v in enumerate(refs[:4]):
        one, _ = _run(sc, st, [v], masks)
        _same(one, maps, [0], [j])
    sc.close()


@pytest.mark.parametrize("mode", ["warp", "thread"])
def test_untextured_background_equals_unmasked(mode):
    """T2's background is flat grey: an optimisation there fails, so wherever the unmasked run filled no background pixel,
    the masked maps equal the unmasked ones on the foreground (one implementation forced: the per-view choice counts
    the background patches; no threshold: the histograms count them too)."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    sc = dmrecon.Scene.from_synth(s)
    st = _settings(s)
    refs = list(range(s.n_views))
    masks = _silhouettes(s, refs)
    plain, _ = _run(sc, st, refs, mode=mode)
    maps, _ = _run(sc, st, refs, masks, mode=mode)
    held = 0
    for j, v in enumerate(refs):
        H, W = plain[j]["depth"].shape
        bg = background_map(masks[v], W, H)
        if (plain[j]["depth"][bg] > 0).any():
            continue
        held += 1
        for k in KEYS:
            assert plain[j][k].tobytes() == maps[j][k].tobytes(), (v, k)      # the background is unfilled in both
    print("untextured background, %s: the precondition held for %d of %d views" % (mode, held, len(refs)))
    assert held > 0
    sc.close()


def test_routes_agree():
    """Device maps, point sets (host and on-device handles), a budget that splits the batch into groups out of order and
    a frontier small enough to resume: the host route's masked maps and what is built from them."""
    import torch
    from mve_b200 import dmrecon
    from tests.test_gpu_reconstruct_pointset import F_SET, host_route, same
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    masks = _silhouettes(s, refs)
    sc = dmrecon.Scene.from_synth(s)
    want, wc = _run(sc, st, refs, masks)

    dev, _ = sc.reconstruct(st, refs, on_device=True)
    torch.cuda.synchronize()
    for j in range(len(refs)):
        for k in KEYS:
            assert dev[j][k].cpu().numpy().tobytes() == want[j][k].tobytes(), (j, k)

    for opts in (F_SET, dict(correspondence=True)):
        full, hmaps = host_route(sc, s, st, refs, opts)
        assert all(m["depth"].tobytes() == w["depth"].tobytes() for m, w in zip(hmaps, want))
        got, stats = sc.reconstruct_pointset(st, refs, opts)
        same(got, full)
        assert stats.n_filled == wc["n_filled"] and stats.n_seeds_processed == wc["n_seeds_processed"]
        on_dev, _ = sc.reconstruct_pointset(st, refs, opts, on_device=True)
        for key in ("vertices", "normals", "confidences"):
            if full[key] is not None:
                assert on_dev[key].cpu().numpy().tobytes() == full[key].tobytes(), key
        if opts.get("correspondence"):
            pix = full["correspondence"]["pixels"]
            views = full["correspondence"]["views"]
            assert len(pix) > 0
            for k, (vid, w, h, first) in enumerate(views):
                end = views[k + 1][3] if k + 1 < len(views) else len(pix)
                bg = background_map(masks[vid], w, h)
                p = pix[first:end].astype(np.int64)
                assert not bg[p[:, 1], p[:, 0]].any(), vid

    sc.set_frontier_capacity(0.01, 1)
    got, _ = _run(sc, st, refs, masks)
    assert sc.frontier_info()["resumes"] >= 1
    _same(got, want, range(len(refs)), range(len(refs)))
    sc.set_frontier_capacity()
    sc.close()

    lazy = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = lazy.memory_stats().fixed
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
    got, _ = _run(lazy, st, refs, masks)
    assert lazy.memory_stats().n_groups == chosen[1]
    _same(got, want, range(len(refs)), range(len(refs)))
    lazy.close()


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built (needs the reference sources at build time)")
def test_cli_reads_mask_embedding():
    """B200MVS_RECON_MASK=mask: the unmodified CLI writes the depth and conf maps of the Python route with the same masks;
    a view without the embedding, or with a 3-channel one, is reconstructed unmasked with scene2pset's message."""
    from mve_b200 import dmrecon, synth
    s = golden_scene("T2")
    st = _settings(s)
    views = [0, 3, 7, 8]
    masks = _silhouettes(s, views)
    sc = dmrecon.Scene.from_synth(s)
    want = {v: _run(sc, st, [v], {v: masks[v]} if v in (0, 3) else None)[0][0] for v in views}
    sc.close()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        for v in (0, 3):
            synth.write_mvei(os.path.join(tmp, "views", "view_%04d.mve" % v, "mask.mvei"), masks[v])
        synth.write_mvei(os.path.join(tmp, "views", "view_0008.mve", "mask.mvei"), np.repeat(masks[8][:, :, None], 3, 2))
        cmd = [CLI, "-s%d" % s.scale, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--progress=silent",
               "--force", "-l" + ",".join(str(v) for v in views), tmp]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, B200MVS_RECON_MASK="mask"))
        assert out.returncode == 0, out.stdout + out.stderr
        assert 'Mask not found for image "0007", skipping.' in out.stdout, out.stdout
        assert 'Expected 1-channel mask for image "0008", skipping.' in out.stdout, out.stdout
        for v in views:
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            depth = synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % s.scale))[:, :, 0]
            conf = synth.read_mvei(os.path.join(vd, "conf-L%d.mvei" % s.scale))[:, :, 0]
            assert depth.tobytes() == want[v]["depth"].tobytes(), v
            assert conf.tobytes() == want[v]["conf"].tobytes(), v
