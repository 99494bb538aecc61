"""Size-independent properties of the GPU path (-m gpu), also at a BASELINE-sized view, plus the error behaviour
of the C ABI (mirrors the exceptions of libs/dmrecon/dmrecon.cc:37-75,222-223)."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden_scene

pytestmark = pytest.mark.gpu


def _gt_depth(scene, view, scale):
    """Analytic ground truth: distance along each pixel's ray to the synthetic surface (mve_b200.synth), through the
    float64 calibration of the view's pyramid level `scale` (tests/camera_reference.py)."""
    import torch
    from mve_b200 import synth
    from tests import camera_reference as CR
    cfg = scene.meta
    surf = synth._Surface(cfg["surface"], np.random.default_rng(0))
    W, H, K = CR.view_levels(scene, view)[scale][:3]
    R = torch.as_tensor(scene.rot[view].astype(np.float64).reshape(3, 3))
    Cc = -(R.T @ torch.as_tensor(scene.trans[view].astype(np.float64)))
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    d = torch.stack([(xs + 0.5 - K[0, 2]) / K[0, 0], (ys + 0.5 - K[1, 2]) / K[1, 1], torch.ones_like(xs)], -1) @ R
    d = d / d.norm(dim=-1, keepdim=True)
    pts, valid = surf.intersect(Cc, d)
    return (pts - Cc).norm(dim=-1).numpy()


FULL_SIZE_CASES = {
    # BASELINE config geometry, reduced number of views so that scene generation stays short; the reference view is
    # reconstructed at the config's full resolution
    "C2": dict(base="C2", over=dict(views=9, grid=(3, 3), features=1500), ref=4, min_fill=0.6),
    "C3": dict(base="C3", over=dict(views=12, grid=(4, 3), features=2500), ref=5, min_fill=0.5),
    "C4": dict(base="C4", over=dict(views=9, grid=(3, 3), features=2500), ref=4, min_fill=0.5),
    "C5": dict(base="C5", over=dict(views=32, features=6000, orbit_views_per_ring=16), ref=3, min_fill=0.15),
}


@pytest.mark.parametrize("case", ["C2", "C3", "C4", "C5"])
def test_full_size_view_properties(case):
    """One reference view at a BASELINE config's full size: structural invariants, ground-truth accuracy, patch-level
    parity with the oracle on inputs taken from the GPU's own result (fixed-point property), idempotence."""
    from mve_b200 import dmrecon, synth
    from oracle import oracle_py as O
    c = FULL_SIZE_CASES[case]
    s = synth.make_scene(c["base"], device="cuda", **c["over"])
    ref = c["ref"]
    g = dmrecon.Scene.from_synth(s)
    gs = dmrecon.Settings(scale=s.scale)
    maps, st = g.reconstruct(gs, [ref])
    m = maps[0]
    H, W = m["depth"].shape
    Ws, Hs = s.width, s.height
    for _ in range(s.scale):
        Ws, Hs = (Ws + 1) // 2, (Hs + 1) // 2
    assert (W, H) == (Ws, Hs)
    filled = m["conf"] > 0
    assert filled.mean() > c["min_fill"], filled.mean()
    assert int(st.n_filled) == int(filled.sum())
    # depth > 0 exactly where conf > 0; confidence is (mean NCC - 0.6) / 0.4 in (0, 1]
    assert ((m["depth"] > 0) == filled).all()
    assert m["conf"].max() <= 1.0 + 1e-6 and m["conf"].min() >= 0.0
    # border band of 2 px is never reconstructed (patch_sampler.cc:47-50)
    assert not filled[:2].any() and not filled[-2:].any() and not filled[:, :2].any() and not filled[:, -2:].any()
    # exactly nrReconNeighbors distinct, ascending local views from the global selection on every filled pixel
    ids = m["view_ids"][filled]
    gsel = g.global_view_selection(gs, ref)
    assert (ids >= 0).all() and (np.diff(ids, axis=1) > 0).all()
    assert set(np.unique(ids)).issubset(set(gsel))
    # unit normals
    n = m["normal"][filled]
    assert np.allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-4)
    # accuracy against the analytic surface
    gt = _gt_depth(s, ref, s.scale)
    err = np.abs(m["depth"] - gt)[filled] / gt[filled]
    assert np.median(err) < 1e-3 and np.percentile(err, 95) < 1e-2
    # fixed point + patch-level parity at full size: re-optimise sampled filled pixels from their own result, on the
    # GPU and with the CPU restatement (only the views of the global selection are loaded into the oracle)
    ys, xs = np.nonzero(filled)
    pick = np.random.default_rng(3).choice(len(ys), 3000, replace=False)
    pin = np.zeros(len(pick), dmrecon.PATCH_IN)
    pin["x"], pin["y"] = xs[pick], ys[pick]
    pin["depth"] = m["depth"][ys[pick], xs[pick]]
    pin["dz_i"], pin["dz_j"] = m["dz"][ys[pick], xs[pick], 0], m["dz"][ys[pick], xs[pick], 1]
    pin["n_local"] = 4
    pin["local_ids"] = m["view_ids"][ys[pick], xs[pick]]
    out = g.optimize_patches(gs, ref, gsel, pin)
    ok = out["conf"] > 0
    assert ok.mean() > 0.97
    assert np.percentile(np.abs(out["depth"] - pin["depth"])[ok] / pin["depth"][ok], 99) < 3e-3
    assert np.percentile(np.abs(out["conf"][ok] - m["conf"][ys[pick], xs[pick]][ok]), 99) < 4e-2
    need = sorted(set(gsel) | {ref})
    remap = {v: i for i, v in enumerate(need)}
    sub = synth.Scene(name=s.name, width=s.width, height=s.height, images=[s.images[v] for v in need], flen=s.flen[need],
                      paspect=s.paspect[need], ppoint=s.ppoint[need], rot=s.rot[need], trans=s.trans[need],
                      feat_pos=s.feat_pos[:1], feat_refs=[np.array([0, 1], np.int32)], scale=s.scale)
    osc = O.OracleScene(sub)
    pin_o = pin.copy()
    pin_o["local_ids"] = np.vectorize(remap.get)(pin["local_ids"])
    oout = osc.optimize_patches(O.default_settings(scale=s.scale), remap[ref], [remap[v] for v in gsel], pin_o)
    both = ok & (oout["conf"] > 0)
    assert (ok != (oout["conf"] > 0)).sum() <= 0.004 * len(pick)
    rel = np.abs(out["depth"] - oout["depth"])[both] / oout["depth"][both]
    assert np.percentile(rel, 99) < 2e-5 and np.percentile(rel, 99.9) < 1e-3
    assert np.percentile(np.abs(out["conf"] - oout["conf"])[both], 99) < 1e-4
    got_ids = np.vectorize(remap.get)(out["local_ids"])
    assert (got_ids != oout["local_ids"]).any(-1)[both].sum() <= 0.004 * len(pick)
    # idempotence of the whole run
    maps2, _ = g.reconstruct(gs, [ref])
    assert (maps2[0]["depth"] == m["depth"]).all() and (maps2[0]["conf"] == m["conf"]).all()


def test_error_behaviour():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    g = dmrecon.Scene.from_synth(s)
    ok = dmrecon.Settings()
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(ok, [99])
    assert e.value.code == -1 and "Master view index out of bounds" in str(e.value)        # dmrecon.cc:37-38
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(dmrecon.Settings(scale=-1), [0])
    assert "Invalid scale factor" in str(e.value)                                           # dmrecon.cc:41-42
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(dmrecon.Settings(scale=9), [0])
    assert "Invalid scale factor" in str(e.value)
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(dmrecon.Settings(filter_width=7), [0])
    assert e.value.code == -6
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(dmrecon.Settings(nr_recon_neighbors=5), [0])
    assert e.value.code == -6
    # a scene whose features never reference the master view: "Global View Selection failed" (dmrecon.cc:222-223)
    g2 = dmrecon.Scene.from_synth(s)
    g2.set_features(s.feat_pos[:3], [np.array([1, 2], np.int32)] * 3)
    with pytest.raises(dmrecon.B200MVSError) as e:
        g2.reconstruct(ok, [0])
    assert e.value.code == -3 and "Global View Selection failed" in str(e.value)
    # a view that was never uploaded is an invalid master view (dmrecon.cc:73-75)
    g3 = dmrecon.Scene(3)
    with pytest.raises(dmrecon.B200MVSError) as e:
        g3.reconstruct(ok, [0])
    assert "Invalid master view" in str(e.value)
    # nrReconNeighbors > available views: zero pixels, no error (SURVEY §8a quirk)
    s4 = golden_scene("T0")
    g4 = dmrecon.Scene.from_synth(s4, views=[0, 1, 2])
    maps, st = g4.reconstruct(ok, [0])
    assert int(st.n_filled) == 0 and not (maps[0]["depth"] > 0).any()


def test_camera_only_views_and_missing_images():
    """SingleView::create vs loadColorImage: cameras of all views, images only where needed (dmrecon.cc:78,238-240)."""
    from mve_b200 import dmrecon
    s = golden_scene("T3")          # 40 views, 20 selected
    st = dmrecon.Settings()
    full = dmrecon.Scene.from_synth(s)
    ref = 7
    want, _ = full.reconstruct(st, [ref])
    g = dmrecon.Scene(s.n_views)
    for v in range(s.n_views):
        g.set_view_camera(v, s.width, s.height, s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    g.set_features(s.feat_pos, s.feat_refs)
    sel = g.global_view_selection(st, ref)
    assert sel == full.global_view_selection(st, ref) and len(sel) == 20
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(st, [ref])
    assert e.value.code == -1 and "not loaded" in str(e.value)
    for v in [ref] + sel[:-1]:
        g.set_view(v, s.images[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(st, [ref])
    assert "selected neighbour" in str(e.value)
    v = sel[-1]
    g.set_view(v, s.images[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    got, _ = g.reconstruct(st, [ref])
    for k in ("depth", "conf", "dz", "view_ids"):
        assert (got[0][k] == want[0][k]).all()


def test_cancel():
    """Progress::cancelled is polled once per frontier round (dmrecon.cc:353) -> B200MVS_ERR_CANCELLED."""
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    g = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings()
    prog = (dmrecon.Progress * 1)()
    prog[0].cancelled = 1
    refs = np.asarray([0], np.int32)
    rc = g._lib.b200mvs_reconstruct(g._h, C.byref(st), 1, refs.ctypes.data_as(C.c_void_p), None, prog, None, None)
    assert rc == -4
    assert prog[0].status == 5


def test_cancel_while_running():
    """A cancel request raised from another thread while the persistent kernel runs (UMVE's cancel button,
    apps/umve/viewinspect/imageoperations.cc:177-184) stops the batch at the next frontier round; live progress
    (filled / queue_size, fancy_progress_printer.cc:84-91) is visible meanwhile."""
    import threading
    import time
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    g = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings(scale=s.scale, frontier_topk=1)          # one pop per round and view: thousands of rounds
    full, stats_full = g.reconstruct(st, [4])
    prog = (dmrecon.Progress * 1)()
    seen = []

    def canceller():
        t0 = time.time()
        while time.time() - t0 < 20.0:
            if prog[0].filled > 200:
                seen.append((int(prog[0].filled), int(prog[0].queue_size), int(prog[0].status)))
                prog[0].cancelled = 1
                return
            time.sleep(0.0005)
    th = threading.Thread(target=canceller)
    th.start()
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.reconstruct(st, [4], progress=prog)
    th.join()
    assert e.value.code == -4
    assert seen and seen[0][2] == 3 and seen[0][1] > 0
    assert prog[0].status == 5
    assert 200 < prog[0].filled < stats_full.n_filled


def test_cancel_one_view_of_a_batch():
    """Cancelling ONE view of a running batch drops only that view's queue (status RECON_CANCELLED, no maps); the other
    view finishes with exactly the maps it gets alone."""
    import threading
    import time
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    g = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings(scale=s.scale, frontier_topk=4)
    alone, _ = g.reconstruct(st, [2])
    prog = (dmrecon.Progress * 2)()

    def canceller():
        t0 = time.time()
        while time.time() - t0 < 20.0:
            if prog[1].filled > 200:
                prog[1].cancelled = 1
                return
            time.sleep(0.0005)
    th = threading.Thread(target=canceller)
    th.start()
    maps, stats = g.reconstruct(st, [2, 4], progress=prog)
    th.join()
    assert prog[1].status == 5 and prog[0].status == 0
    assert 200 < prog[1].filled
    for k in ("depth", "conf", "dz", "view_ids"):
        assert (maps[0][k] == alone[0][k]).all()


def test_planned_views_give_the_same_maps():
    """b200mvs_plan_views only moves the host part of DMRecon::start ahead of the call: same maps with and without a prepared
    plan, a plan is consumed once, a plan made for other settings is ignored."""
    import threading
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    g = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings(scale=s.scale)
    base, _ = g.reconstruct(st, [2, 5])
    g.plan_views(st, [2, 5])
    a, _ = g.reconstruct(st, [2, 5])
    g.plan_views(dmrecon.Settings(scale=s.scale, global_vs_max=3), [2, 5])      # other settings: must not be used
    b, _ = g.reconstruct(st, [2, 5])
    # planning the next batch from another thread while a batch runs
    th = threading.Thread(target=g.plan_views, args=(st, [2, 5]))
    th.start()
    c, _ = g.reconstruct(st, [4])
    th.join()
    d, _ = g.reconstruct(st, [2, 5])
    for got in (a, b, d):
        for j in range(2):
            for k in ("depth", "conf", "dz", "view_ids"):
                assert (got[j][k] == base[j][k]).all()


def test_image_channel_variants():
    """Grey and RGBA inputs are expanded / stripped like image_pyramid.cc:65-73."""
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    g = dmrecon.Scene(2)
    grey = s.images[0][:, :, 1]
    rgba = np.concatenate([s.images[0], np.full(s.images[0].shape[:2] + (1,), 7, np.uint8)], -1)
    g.set_view(0, grey, s.flen[0], s.paspect[0], s.ppoint[0], s.rot[0], s.trans[0])
    g.set_view(1, rgba, s.flen[0], s.paspect[0], s.ppoint[0], s.rot[0], s.trans[0])
    assert (g.level(0, 0) == np.repeat(grey[:, :, None], 3, 2)).all()
    assert (g.level(1, 0) == s.images[0]).all()
