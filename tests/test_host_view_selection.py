"""Host logic of the product without a GPU: the planning context (B200MVS_DEVICE_NONE) runs the library's own
analyzeFeatures + GlobalViewSelection (dmrecon.cc:179-241, global_view_selection.cc) - restructured for speed in
mve_b200/csrc/b200mvs.cu - and must reproduce the reference's printed selections exactly (golden lines from
oracle/_ref/dmrecon, tests/golden/make_golden.py); compute entry points must refuse to run."""
import os
import re

import numpy as np
import pytest

from tests.util import ROOT, golden_ref, golden_scene


def _planning_scene(s, n_views=None):
    from mve_b200 import dmrecon
    g = dmrecon.Scene(n_views or s.n_views, device=-1)
    for v in range(s.n_views):
        g.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    g.set_features(s.feat_pos, s.feat_refs)
    return g


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T3", "T4", "T5", "T6"])
def test_global_view_selection_matches_reference(name):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    ref = golden_ref(name)
    g = _planning_scene(s)
    for tag, gmax in (("gvs_default", 20), ("gvs_n3", 3)):
        st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, global_vs_max=gmax)
        for v in range(s.n_views):
            assert g.global_view_selection(st, v) == ref["%s_%d" % (tag, v)].tolist(), (name, tag, v)


def test_matches_oracle_on_a_wide_tiled_scene():
    """The weak-scaling bench scene (tiled 4x4 camera blocks): many views, every selection saturates at globalVSMax."""
    from mve_b200 import dmrecon, synth
    from oracle import oracle_py as O
    cfg = dict(synth.CONFIGS["C2"])
    cfg.update(views=48, grid=(12, 4), blocks=3, features=6000, width=96, height=54, name="C2x3")
    s = synth.make_scene(cfg)
    g = _planning_scene(s)
    o = O.OracleScene(s)
    gs, os_ = dmrecon.Settings(scale=0), O.default_settings(scale=0)
    for v in (0, 7, 16, 23, 31, 47):
        got = g.global_view_selection(gs, v)
        assert got == o.global_view_selection(os_, v)
        assert len(got) == 20


def test_planning_context_refuses_compute():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    g = _planning_scene(s)
    st = dmrecon.Settings()
    for call in (lambda: g.set_view(0, s.images[0], s.flen[0], s.paspect[0], s.ppoint[0], s.rot[0], s.trans[0]),
                 lambda: g.reconstruct(st, [0]),
                 lambda: g.optimize_patches(st, 0, [1, 2, 3, 4, 5], np.zeros(1, dmrecon.PATCH_IN))):
        with pytest.raises(dmrecon.B200MVSError) as e:
            call()
        assert e.value.code == -2 and "no CPU fallback" in str(e.value)
    # argument validation still mirrors the reference's exceptions
    with pytest.raises(dmrecon.B200MVSError) as e:
        g.global_view_selection(st, 99)
    assert "Master view index out of bounds" in str(e.value)


BAD_PLANNING_INPUTS = {          # reference view (None: a view without a camera), settings, code, message
    "view_99": (99, {}, -1, "Master view index out of bounds"),
    "view_without_camera": (None, {}, -1, "Invalid master view"),
    "scale_9": (0, dict(scale=9), -1, "Invalid scale factor"),
    "filter_width_7": (0, dict(filter_width=7), -6, "filterWidth must be 5"),
    "nr_recon_neighbors_5": (0, dict(nr_recon_neighbors=5), -6, "nrReconNeighbors must be in 1..4"),
    "global_vs_max_33": (0, dict(global_vs_max=33), -6, "globalVSMax must be in 1..32"),
    "frontier_band_2": (0, dict(frontier_band=2.0), -1, "frontier_band must be in [0, 1]"),
}


@pytest.mark.parametrize("case", list(BAD_PLANNING_INPUTS))
def test_planning_entry_points_reject_the_same_inputs(case):
    """plan_views, global_view_selection, working_set and plan_batches check settings and reference views alike: each bad
    input fails all four with the same code and message.  plan_views goes first, so no earlier message can stand in for
    its own."""
    from mve_b200 import dmrecon
    ref, settings, code, message = BAD_PLANNING_INPUTS[case]
    s = golden_scene("T0")
    g = _planning_scene(s, n_views=s.n_views + 1)           # the last view has no camera
    ref = s.n_views if ref is None else ref
    st = dmrecon.Settings(**{"scale": s.scale, **settings})
    calls = {"plan_views": lambda: g.plan_views(st, [ref]),
             "global_view_selection": lambda: g.global_view_selection(st, ref),
             "working_set": lambda: g.working_set(st, [ref]),
             "plan_batches": lambda: g.plan_batches(st, [ref], 1 << 40)}
    got = {}
    for name, call in calls.items():
        with pytest.raises(dmrecon.B200MVSError) as e:
            call()
        got[name] = (e.value.code, str(e.value))
    assert len(set(got.values())) == 1, got
    assert got["plan_views"][0] == code and got["plan_views"][1].startswith("b200mvs error %d: %s" % (code, message)), got


def test_plan_views_runs_on_host_threads_without_a_gpu():
    """b200mvs_plan_views (global view selection + seed lists ahead of the reconstruct call) is pure host work: it runs in the
    planning context, also from several threads at once; bad views are reported."""
    import threading
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    g = _planning_scene(s)
    st = dmrecon.Settings(scale=s.scale)
    g.plan_views(st, list(range(s.n_views)))
    th = [threading.Thread(target=g.plan_views, args=(st, [v])) for v in range(4)]
    [t.start() for t in th]
    [t.join() for t in th]
    with pytest.raises(dmrecon.B200MVSError):
        g.plan_views(st, [99])
    with pytest.raises(dmrecon.B200MVSError):
        g.reconstruct(st, [0])            # planning context: no compute, no CPU fallback


def test_planned_selection_is_what_global_view_selection_returns(monkeypatch):
    """A prepared plan answers b200mvs_global_view_selection (the shim's leader asks for the selection of views its callers
    planned on their own threads); the answer is the reference's selection whether it is computed or looked up, with one
    planning thread (B200MVS_HOST_THREADS) or many, and a plan made under other settings is not used."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    ref = golden_ref("T2")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, global_vs_max=20)
    st3 = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, global_vs_max=3)
    for threads in ("1", "3"):
        monkeypatch.setenv("B200MVS_HOST_THREADS", threads)
        g = _planning_scene(s)
        g.plan_views(st, list(range(s.n_views)))
        for v in range(s.n_views):
            assert g.global_view_selection(st, v) == ref["gvs_default_%d" % v].tolist(), (threads, v)       # looked up
            assert g.global_view_selection(st3, v) == ref["gvs_n3_%d" % v].tolist(), (threads, v)           # other settings: computed


def test_planning_arithmetic_is_written_once():
    """The host planner calls the planning helpers of plan_device.cuh, the ones the device planner calls, and reads the
    features in the arrays both planners share: b200mvs.cu defines no copy of a helper, no feature record of its own and
    no second seed type."""
    src = open(os.path.join(ROOT, "mve_b200", "csrc", "b200mvs.cu")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    helpers = ("fadd", "fmul", "fdiv", "fsqrt", "ddiv", "ffloor", "fceil", "dot3", "world_to_cam", "mat3_mul",
               "point_in_frustum", "in_aabb", "unit_dir", "foot_print", "round_mve", "seen_in_box", "footprint_ratio",
               "seed_of")
    for name in helpers:
        assert not re.search(r"\b(float|double|bool|void|auto)\s+%s\s*[(=]" % name, src), name
    for gone in ("HostFeature", "SeedPoint"):
        assert not re.search(r"\b%s\b" % gone, src), gone
