"""General pinhole cameras on the GPU (-m gpu), every call through the C ABI.  The parity tests of tests/test_gpu_parity.py
(pyramid bytes, global selection, patches in both modes against the reference and the oracle, maps under the same schedule
and against the reference CLI) and the drop-in CLI test run on T5 and T6 as well; tests/test_cameras.py shows which camera
cases those fixtures reach.  This file holds what only scenes with mixed cameras and sizes can check."""
import numpy as np
import pytest

from tests import camera_reference as CR
from tests.test_gpu_properties import _gt_depth
from tests.util import golden_scene

pytestmark = pytest.mark.gpu

MAP_KEYS = ("depth", "conf", "dz", "normal", "view_ids")


@pytest.mark.parametrize("name,views", [("T5", (1, 6)), ("T6", (2, 3))])
def test_batch_of_mixed_cameras_equals_single_views(name, views):
    """All views in one batch - different focal lengths, pixel aspects, principal points and (T6) image sizes, so the
    batch's maps have different shapes - give the same maps as one call per view, bitwise."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    g = dmrecon.Scene.from_synth(s)
    gs = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    batch, _ = g.reconstruct(gs, list(range(s.n_views)))
    assert [m["depth"].shape[::-1] for m in batch] == [CR.view_levels(s, v)[s.scale][:2] for v in range(s.n_views)]
    for v in views:
        single, _ = g.reconstruct(gs, [v])
        for k in MAP_KEYS:
            assert (batch[v][k] == single[0][k]).all(), (v, k)
    assert (batch[views[0]]["depth"] > 0).mean() > 0.4


def test_lazy_images_of_mixed_sizes():
    """from_synth(lazy=True) registers each view at its own size and loads the images on demand: the maps equal those of
    the uploaded scene, bitwise."""
    from mve_b200 import dmrecon
    s = golden_scene("T6")
    gs = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    eager, _ = dmrecon.Scene.from_synth(s).reconstruct(gs, [2, 3, 6])
    g = dmrecon.Scene.from_synth(s, lazy=True)
    assert [g.num_levels(v) for v in range(s.n_views)] == [len(CR.view_levels(s, v)) for v in range(s.n_views)]
    lazy, _ = g.reconstruct(gs, [2, 3, 6])
    for a, b in zip(eager, lazy):
        for k in MAP_KEYS:
            assert (a[k] == b[k]).all(), k


@pytest.mark.parametrize("view", [1, 4])
def test_ground_truth_accuracy_general_cameras(view):
    """T5 at scale 0 against the analytic surface, through the same calibration the scene was rendered with: the bounds of
    the full-size views in test_gpu_properties (median 1e-3, p95 1e-2)."""
    from mve_b200 import dmrecon, synth
    s = synth.make_scene("T5")
    g = dmrecon.Scene.from_synth(s)
    maps, _ = g.reconstruct(dmrecon.Settings(scale=s.scale), [view])
    m = maps[0]
    filled = m["conf"] > 0
    assert filled.mean() > 0.4
    gt = _gt_depth(s, view, s.scale)
    err = np.abs(m["depth"] - gt)[filled] / gt[filled]
    assert np.median(err) < 1e-3 and np.percentile(err, 95) < 1e-2, (np.median(err), np.percentile(err, 95))
