"""General pinhole cameras on the CPU.  T5 (portrait 101x135, non-square pixels, off-centre principal points, rolls, one
wide and two zoomed views, scale 0) and T6 (179x180 views whose aspect branch flips between level 0 and 1, 118x58 and
58x118 crops with long focal lengths, scale 1) reach code that the other scenes, all landscape with one camera model,
never run: the portrait branch of the calibration, ax != ay, pyramid levels >= 2, the level clamp and the resolution
terms of both view selections.

The float64 restatement of tests/camera_reference.py is pinned against the oracle's pyramid calibration, then used to
show that each of those cases occurs on the golden patch inputs - so the parity tests on T5 / T6 (test_oracle_vs_reference,
test_host_view_selection, test_device_code_emulated, test_gpu_parity) check them - and to pick the patches on which the
product's device code runs in the SIMT emulation."""
import numpy as np
import pytest

from oracle import oracle_py as O
from tests import camera_reference as CR
from tests.test_device_code_emulated import _run, emu  # noqa: F401  (emu is a fixture)
from tests.util import golden_ref, golden_scene, patch_compare


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T3", "T4", "T5", "T6"])
def test_level_calibration_matches_oracle(name):
    """Per view and level: the size and the aspect branch are those of the oracle, the float32 evaluation of the same
    expressions gives the oracle's K and K^-1 bit for bit, and they are within 2 ulp of float32 of the float64 values.
    The entries are up to three float32 roundings deep (ax = flen * h / paspect, then 1 / ax) and the principal point
    is corrected in float32 at every odd level: the largest distance measured on T0-T6 is 1.52 ulp (K^-1 [0, 2])."""
    s = golden_scene(name)
    osc = O.OracleScene(s)
    for v in range(s.n_views):
        lv64, lv32 = CR.view_levels(s, v), CR.view_levels(s, v, np.float32)
        assert osc.num_levels(v) == len(lv64) == len(lv32), v
        for l, (a, b) in enumerate(zip(lv64, lv32)):
            w, h, K, Ki, portrait = a
            assert (w, h, portrait) == (b[0], b[1], b[4]), (v, l)
            assert osc.level(v, l).shape[:2] == (h, w), (v, l)
            k, ki = osc.level_calib(v, l)
            assert (k == b[2].reshape(-1)).all() and (ki == b[3].reshape(-1)).all(), (v, l)
            for got, want in ((k, K), (ki, Ki)):
                want = want.reshape(-1)
                assert (np.abs(got - want) <= 2 * np.spacing(np.abs(want).astype(np.float32))).all(), (v, l, got, want)


def test_aspect_branches():
    """T5 is portrait at every level, T6's 179x180 views flip from portrait at level 0 to landscape at level 1, its crops
    are of both orientations, and every other scene is landscape throughout."""
    def branches(name):
        s = golden_scene(name)
        return [[lv[4] for lv in CR.view_levels(s, v)] for v in range(s.n_views)]
    assert all(all(b) for b in branches("T5"))
    t6 = branches("T6")
    wide = [b for v, b in enumerate(t6) if golden_scene("T6").size(v) == (179, 180)]
    assert len(wide) == 5 and all(b[0] and not any(b[1:]) for b in wide)
    assert {tuple(b) for b in t6} >= {(True, True), (False, False)}
    for name in ("T0", "T1", "T2", "T3", "T4"):
        assert not any(any(b) for b in branches(name)), name


# floors on the golden patch inputs (the measured counts are 2-4x higher; see camera_cases for the definitions)
CASE_FLOORS = {"T5": dict(level_ge2=40, penalised=1000, gvs_ratio_gt2=1000),
               "T6": dict(clamped=50, requested_ge3=10, gvs_ratio_gt2=1000)}


@pytest.mark.parametrize("name", ["T5", "T6"])
def test_camera_cases_occur_on_golden_patches(name):
    s = golden_scene(name)
    ref = golden_ref(name)
    cases = CR.camera_cases(s, int(ref["patch_ref_view"]), s.scale, ref["patch_gvs"].tolist(), ref["patch_in"],
                            ref["patch_out"])
    counts = {k: int(m.sum()) for k, m in cases.items()}
    for k, floor in CASE_FLOORS[name].items():
        assert counts[k] >= floor, (k, counts)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name,view,case", [("T5", 1, "level_ge2"), ("T6", 2, "clamped")])
def test_kernel_body_on_zoomed_and_clamped_levels(emu, name, view, case, mode):  # noqa: F811
    """The device code in the SIMT emulation on the oracle's trace, on every patch that samples a view at level >= 2 (T5)
    or at a clamped level (T6) plus a stride of the rest, at the tolerances of test_kernel_body_on_oracle_trace."""
    s = golden_scene(name)
    osc = O.OracleScene(s)
    st = O.default_settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    gsel = osc.global_view_selection(st, view)
    r = osc.reconstruct(st, view, trace_cap=100000)
    tin, tout = r["trace_in"], r["trace_out"]
    hit = np.nonzero(CR.camera_cases(s, view, s.scale, gsel, tin, tout)[case])[0]
    assert len(hit) >= 40, len(hit)
    pick = np.unique(np.concatenate([hit, np.arange(0, len(tin), max(1, len(tin) // 100))]))
    got, raw = _run(emu, s, osc, view, gsel, st, tin[pick], mode)
    c = patch_compare(got, tout[pick])
    n = c["n"]
    assert c["ok_mismatch"] <= max(1, 0.01 * n), (c["ok_mismatch"], n)
    assert c["ids_mismatch"] <= max(1, 0.01 * n), (c["ids_mismatch"], n)
    assert (got["iterations"] != tout[pick]["iterations"])[c["both"]].mean() < 0.02
    assert np.percentile(c["rel"], 99) < 5e-5
    assert np.percentile(c["conf_abs"], 99) < 2e-4
    assert np.percentile(c["nrm_abs"], 99) < 1e-3
    # the patches of the case itself succeed as often in the emulation as in the oracle
    both_hit = np.isin(pick, hit)
    assert ((got["conf"] > 0) != (tout[pick]["conf"] > 0))[both_hit].sum() <= max(1, 0.01 * both_hit.sum())
