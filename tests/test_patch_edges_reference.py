"""One PatchOptimization where its samples meet the level borders, the master border and the level switches, on the CPU.

The inputs are those of tests/golden/patch_edges_ref.npz, built by tests/patch_edges.py from the oracle's execution trace
and run through the unmodified reference (tests/golden/make_golden.py, group patch_edges).  This module shows that each
edge class occurs on them, with the margin rule, and that the reference does not answer all of them the same way; pins
the float64 restatement of the geometry; and runs the oracle and the product's device code (in the SIMT emulation of
tests/test_device_code_emulated.py) on them against the reference.  In the emulation the assert of PatchT::Sweep::stage
("the 2x2 quad lies in the level") runs on every constructed edge: the CPU check of the peeled samples and of `ok`.

Measured on the fixture (T0, T4, T5, T6): the oracle and the emulation in both modes flip no success and no local view id
of any class, and their depth rel p99 is <= 9e-7 on every scene."""
import numpy as np
import pytest

from oracle import oracle_py as O
from tests import camera_reference as CR
from tests import patch_edges as PE
from tests.test_device_code_emulated import _run, emu  # noqa: F401  (emu is a fixture)
from tests.util import GOLD, golden_scene, patch_compare

SCENES = ("T0", "T4", "T5", "T6")
# the classes each scene's geometry reaches (the measured counts are 24-2000; T4's one_out_tail is the smallest, 24).
# T0 is the control: every level width is a multiple of 4, so nothing sits next to row padding.  Its neighbours and those
# of T4 are displaced sideways: a depth change moves their samples along the rows, never onto the bottom border of T4.
COMMON = ("near_edge_in", "one_out_tail", "one_out_head", "one_out_mid", "master_border", "master_outside")
REQUIRED = {"T0": COMMON + ("bottom",),
            "T4": COMMON + ("padded_right", "level_switch"),
            "T5": COMMON + ("padded_right", "bottom", "level_switch"),
            "T6": COMMON + ("padded_right", "bottom", "level_switch", "level_clamped")}
MIN_CLASS = 20


def edge_fixture(name):
    """(scene, reference view, global selection, inputs, reference results, class masks) of one scene of the fixture."""
    import os
    d = np.load(os.path.join(GOLD, "patch_edges_ref.npz"))
    s = golden_scene(name)
    ref, gsel = int(d[name + "_patch_ref_view"]), d[name + "_patch_gvs"].tolist()
    pin, pout = d[name + "_patch_in"], d[name + "_patch_out"]
    return s, ref, gsel, pin, pout, PE.edge_classes(s, ref, s.scale, gsel, pin)


@pytest.fixture(scope="module")
def fixture():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = edge_fixture(name)
        return cache[name]
    return get


def class_flips(got, want, cls):
    """Per class: (patches, success flips, local-id flips among patches both succeed on)."""
    ok_g, ok_r = got["conf"] > 0, want["conf"] > 0
    ids = (got["local_ids"] != want["local_ids"]).any(-1) & ok_g & ok_r
    return {k: (int(m.sum()), int((m & (ok_g != ok_r)).sum()), int((m & ids).sum())) for k, m in cls.items()}


@pytest.mark.parametrize("name", SCENES)
def test_every_class_occurs(fixture, name):
    """At least MIN_CLASS patches of each class the scene's geometry reaches; the reference succeeds on a fair share of each
    (on at least 10 % of a class and at least 10 patches: the edge view fails the copies that are given it as a local
    view), fails on every master_outside patch; and the margin rule holds on every input that samples a view (a
    master_outside input fails before it samples one)."""
    s, ref, gsel, pin, pout, cls = fixture(name)
    assert 1500 <= len(pin) <= 3000
    assert cls["conditioned"][~cls["master_outside"]].all()
    ok = pout["conf"] > 0
    for k in REQUIRED[name]:
        assert cls[k].sum() >= MIN_CLASS, (k, int(cls[k].sum()))
        if k != "master_outside":
            assert ok[cls[k]].sum() >= 10 and ok[cls[k]].mean() >= 0.1, (k, ok[cls[k]].mean())
    assert not ok[cls["master_outside"]].any()
    # seeds and propagated inputs of every sample class
    for k in PE.SAMPLE_CLASSES:
        assert (cls[k] & (pin["n_local"] == 0)).sum() >= MIN_CLASS // 2 and (cls[k] & (pin["n_local"] == 4)).sum() >= MIN_CLASS // 2, k
    if name == "T0":
        assert not cls["padded_right"].any()


@pytest.mark.parametrize("name", SCENES)
def test_classes_hold_per_view(fixture, name):
    """The sample classes are about one view at its chosen level: on that view exactly one sample is outside (or none, and
    the closest is within NEAR), and every other view a patch samples keeps every sample MARGIN px from the border."""
    s, ref, gsel, pin, pout, cls = fixture(name)
    pv = PE.edge_classes(s, ref, s.scale, gsel, pin, per_view=True)
    use = PE.sampled_views(gsel, pin)
    for k in PE.SAMPLE_CLASSES:
        assert ((pv[k] & use).any(1) == cls[k]).all()
    assert (pv["conditioned"] | ~use)[~cls["master_outside"]].all()


@pytest.mark.parametrize("name", SCENES)
def test_restatement_pinned(fixture, name):
    """patch_points' centre is camera_reference.patch_centres (the oracle does not expose its sample positions).  The same
    expressions evaluated in float32 - points formed in world space, then transformed, the reference's own order - stay
    within 4 ulp of the depth of the float64 points, and their projections within 1.5e-4 px (measured: 2.7 ulp and
    8.3e-5 px, from the cancellation in R X + t).  So even the reference's float32 chain moves a sample by less than a
    sixth of the 1e-3 px margin; the device's chain is within 2 ulp of the reference's (DESIGN.md section 3)."""
    s, ref, gsel, pin, pout, cls = fixture(name)
    args = (pin["x"], pin["y"], pin["depth"], pin["dz_i"], pin["dz_j"])
    X64 = PE.patch_points(s, ref, s.scale, *args)
    assert np.allclose(X64[:, PE.NS // 2], CR.patch_centres(s, ref, s.scale, pin), rtol=1e-12, atol=1e-12)
    X32 = PE.patch_points(s, ref, s.scale, *args, dtype=np.float32)
    assert X32.dtype == np.float32
    assert (np.abs(X32 - X64) <= 4 * np.spacing(pin["depth"])[:, None, None]).all()
    for v in gsel:
        st = PE.view_state(s, ref, s.scale, v, *(a.astype(np.float64) for a in args))
        q32 = PE.project(s, v, st["level"], X32, np.float32)
        assert q32.dtype == np.float32
        err = np.abs(q32 - PE.project(s, v, st["level"], X64))[st["ok"]]
        assert err.max() <= 1.5e-4, (v, err.max())


@pytest.mark.parametrize("name", SCENES)
def test_oracle_vs_reference_on_edges(fixture, name):
    """The CPU restatement (oracle/mvs_oracle.cc) on the edge inputs, under the bounds of
    test_oracle_vs_reference.py::test_patch_optimization_vs_reference, over the scene and per class."""
    s, ref, gsel, pin, pout, cls = fixture(name)
    st = O.default_settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    got = O.OracleScene(s).optimize_patches(st, ref, gsel, pin)
    c = patch_compare(got, pout)
    n = c["n"]
    assert c["ok_mismatch"] <= max(1, 0.002 * n) and c["ids_mismatch"] <= max(1, 0.002 * n)
    assert np.percentile(c["rel"], 99) < 2e-5
    assert np.percentile(c["rel"], 99.9) < 1e-3
    assert np.percentile(c["conf_abs"], 99) < 1e-4
    assert np.percentile(c["dz_abs"], 99) < 1e-4
    for k, (m, fo, fi) in class_flips(got, pout, cls).items():
        assert fo <= max(1, 0.002 * m) and fi <= max(1, 0.002 * m), (k, m, fo, fi)
    assert not (got["conf"][cls["master_outside"]] > 0).any()
    assert ((got["conf"] > 0) == (pout["conf"] > 0))[cls["master_border"]].all()


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", SCENES)
def test_device_code_emulated_on_edges(emu, fixture, name, mode):   # noqa: F811
    """The product's device code (mode 1: PatchW, mode 2: PatchT) in the SIMT emulation on the edge inputs, under the bounds
    of test_device_code_emulated.py::test_kernel_body_vs_reference_golden, and per class.  PatchT runs every input; PatchW,
    whose emulation runs 32 host threads per patch, every third."""
    s, ref, gsel, pin, pout, cls = fixture(name)
    pick = np.arange(len(pin)) if mode == 2 else np.arange(0, len(pin), 3)
    st = O.default_settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    got, _ = _run(emu, s, O.OracleScene(s), ref, gsel, st, pin[pick], mode)
    c = patch_compare(got, pout[pick])
    assert c["ok_mismatch"] <= 1 and c["ids_mismatch"] <= 1, (c["ok_mismatch"], c["ids_mismatch"])
    assert np.percentile(c["rel"], 99) < 5e-5
    for k, (m, fo, fi) in class_flips(got, pout[pick], {k: v[pick] for k, v in cls.items()}).items():
        assert fo <= max(1, 0.002 * m) and fi <= max(1, 0.002 * m), (k, m, fo, fi)
    assert not (got["conf"][cls["master_outside"][pick]] > 0).any()
    assert ((got["conf"] > 0) == (pout[pick]["conf"] > 0))[cls["master_border"][pick]].all()
