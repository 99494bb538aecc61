"""The restatement of scene2pset's scene-level filters (tests/pset_reference.py) against the unmodified reference app
(oracle/_ref/scene2pset, built by oracle/scene2pset.mk), without a GPU.  The app runs on one thread (OMP_NUM_THREADS=1), so
its views come in the scene's order.  Depth maps: the reference dmrecon's own maps of the golden scenes T0, T5 and T6, plus
hand-made maps.  Every decision is checked on the reference's own vertices: the bounding box (faces placed exactly on vertex
coordinates), the silhouette masks (zero regions through the points; masks larger, smaller and of the map's size, views
without a mask, a 3-channel mask) with num_filtered, the fill fraction (including a map of more than 2^24 pixels) and the
correspondence CSVs byte for byte."""
import os
import tempfile

import numpy as np
import pytest

from tests import dm_reference as R
from tests import pset_reference as S

pytestmark = pytest.mark.skipif(not os.path.exists(S.REF_APP), reason="oracle/_ref/scene2pset not built (needs the reference sources at build time)")
F32 = np.float32
MASKS = {"T0": {0: "same", 1: "double", 3: "odd", 4: "rgb"}, "T5": {1: "same", 2: "odd", 5: "double"},
         "T6": {2: "same", 3: "double", 6: "rgb"}}
HAND = {"T0": (1,), "T5": (4,), "T6": (5,)}


def _scene(tmp, name, **kw):
    kw.setdefault("hand_views", HAND[name])
    kw.setdefault("mask_kinds", MASKS[name])
    return S.build_scene(tmp, name, **kw)


def _dm_arg(sc):
    return ["-d", "depth-L%d" % sc["scene"].scale] + (["-i", "undist-L%d" % sc["scene"].scale] if sc["scene"].scale else [])


@pytest.mark.parametrize("name", S.SCENES)
def test_mask_and_box_decisions_match_the_reference(name):
    with tempfile.TemporaryDirectory() as tmp:
        sc = _scene(tmp, name)
        s = sc["scene"]
        out = os.path.join(tmp, "all.ply")
        S.run(S.REF_APP, _dm_arg(sc), tmp, out)
        _, allv = S.read_ply(out)
        V = S.xyz(allv)
        assert len(V) > 1000
        # -m: decisions of the restatement on the reference's own vertices
        masks = [(m, S.camera_of(s, v)) for v, m in sorted(sc["masks"].items()) if m.ndim == 2]
        stdout = S.run(S.REF_APP, _dm_arg(sc) + ["-m", "mask"], tmp, os.path.join(tmp, "m.ply"))
        _, mv = S.read_ply(os.path.join(tmp, "m.ply"))
        dele = S.mask_deleted(V, masks)
        assert 0.05 * len(V) < dele.sum() < 0.95 * len(V), dele.sum()
        assert S.num_filtered(stdout) == int(dele.sum())
        np.testing.assert_array_equal(S.xyz(mv), V[~dele])
        assert stdout.count("Expected 1-channel mask") == sum(m.ndim == 3 for m in sc["masks"].values())
        assert stdout.count("Mask not found") == s.n_views - len(sc["masks"])
        # -b with faces exactly on vertex coordinates
        lo = np.array([np.percentile(V[:, k], 20, method="nearest") for k in range(3)], F32)
        hi = np.array([np.percentile(V[:, k], 85, method="nearest") for k in range(3)], F32)
        box = ",".join("%.9g" % x for x in np.concatenate([lo, hi]))
        S.run(S.REF_APP, _dm_arg(sc) + ["--bounding-box=" + box], tmp, os.path.join(tmp, "b.ply"))
        _, bv = S.read_ply(os.path.join(tmp, "b.ply"))
        keep = S.aabb_keep(V, lo, hi)
        on_face = ((V == lo) | (V == hi)).any(-1)
        assert (keep & on_face).sum() > 0
        np.testing.assert_array_equal(S.xyz(bv), V[keep])


@pytest.mark.parametrize("name", S.SCENES)
def test_fill_fraction_and_views_match_the_reference(name):
    with tempfile.TemporaryDirectory() as tmp:
        sc = _scene(tmp, name, mask_kinds={})
        maps = sc["maps"]
        fr = {v: S.fill_fraction(d) for v, d in maps.items()}
        # a threshold equal to one view's fraction keeps it (fraction < min skips); one ulp above skips it
        v0 = sorted(maps)[0]
        for f, want_skip in ((fr[v0], False), (np.nextafter(fr[v0], F32(1)), True)):
            stdout = S.run(S.REF_APP, _dm_arg(sc) + ["-f", "%.9g" % f], tmp, os.path.join(tmp, "f.ply"))
            skipped = {int(n) for n, _ in S.skipped_views(stdout)}
            assert skipped == {v for v in maps if fr[v] < f}, (skipped, fr, f)
            assert (v0 in skipped) == want_skip
            for n, pct in S.skipped_views(stdout):
                assert pct == "%.2f" % (fr[int(n)] * F32(100.0))
        # -v picks views; views without a map are passed over
        stdout = S.run(S.REF_APP, _dm_arg(sc) + ["-v", str(v0)], tmp, os.path.join(tmp, "v.ply"))
        assert [int(x) for x in S.processed_views(stdout)] == [v0]


def big_fill_map():
    h, w = 4101, 8203
    dm = np.zeros((h, w), F32)
    dm[0::2] = 1.0
    dm[1::2, :50] = 1.0
    dm[1, 50:57] = 1.0
    return dm


def test_fill_fraction_above_2_to_the_24_pixels():
    """A synthetic 8203 x 4101 map (33.6 M px) whose 16.9 M filled pixels exceed 2^24: the reference's float lane sums
    round and its last increments are lost, so its fraction is not count / n.  Odd rows are empty except for their first
    50 pixels, so no triangle forms and the run stays short.  Each lane holds about 2.1 M here: the saturation of one lane
    at 2^24 needs more than 134 M filled pixels and is not exercised."""
    dm = big_fill_map()
    f = S.fill_fraction(dm)
    exact = F32(F32(int((dm > 0).sum())) / F32(dm.size))
    assert int((dm > 0).sum()) > 1 << 24 and f != exact, (f, exact)
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, "T0", extra_maps={2: dm})
        for thr, skip in ((f, False), (np.nextafter(f, F32(1)), True)):
            stdout = S.run(S.REF_APP, ["-v", "2", "-i", "no-such-image", "-f", "%.9g" % thr], tmp, os.path.join(tmp, "big.ply"))
            assert (len(S.skipped_views(stdout)) == 1) == skip, stdout


def test_correspondence_csvs_equal_the_restatement():
    with tempfile.TemporaryDirectory() as tmp:
        sc = _scene(tmp, "T0", mask_kinds={})
        s = sc["scene"]
        out = os.path.join(tmp, "c.ply")
        S.run(S.REF_APP, ["-C"], tmp, out)
        per_view = []
        for v in sorted(sc["maps"]):
            ip = np.linalg.inv(S.calibration(S.camera_of(s, v), *sc["maps"][v].shape[::-1]).reshape(3, 3).astype(np.float64))
            per_view.append((v, R.triangulate(sc["maps"][v], ip.astype(F32), 5.0)["vertex_ids"]))
        data, meta = S.correspondence_csv(per_view)
        assert open(out + "_correspondence-metadata.csv").read() == meta
        assert open(out + "_correspondence-data.csv").read() == data
