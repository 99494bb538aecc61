"""The drop-in scene2pset_b200 (-m gpu) against the unmodified reference app oracle/_ref/scene2pset run on one thread
(OMP_NUM_THREADS=1, so its views come in the scene's order), on the same scene directories as
tests/test_scene_pointset_reference.py: the reference dmrecon's maps of T0, T5 and T6 plus hand-made maps, with masks.

PLY headers identical, point counts and order exact; world-frame vertices within 2e-6 of the largest coordinate (the
reference contracts its float expressions), normals p99.9 within 1e-4 (device acosf), confidences exact, scale values within 3e-5
relative, colours exact (DESIGN.md §5).  Every box, mask and fill decision on the device's own vertices is exactly what
tests/pset_reference.py decides; against the reference's vertices a decision may differ only for points within the vertex
tolerance of a box face or mask-pixel edge, and those are counted and printed.  The Python scene_pointset equals the CLI,
and the handle's peak device bytes do not grow with the number of views."""
import os
import tempfile

import numpy as np
import pytest

from tests import pset_reference as S
from tests.test_scene_pointset_reference import HAND, MASKS, big_fill_map

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (os.path.exists(S.CLI) and os.path.exists(S.REF_APP)),
                                                  reason="oracle/_ref/scene2pset or shim/scene2pset_b200 not built")]
F32 = np.float32


def _dm_args(s):
    return ["-d", "depth-L%d" % s.scale] + (["-i", "undist-L%d" % s.scale] if s.scale else [])


def compare_ply(a_path, b_path):
    """a = drop-in, b = reference."""
    ha, a = S.read_ply(a_path)
    hb, b = S.read_ply(b_path)
    assert ha == hb
    assert len(a) == len(b)
    if not len(a):
        return a, b
    va, vb = S.xyz(a), S.xyz(b)
    vmax = float(np.abs(vb).max())
    # world-frame vertices: the reference contracts mesh_transform, the device rounds each product (measured 1.5e-6 on
    # T6); tests/test_gpu_depthmap_ops.py states the same 2e-6 bound for cam_to_world
    assert np.abs(va - vb).max() <= 2e-6 * vmax, np.abs(va - vb).max() / vmax
    names = a.dtype.names
    if "nx" in names:
        na = np.stack([a["nx"], a["ny"], a["nz"]], -1)
        nb = np.stack([b["nx"], b["ny"], b["nz"]], -1)
        dn = np.abs(na - nb).max(-1)
        scale = np.maximum(1.0, np.abs(nb).max(-1))       # -p: normals scaled by confidences <= 1
        assert np.percentile(dn / scale, 99.9) <= 1e-4 and dn.max() <= 2e-3
    if "confidence" in names:
        np.testing.assert_array_equal(a["confidence"], b["confidence"])
    if "value" in names:
        smax = max(float(np.abs(b["value"]).max()), 1e-30)
        assert np.abs(a["value"] - b["value"]).max() <= 3e-5 * smax
    for c in ("red", "green", "blue"):
        if c in names:
            np.testing.assert_array_equal(a[c], b[c])
    return a, b


def _both(tmp, args, out_name, threads=1):
    a, b = os.path.join(tmp, "gpu_" + out_name), os.path.join(tmp, "ref_" + out_name)
    oa = S.run(S.CLI, args, tmp, a)
    ob = S.run(S.REF_APP, args, tmp, b, threads=threads)
    return a, b, oa, ob


CASES = [("plain", []), ("nsc", ["-n", "-c", "-s"]), ("poisson", ["-p"]), ("scale", ["-n", "-s", "-S", "1.75"]),
         ("views", ["-n", "-v", "VIEWS"])]


@pytest.mark.parametrize("name", S.SCENES)
@pytest.mark.parametrize("case,extra", CASES, ids=[c for c, _ in CASES])
def test_cli_matches_reference(name, case, extra):
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, name, hand_views=HAND[name], mask_kinds=MASKS[name])
        s = sc["scene"]
        extra = [",".join(str(v) for v in sorted(sc["maps"])[::-1][:1] + [0, 5]) if x == "VIEWS" else x for x in extra]
        a, b, oa, ob = _both(tmp, _dm_args(s) + extra, "p.ply")
        assert S.processed_views(oa) == S.processed_views(ob)
        compare_ply(a, b)


@pytest.mark.parametrize("name", S.SCENES)
def test_cli_fssr_npts_and_missing_colour(name):
    with tempfile.TemporaryDirectory() as tmp:
        # -F<s> takes depth-L<s> and undistorted / undist-L<s>; the scene stores undist-L<s> as MVEI (see pset_reference)
        sc = S.build_scene(tmp, name, hand_views=HAND[name], mask_kinds={}, drop_color=(HAND[name][0],))
        s = sc["scene"]
        a, b, oa, ob = _both(tmp, ["-F%d" % s.scale], "f.ply")
        assert "(with colors)" in oa and oa.count("(with colors)") == ob.count("(with colors)")
        ha, pa = S.read_ply(a)
        assert "red" not in pa.dtype.names          # one view without colours: the colour list is short, none are written
        compare_ply(a, b)
        # .npts: normals on, scale and confidence off; written by save_mesh
        a, b, _, _ = _both(tmp, _dm_args(s), "p.npts")
        assert open(a, "rb").read().count(b"\n") == open(b, "rb").read().count(b"\n")
        ta = np.loadtxt(a, ndmin=2)
        tb = np.loadtxt(b, ndmin=2)
        assert ta.shape == tb.shape
        assert np.abs(ta[:, :3] - tb[:, :3]).max() <= 1e-5 * np.abs(tb[:, :3]).max()
        # -m with a view that has no colour image: the short colour list is cleaned like delete_vertices does
        sc2 = S.build_scene(tmp, name, hand_views=HAND[name], mask_kinds=MASKS[name], drop_color=(HAND[name][0],))
        a, b, oa, ob = _both(tmp, _dm_args(s) + ["-m", "mask"], "mc.ply")
        ha, pa = S.read_ply(a)
        hb, pb = S.read_ply(b)
        assert ha == hb


def _decisions(tmp, s, sc, args_all, args_f, restate, near):
    """Runs both apps without and with a filter; the device's filtered set must be exactly what `restate` decides on the
    device's own vertices; against the reference the kept sets may differ only at `near` points."""
    ga, ra, _, _ = _both(tmp, args_all, "all.ply")
    gf, rf, og, orf = _both(tmp, args_f, "filt.ply")
    Vg = S.xyz(S.read_ply(ga)[1])
    Vr = S.xyz(S.read_ply(ra)[1])
    keep_g = restate(Vg)
    np.testing.assert_array_equal(S.xyz(S.read_ply(gf)[1]), Vg[keep_g])
    keep_r = restate(Vr)
    np.testing.assert_array_equal(S.xyz(S.read_ply(rf)[1]), Vr[keep_r])
    differ = keep_g != keep_r
    print("decisions that differ between device and reference vertices: %d of %d (all near an edge)" % (differ.sum(), len(Vg)))
    assert near(Vr)[differ].all()
    return og, orf, keep_g


@pytest.mark.parametrize("name", S.SCENES)
def test_box_and_mask_decisions(name):
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, name, hand_views=HAND[name], mask_kinds=MASKS[name])
        s = sc["scene"]
        base = _dm_args(s)
        Vr = S.xyz(S.read_ply(_both(tmp, base, "probe.ply")[1])[1])
        lo = np.array([np.percentile(Vr[:, k], 20, method="nearest") for k in range(3)], F32)
        hi = np.array([np.percentile(Vr[:, k], 85, method="nearest") for k in range(3)], F32)
        box = ",".join("%.9g" % x for x in np.concatenate([lo, hi]))
        tol = 1e-6 * float(np.abs(Vr).max())
        _decisions(tmp, s, sc, base, base + ["--bounding-box=" + box], lambda V: S.aabb_keep(V, lo, hi),
                   lambda V: (np.minimum(np.abs(V - lo), np.abs(V - hi)) <= tol).any(-1))
        masks = [(m, S.camera_of(s, v)) for v, m in sorted(sc["masks"].items()) if m.ndim == 2]
        og, orf, keep = _decisions(tmp, s, sc, base, base + ["-m", "mask"], lambda V: ~S.mask_deleted(V, masks),
                                   lambda V: S.edge_distance(V, masks) <= 1e-3)
        assert S.num_filtered(og) == int((~keep).sum())
        assert og.count("Expected 1-channel mask") == orf.count("Expected 1-channel mask")
        assert og.count("Mask not found") == orf.count("Mask not found")


def test_fill_fraction_and_correspondence():
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, "T0", hand_views=HAND["T0"], mask_kinds={}, extra_maps={2: big_fill_map()})
        fr = {v: S.fill_fraction(d) for v, d in sc["maps"].items()}
        for v, f in fr.items():
            for thr, skip in ((f, False), (np.nextafter(f, F32(1)), True)):
                og = S.run(S.CLI, ["-v", str(v), "-i", "no-such-image", "-f", "%.9g" % thr], tmp, os.path.join(tmp, "f.ply"))
                sk = S.skipped_views(og)
                assert (len(sk) == 1) == skip, og
                if skip:
                    assert sk[0][1] == "%.2f" % (f * F32(100.0))
        # -C: both CSVs byte for byte (views 0, 1 and 3 of T0)
        a, b, _, _ = _both(tmp, ["-C", "-v", "0,1,3"], "c.ply")
        for suffix in ("_correspondence-data.csv", "_correspondence-metadata.csv"):
            assert open(a + suffix, "rb").read() == open(b + suffix, "rb").read()
        compare_ply(a, b)


def test_python_scene_pointset_equals_cli_and_memory_is_bounded():
    from mve_b200 import depthmap as D
    from mve_b200 import synth
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, "T0", hand_views=HAND["T0"], mask_kinds=MASKS["T0"])
        s = sc["scene"]
        out = os.path.join(tmp, "cli.ply")
        S.run(S.CLI, ["-n", "-c", "-s", "-m", "mask"], tmp, out)
        _, cli = S.read_ply(out)
        views = [dict(id=v, depth=sc["maps"][v], camera=S.camera_of(s, v),
                      color=synth.read_mvei(os.path.join(tmp, "views", "view_%04d.mve" % v, "undistorted.mvei")))
                 for v in sorted(sc["maps"])]
        masks = [dict(mask=m, camera=S.camera_of(s, v)) for v, m in sorted(sc["masks"].items()) if m.ndim == 2]
        r = D.scene_pointset(views, dict(with_normals=True, with_conf=True, with_scale=True), masks=masks)
        np.testing.assert_array_equal(r["vertices"], S.xyz(cli))
        np.testing.assert_array_equal(r["normals"], np.stack([cli["nx"], cli["ny"], cli["nz"]], -1))
        np.testing.assert_array_equal(r["confidences"], cli["confidence"])
        np.testing.assert_array_equal(r["values"], cli["value"])
        assert r["num_filtered"] > 0 and all(v["added"] for v in r["views"])
        # the handle's device bytes do not grow with the number of views: 4 and 32 views of one size
        v0 = views[0]
        peaks = [D.scene_pointset([dict(v0, id=i) for i in range(k)], dict(with_normals=True, with_conf=True, with_scale=True),
                                  masks=masks)["info"]["peak_device_bytes"] for k in (4, 32)]
        assert peaks[0] == peaks[1] and peaks[0] > 0, peaks


def test_short_colour_list_under_masks():
    """A view without a colour image leaves the colour list shorter than the point list.  mve::TriangleMesh::delete_vertices
    then leaves that list as it is (it cleans a list only when it has one entry per point), and save_ply_mesh writes colours
    only when the counts are equal.  Here the colourless view is the last one and its all-zero mask deletes every point of
    it and some points of the other views: the colour list keeps its length, is longer than the point list, and neither
    app writes colours.  The Python scene_pointset returns the colour list untouched."""
    from mve_b200 import depthmap as D
    from mve_b200 import synth
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.build_scene(tmp, "T0", hand_views=HAND["T0"], mask_kinds={0: "same", 3: "zero"}, drop_color=(3,))
        s = sc["scene"]
        assert max(sc["maps"]) == 3
        a, b, oa, ob = _both(tmp, ["-m", "mask"], "m.ply")
        ha, pa = S.read_ply(a)
        compare_ply(a, b)
        assert "red" not in pa.dtype.names
        views = [dict(id=v, depth=sc["maps"][v], camera=S.camera_of(s, v),
                      color=None if v == 3 else synth.read_mvei(os.path.join(tmp, "views", "view_%04d.mve" % v, "undistorted.mvei")))
                 for v in sorted(sc["maps"])]
        masks = [dict(mask=m, camera=S.camera_of(s, v)) for v, m in sorted(sc["masks"].items())]
        full = D.scene_pointset(views)
        r = D.scene_pointset(views, masks=masks)
        n3 = full["views"][-1]["n_points"]
        assert r["num_filtered"] > n3 > 0                  # all of view 3 and some points of views 0 and 1
        assert len(r["vertices"]) == len(full["vertices"]) - r["num_filtered"] == len(pa)
        np.testing.assert_array_equal(r["colors"], full["colors"])
        assert len(r["colors"]) == len(full["vertices"]) - n3 > len(r["vertices"])
