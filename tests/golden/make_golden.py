"""Mints the committed golden fixtures from the REFERENCE ITSELF (oracle/_ref, built by oracle/Makefile from
/root/reference).  Run in the build container only:   python tests/golden/make_golden.py

Outputs (all under tests/golden/):
  srgb2lin.npy            the 256-entry table of libs/dmrecon/mvs_tools.cc:30-95, parsed from the source
  <S>_scene.npz           the synthetic scene (images, cameras, features) so that fixtures are self-contained
  <S>_ref.npz             reference results for that scene:
      gvs_default / gvs_n3     "Global View Selection:" line of the reference per view (default and -n 3)
      patch_in / patch_out     inputs and mvs::PatchOptimization results through oracle/_ref/ref_harness
      depth_v / conf_v / dz_v  maps written by oracle/_ref/dmrecon for views v (apps/dmrecon CLI, unmodified)
      undist_v                 pyramid level `scale` written by the reference (scale != 0 only)
  C2_view5_ref.npz, C5r_view3_ref.npz   reference CLI maps at BASELINE size, reduced by sampled_map()
  depthmap_ops_ref.npz    libs/mve/depthmap.cc results for tests/test_gpu_depthmap_ops.py
  depthmap_edges_ref.npz  the same at the decision boundaries and edge shapes of tests/test_gpu_depthmap_edges.py
  T0s77_ref.npz           mvs::PatchOptimization results on a scene generated with seed 77
  T5_*, T6_*              like <S>_* above for the scenes with general cameras (group `cameras`); their patch slices
                          also keep the patches that sample the zoomed views (T5) or the crops (T6)
  T0_ply_ref.npz          .xf files and PLY headers written by the reference CLI with -p
  patch_edges_ref.npz     mvs::PatchOptimization results on the inputs of tests/patch_edges.py that sit on the level
                          borders, the master border and the level switches: <S>_patch_in / _patch_out / _patch_gvs /
                          _patch_ref_view for T0, T4, T5, T6 (tests/test_patch_edges_reference.py, test_gpu_patch_edges.py)

`python tests/golden/make_golden.py [tiny] [cameras] [baseline_size] [depthmap_ops] [depthmap_edges] [fresh_scene_patches] [ply] [patch_edges]`
mints only the named groups (default: all).
"""
import hashlib
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from mve_b200 import synth            # noqa: E402
from oracle import oracle_py as O     # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.path.join(ROOT, "oracle", "_ref")


def parse_lut():
    src = open("/root/reference/libs/dmrecon/mvs_tools.cc").read()
    a = src.index("srgb2lin[256] = {")
    body = src[a:src.index("};", a)]
    vals = [np.float32(x.rstrip("f")) for x in re.findall(r"[0-9.]+(?:e-?[0-9]+)?f", body)]
    assert len(vals) == 256
    return np.asarray(vals, np.float32)


def run_cli(scene_dir, scale, nrn, extra=()):
    cmd = [os.path.join(REF, "dmrecon"), "-s%d" % scale, "--local-neighbors=%d" % nrn, "--keep-conf", "--keep-dz",
           "--progress=silent", "--force"] + list(extra) + [scene_dir]
    return subprocess.run(cmd, capture_output=True, text=True, check=True, env=dict(os.environ, OMP_NUM_THREADS="1")).stdout


def gvs_lines(scene_dir, scale, nrn, n_views, extra=()):
    out = {}
    for v in range(n_views):
        txt = subprocess.run([os.path.join(REF, "dmrecon"), "-s%d" % scale, "--local-neighbors=%d" % nrn,
                              "--progress=simple", "--force", "-l%d" % v] + list(extra) + [scene_dir],
                             capture_output=True, text=True).stdout
        m = re.search(r"Global View Selection:([ 0-9]*)", txt)
        out[v] = np.asarray([int(x) for x in m.group(1).split()], np.int32) if m else np.zeros(0, np.int32)
    return out


def mint_gvs_only(name):
    """Only the printed global view selections (many-candidate scene)."""
    s = synth.make_scene(name)
    synth.save_scene_npz(s, os.path.join(GOLD, "%s_scene.npz" % name))
    s = synth.load_scene_npz(os.path.join(GOLD, "%s_scene.npz" % name))
    tmp = tempfile.mkdtemp(prefix="golden_")
    try:
        synth.write_mve_scene(s, tmp)
        data = {}
        for tag, extra in (("gvs_default", ()), ("gvs_n3", ("-n3",))):
            for v, ids in gvs_lines(tmp, s.scale, s.nr_recon_neighbors, s.n_views, extra).items():
                data["%s_%d" % (tag, v)] = ids
        np.savez_compressed(os.path.join(GOLD, "%s_ref.npz" % name), **data)
        print(name, "gvs only;", "view 0 ->", data["gvs_default_0"])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def mint(name, map_views, n_patches=1500, focus=()):
    """focus: views whose patches are kept beyond the random slice - every traced PatchOptimization that samples one of
    them, up to 1000."""
    s = synth.make_scene(name)
    synth.save_scene_npz(s, os.path.join(GOLD, "%s_scene.npz" % name))
    s = synth.load_scene_npz(os.path.join(GOLD, "%s_scene.npz" % name))
    tmp = tempfile.mkdtemp(prefix="golden_")
    try:
        synth.write_mve_scene(s, tmp)
        data = {}
        for tag, extra in (("gvs_default", ()), ("gvs_n3", ("-n3",))):
            g = gvs_lines(tmp, s.scale, s.nr_recon_neighbors, s.n_views, extra)
            for v, ids in g.items():
                data["%s_%d" % (tag, v)] = ids
        run_cli(tmp, s.scale, s.nr_recon_neighbors)
        for v in map_views:
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            data["depth_%d" % v] = synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % s.scale))[:, :, 0]
            data["conf_%d" % v] = synth.read_mvei(os.path.join(vd, "conf-L%d.mvei" % s.scale))[:, :, 0]
            data["dz_%d" % v] = synth.read_mvei(os.path.join(vd, "dz-L%d.mvei" % s.scale))
            if s.scale:
                data["undist_%d" % v] = synth.read_mvei(os.path.join(vd, "undist-L%d.png" % s.scale))
        # patch-level vectors: realistic inputs = a slice of the oracle's own execution trace (seeds + queue)
        osc = O.OracleScene(s)
        st = O.default_settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
        ref = map_views[0]
        r = osc.reconstruct(st, ref, trace_cap=200000)
        tin = r["trace_in"]
        seeds = np.nonzero(tin["n_local"] == 0)[0]
        rest = np.nonzero(tin["n_local"] != 0)[0]
        rng = np.random.default_rng(7)
        pick = np.concatenate([seeds, rng.choice(rest, size=min(n_patches, len(rest)), replace=False)])
        if focus:
            tout = r["trace_out"]
            near = np.nonzero(np.isin(tin["local_ids"], focus).any(1) | np.isin(tout["local_ids"], focus).any(1))[0]
            pick = np.concatenate([pick, rng.choice(near, size=min(1000, len(near)), replace=False)])
        pick = np.unique(pick)
        pin = np.ascontiguousarray(tin[pick])
        # a few hostile inputs: image border, negative depth slope, far-off depth
        extra = np.zeros(6, O.PATCH_IN)
        extra["local_ids"] = -1
        extra[0] = (1, 1, 5.0, 0, 0, 0, [-1] * 4)
        extra[1] = (s.size(ref)[0] // (2 ** s.scale) - 2, 10, 5.0, 0, 0, 0, [-1] * 4)
        extra[2] = (40, 40, 5.0, -3.0, 0.0, 0, [-1] * 4)
        extra[3] = (40, 40, 50.0, 0, 0, 0, [-1] * 4)
        extra[4] = (40, 40, 0.5, 0, 0, 0, [-1] * 4)
        extra[5] = (40, 40, -1.0, 0, 0, 0, [-1] * 4)
        pin = np.concatenate([pin, extra])
        fin, fout = os.path.join(tmp, "pin.bin"), os.path.join(tmp, "pout.bin")
        pin.tofile(fin)
        txt = subprocess.run([os.path.join(REF, "ref_harness"), "patches", tmp, str(ref), str(s.scale),
                              str(s.nr_recon_neighbors), fin, fout], capture_output=True, text=True, check=True).stdout
        m = re.search(r"Global View Selection:([ 0-9]*)", txt)
        data["patch_gvs"] = np.asarray([int(x) for x in m.group(1).split()], np.int32)
        data["patch_ref_view"] = np.int32(ref)
        data["patch_in"] = pin
        data["patch_out"] = np.fromfile(fout, dtype=O.PATCH_OUT)
        np.savez_compressed(os.path.join(GOLD, "%s_ref.npz" % name), **data)
        print(name, "patches", len(pin), "maps", map_views)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def sampled_map(maps, n_sample, seed=0):
    """A full-size reference map reduced for storage: the fill mask in full (bit-packed) and depth / conf / dz at a seeded
    sample of the filled pixels."""
    depth = maps["depth"]
    filled = np.flatnonzero(depth > 0)
    idx = np.sort(np.random.default_rng(seed).choice(filled, size=min(n_sample, len(filled)), replace=False)).astype(np.int32)
    return dict(shape=np.asarray(depth.shape, np.int32), mask=np.packbits(depth.reshape(-1) > 0), idx=idx,
                depth=depth.reshape(-1)[idx], conf=maps["conf"].reshape(-1)[idx], dz=maps["dz"].reshape(-1, 2)[idx])


def mint_baseline_size():
    """Reference CLI maps of the BASELINE-sized views of tests/test_gpu_parity_baseline_size.py (scenes generated on the CPU)."""
    from tests.test_gpu_parity_baseline_size import C5R
    from tests.util import reference_cli_maps
    for name, s, view in (("C2_view5", synth.make_scene("C2"), 5), ("C5r_view3", synth.make_scene("C5", **C5R), 3)):
        ref = reference_cli_maps(s, [view])[view]
        np.savez_compressed(os.path.join(GOLD, "%s_ref.npz" % name), **sampled_map(ref, 4096))
        print(name, int((ref["depth"] > 0).sum()), "filled px")


def mint_depthmap_ops():
    """libs/mve/depthmap.cc through ref_harness dmops on the cases of tests/test_gpu_depthmap_ops.py: bit-exact results as
    SHA-256 digests, float results of triangulate at up to 256 seeded vertices."""
    from tests.test_gpu_depthmap_ops import CLEANUP_THRES, TRI_CASES, depth_case, tri_inputs
    harness = os.path.join(REF, "ref_harness")
    data = {}
    with tempfile.TemporaryDirectory() as tmp:
        for kind in ("golden", "ragged", "large"):
            dm, cm = depth_case(kind)
            h, w = dm.shape
            dm.tofile(os.path.join(tmp, "dm.f32")); cm.tofile(os.path.join(tmp, "cm.f32"))
            subprocess.run([harness, "dmops", "confclean", str(w), str(h), os.path.join(tmp, "dm.f32"), os.path.join(tmp, "cm.f32"),
                            os.path.join(tmp, "cc.f32")], check=True)
            data["confclean_%s" % kind] = sha256(np.fromfile(os.path.join(tmp, "cc.f32"), np.float32))
            for thres in CLEANUP_THRES:
                subprocess.run([harness, "dmops", "cleanup", str(w), str(h), str(thres), os.path.join(tmp, "dm.f32"),
                                os.path.join(tmp, "cl.f32")], check=True)
                data["cleanup_%s_%d" % (kind, thres)] = sha256(np.fromfile(os.path.join(tmp, "cl.f32"), np.float32))
        for kind, dd, color in TRI_CASES:
            dm, invproj, ci = tri_inputs(kind, color)
            h, w = dm.shape
            dm.tofile(os.path.join(tmp, "dm.f32"))
            cpath = "-"
            if ci is not None:
                cpath = os.path.join(tmp, "ci.u8"); ci.tofile(cpath)
            subprocess.run([harness, "dmops", "triangulate", str(w), str(h), repr(dd), os.path.join(tmp, "dm.f32"), cpath,
                            str(channels(ci))] + [repr(float(v)) for v in invproj] + [os.path.join(tmp, "out")], check=True)
            rd = lambda ext, t: np.fromfile(os.path.join(tmp, "out." + ext), t)      # noqa: E731
            vids, faces, confs = rd("vids", np.uint32), rd("faces", np.uint32), rd("confs", np.float32)
            verts, nrm, scl, cols = rd("verts", np.float32).reshape(-1, 3), rd("normals", np.float32).reshape(-1, 3), \
                rd("scales", np.float32), rd("colors", np.float32)
            key = "tri_%s_%g_%d" % (kind, dd, int(color))
            pick = np.sort(np.random.default_rng(0).choice(len(verts), size=min(256, len(verts)), replace=False)).astype(np.int32)
            data[key + "_n"] = np.asarray([len(verts), len(faces) // 3], np.int64)
            data[key + "_sha"] = np.asarray([sha256(vids), sha256(faces), sha256(confs)])
            data[key + "_pick"] = pick
            data[key + "_verts"], data[key + "_normals"], data[key + "_scales"] = verts[pick], nrm[pick], scl[pick]
            data[key + "_scales_absmax"] = np.float32(np.abs(scl).max())
            data[key + "_verts_absmax"] = np.float32(np.abs(verts).max())
            if cols.size:
                data[key + "_colors"] = cols.reshape(-1, 4)[pick]
    np.savez_compressed(os.path.join(GOLD, "depthmap_ops_ref.npz"), **data)
    print("depthmap ops", len(data), "entries")


def channels(ci):
    return 0 if ci is None else (1 if ci.ndim == 2 else ci.shape[2])


def mint_depthmap_edges():
    """libs/mve/depthmap.cc through ref_harness dmops on the cases of tests/test_gpu_depthmap_edges.py, stored like
    depthmap_ops_ref.npz: SHA-256 digests of the exact results (per cleanup threshold, per confidence iteration count) and
    the float results at up to 256 seeded vertices."""
    from tests.test_gpu_depthmap_edges import cleanup_cases, tri_cases
    harness = os.path.join(REF, "ref_harness")
    data = {}
    with tempfile.TemporaryDirectory() as tmp:
        f = lambda name: os.path.join(tmp, name)      # noqa: E731
        for name, (dm, cm, thres) in cleanup_cases().items():
            h, w = dm.shape
            dm.tofile(f("dm.f32")); cm.tofile(f("cm.f32"))
            subprocess.run([harness, "dmops", "confclean", str(w), str(h), f("dm.f32"), f("cm.f32"), f("cc.f32")], check=True)
            data["confclean_%s" % name] = sha256(np.fromfile(f("cc.f32"), np.float32))
            data["cleanup_%s_thres" % name] = np.asarray(thres, np.int64)
            for t in thres:
                subprocess.run([harness, "dmops", "cleanup", str(w), str(h), str(t), f("dm.f32"), f("cl.f32")], check=True)
                data["cleanup_%s_%d" % (name, t)] = sha256(np.fromfile(f("cl.f32"), np.float32))
        for name, c in tri_cases().items():
            dm, ci = c["dm"], c["color"]
            h, w = dm.shape
            dm.tofile(f("dm.f32"))
            cpath = "-"
            if ci is not None:
                cpath = f("ci.u8"); ci.tofile(cpath)
            key = "tri_%s" % name
            for k, it in enumerate(c["ref_iters"]):
                subprocess.run([harness, "dmops", "triangulate", str(w), str(h), repr(c["dd"]), f("dm.f32"), cpath, str(channels(ci))]
                               + [repr(float(v)) for v in c["invproj"]] + [f("out"), str(it), repr(c["scale"])], check=True)
                rd = lambda ext, t: np.fromfile(f("out." + ext), t)      # noqa: E731
                data["%s_confs_%d" % (key, it)] = sha256(rd("confs", np.float32))
                if k:
                    continue
                vids, faces = rd("vids", np.uint32), rd("faces", np.uint32)
                verts, nrm, scl, cols = rd("verts", np.float32).reshape(-1, 3), rd("normals", np.float32).reshape(-1, 3), \
                    rd("scales", np.float32), rd("colors", np.float32)
                pick = np.sort(np.random.default_rng(0).choice(len(verts), size=min(256, len(verts)), replace=False)).astype(np.int32)
                data[key + "_n"] = np.asarray([len(verts), len(faces) // 3], np.int64)
                data[key + "_sha"] = np.asarray([sha256(vids), sha256(faces)])
                data[key + "_pick"] = pick
                data[key + "_verts"], data[key + "_normals"], data[key + "_scales"] = verts[pick], nrm[pick], scl[pick]
                data[key + "_scales_absmax"] = np.float32(np.abs(scl).max(initial=0))
                data[key + "_verts_absmax"] = np.float32(np.abs(verts).max(initial=0))
                if cols.size:
                    data[key + "_colors"] = cols.reshape(-1, 4)[pick]
    np.savez_compressed(os.path.join(GOLD, "depthmap_edges_ref.npz"), **data)
    print("depthmap edges", len(data), "entries")


def mint_fresh_scene_patches():
    """mvs::PatchOptimization of the reference on a slice of the oracle's trace of a scene that no other fixture uses."""
    from tests.test_oracle_vs_reference import fresh_scene_trace
    s, tin = fresh_scene_trace()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        tin.tofile(fin)
        subprocess.run([os.path.join(REF, "ref_harness"), "patches", tmp, "1", "0", "4", fin, fout], check=True, capture_output=True)
        out = np.fromfile(fout, dtype=O.PATCH_OUT)
    np.savez_compressed(os.path.join(GOLD, "T0s77_ref.npz"), patch_in=tin, conf=out["conf"], depth=out["depth"],
                        local_ids=out["local_ids"].astype(np.int8))
    print("fresh scene", len(tin), "patches")


# scene -> reference view of the edge cases (the view of the scene's patch slice in <S>_ref.npz)
EDGE_SCENES = (("T0", 0), ("T4", 1), ("T5", 1), ("T6", 2))


def save_npz_stable(path, **arrays):
    """np.savez_compressed with fixed member timestamps, so that a second run writes the same bytes."""
    import io
    import zipfile
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)


def mint_patch_edges():
    """mvs::PatchOptimization through ref_harness on the edge cases of tests/patch_edges.py.make_cases, built from the
    oracle's execution trace of each scene's reference view (seeded: a second run gives the same bytes)."""
    from tests import patch_edges as PE
    data = {}
    for name, ref in EDGE_SCENES:
        s = synth.load_scene_npz(os.path.join(GOLD, "%s_scene.npz" % name))
        osc = O.OracleScene(s)
        st = O.default_settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
        gsel = osc.global_view_selection(st, ref)
        r = osc.reconstruct(st, ref, trace_cap=200000)
        pin = PE.make_cases(s, ref, s.scale, gsel, r["trace_in"], r["trace_out"], np.random.default_rng(11))
        with tempfile.TemporaryDirectory(prefix="golden_") as tmp:
            synth.write_mve_scene(s, tmp)
            fin, fout = os.path.join(tmp, "pin.bin"), os.path.join(tmp, "pout.bin")
            pin.tofile(fin)
            txt = subprocess.run([os.path.join(REF, "ref_harness"), "patches", tmp, str(ref), str(s.scale),
                                  str(s.nr_recon_neighbors), fin, fout], capture_output=True, text=True, check=True).stdout
            m = re.search(r"Global View Selection:([ 0-9]*)", txt)
            data[name + "_patch_gvs"] = np.asarray([int(x) for x in m.group(1).split()], np.int32)
            data[name + "_patch_out"] = np.fromfile(fout, dtype=O.PATCH_OUT)
        assert data[name + "_patch_gvs"].tolist() == gsel
        data[name + "_patch_in"] = pin
        data[name + "_patch_ref_view"] = np.int32(ref)
        print(name, "edge patches", len(pin), "reference successes", int((data[name + "_patch_out"]["conf"] > 0).sum()))
    save_npz_stable(os.path.join(GOLD, "patch_edges_ref.npz"), **data)


def mint_ply():
    """.xf files and PLY header / element counts written by the reference CLI with -p (tests/test_gpu_dropin_cli.py)."""
    from tests.test_gpu_dropin_cli import PLY_VIEWS, ply_cmd, read_ply_header
    s = synth.load_scene_npz(os.path.join(GOLD, "T0_scene.npz"))
    data = {}
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        subprocess.run(ply_cmd(os.path.join(REF, "dmrecon"), s, tmp), check=True, capture_output=True,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
        for v in PLY_VIEWS:
            name = "mvs-%04d-L%d" % (v, s.scale)
            nv, nf, head = read_ply_header(os.path.join(tmp, "plyout", name + ".ply"))
            data["ply_%d" % v] = np.asarray([nv, nf], np.int64)
            data["ply_props_%d" % v] = np.asarray([l for l in head.splitlines() if l.startswith("property")])
            data["xf_%d" % v] = np.asarray(open(os.path.join(tmp, "plyout", name + ".xf")).read())
    np.savez_compressed(os.path.join(GOLD, "T0_ply_ref.npz"), **data)


if __name__ == "__main__":
    parts = sys.argv[1:] or ["tiny", "cameras", "baseline_size", "depthmap_ops", "depthmap_edges", "fresh_scene_patches", "ply",
                              "patch_edges"]
    if "tiny" in parts:
        np.save(os.path.join(GOLD, "srgb2lin.npy"), parse_lut())
        mint("T0", [0, 3])
        mint("T1", [4])
        mint("T2", [0])
        mint("T4", [1])
        mint_gvs_only("T3")
    if "cameras" in parts:
        mint("T5", [1], focus=(5, 6))
        mint("T6", [2], focus=(1, 3, 5, 7, 9))
    for p in parts:
        if p not in ("tiny", "cameras"):
            globals()["mint_" + p]()
