"""Shared helpers for the parity tests (test infrastructure)."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def golden_scene(name):
    from mve_b200 import synth
    return synth.load_scene_npz(os.path.join(GOLD, "%s_scene.npz" % name))


def golden_ref(name):
    return np.load(os.path.join(GOLD, "%s_ref.npz" % name))


def map_stats(a_depth, b_depth):
    """Fill-mask IoU and relative depth difference percentiles on commonly filled pixels."""
    m1, m2 = a_depth > 0, b_depth > 0
    both = m1 & m2
    iou = both.sum() / max(1, (m1 | m2).sum())
    rel = np.abs(a_depth - b_depth)[both] / a_depth[both]
    return iou, rel, both


def patch_compare(got, ref):
    """Compares PatchOptimization results. Returns dict of mismatch counts / error percentiles."""
    ok_r, ok_g = ref["conf"] > 0, got["conf"] > 0
    both = ok_r & ok_g
    rel = np.abs(got["depth"] - ref["depth"])[both] / np.abs(ref["depth"][both])
    return dict(n=len(ref), ok_mismatch=int((ok_r != ok_g).sum()),
                ids_mismatch=int((got["local_ids"] != ref["local_ids"]).any(-1)[both].sum()),
                rel=rel, conf_abs=np.abs(got["conf"] - ref["conf"])[both],
                dz_abs=np.maximum(np.abs(got["dz_i"] - ref["dz_i"]), np.abs(got["dz_j"] - ref["dz_j"]))[both],
                nrm_abs=np.abs(got["normal"] - ref["normal"]).max(-1)[both], both=both)


def reference_cli_maps(scene, views, threads=None):
    """Runs the UNMODIFIED reference CLI (oracle/_ref/dmrecon, compiled from /root/reference by oracle/Makefile; the
    binary travels to the GPU box) on `scene` for the reference views `views` and returns {view: dict(depth, conf, dz)}.
    One host thread per view like apps/dmrecon/dmrecon.cc:285."""
    import subprocess
    import tempfile
    from mve_b200 import synth
    exe = os.path.join(ROOT, "oracle", "_ref", "dmrecon")
    if not os.path.exists(exe):
        return None
    out = {}
    with tempfile.TemporaryDirectory(prefix="b200mvs_refcli_") as tmp:
        synth.write_mve_scene(scene, tmp)
        cmd = [exe, "-s%d" % scene.scale, "--local-neighbors=%d" % scene.nr_recon_neighbors, "--keep-conf", "--keep-dz",
               "--progress=silent", "--force", "-l" + ",".join(str(v) for v in views), tmp]
        env = dict(os.environ, OMP_NUM_THREADS=str(threads or len(views)))
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=3000)
        assert r.returncode == 0, r.stdout + r.stderr
        for v in views:
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            out[v] = dict(depth=synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % scene.scale))[:, :, 0],
                          conf=synth.read_mvei(os.path.join(vd, "conf-L%d.mvei" % scene.scale))[:, :, 0],
                          dz=synth.read_mvei(os.path.join(vd, "dz-L%d.mvei" % scene.scale)))
    return out


def map_parity_sampled(ref, got):
    """map_parity against a stored reference map (tests/golden/make_golden.py sampled_map): fill figures on the whole
    mask, depth / conf / dz figures on the stored sample of reference pixels that `got` fills too."""
    shape = tuple(int(x) for x in ref["shape"])
    m_ref = np.unpackbits(ref["mask"], count=shape[0] * shape[1]).astype(bool)
    m_got = got["depth"].reshape(-1) > 0
    n_ref = int(m_ref.sum())
    iou = (m_ref & m_got).sum() / max(1, (m_ref | m_got).sum())
    both = m_got[ref["idx"]]
    idx = ref["idx"][both]
    rel = np.abs(ref["depth"][both] - got["depth"].reshape(-1)[idx]) / ref["depth"][both]
    dz = np.abs(ref["dz"][both] - got["dz"].reshape(-1, 2)[idx]).max(-1)
    return dict(iou=float(iou), fill_ratio_diff=float(abs(int(m_got.sum()) - n_ref) / max(1, n_ref)),
                depth_rel_p50=float(np.percentile(rel, 50)), depth_rel_p99=float(np.percentile(rel, 99)),
                depth_rel_le_1e3=float((rel <= 1e-3).mean()), depth_rel_le_1e2=float((rel <= 1e-2).mean()),
                conf_abs_p99=float(np.percentile(np.abs(ref["conf"][both] - got["conf"].reshape(-1)[idx]), 99)),
                dz_abs_p99=float(np.percentile(dz, 99)), n_both=int(both.sum()))


def map_parity(ref, got):
    """SURVEY.md 8c map-level figures of `got` against `ref` (dicts with depth, conf, dz)."""
    iou, rel, both = map_stats(ref["depth"], got["depth"])
    n_ref = int((ref["depth"] > 0).sum())
    res = dict(iou=float(iou), fill_ratio_diff=float(abs(int((got["depth"] > 0).sum()) - n_ref) / max(1, n_ref)),
               depth_rel_p50=float(np.percentile(rel, 50)), depth_rel_p99=float(np.percentile(rel, 99)),
               depth_rel_le_1e3=float((rel <= 1e-3).mean()), depth_rel_le_1e2=float((rel <= 1e-2).mean()),
               conf_abs_p99=float(np.percentile(np.abs(ref["conf"] - got["conf"])[both], 99)),
               dz_abs_p99=float(np.percentile(np.abs(ref["dz"] - got["dz"])[both].max(-1), 99)), n_both=int(both.sum()))
    if "view_ids" in ref and "view_ids" in got:
        res["view_ids_equal"] = float((ref["view_ids"] == got["view_ids"]).all(-1)[both].mean())
        a, b = ref["view_ids"][both], got["view_ids"][both]
        shared = ((a[:, :, None] == b[:, None, :]) & (a[:, :, None] >= 0)).any(-1).sum(-1)
        res["view_ids_shared_mean"] = float(shared.mean())          # of the (up to) 4 local views of a pixel
        res["view_ids_share_ge3"] = float((shared >= 3).mean())
    return res
