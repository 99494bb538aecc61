"""scene2pset on the GPU against the reference app: wall time of the drop-in CLI (oracle/_ref/shim/scene2pset_b200) and of
the unmodified reference (oracle/_ref/scene2pset, OpenMP on all host threads) on the depth maps the engine writes for
BASELINE scenes, with and without silhouette masks.

    python tools/pset_bench.py [--scenes C2,C5] [--out FILE]

Per scene: the engine reconstructs every view; the scene directory gets depth-L<s>.mvei per view and a one-channel
`mask` per view: a silhouette made from the view's own map (filled pixels, holes closed, grown by 8 pixels), 255 inside
and 0 outside, so a view's points survive its own mask and the other views' masks cut what lies outside them.  Both apps
then run `-n -c -s` (plus `-m mask`); scenes at scale > 0 run without colours
(`-i none`: the scene holds colour images at full size only).  The drop-in reports the device time of
each phase (B200MVS_PSET_STATS).  The point counts of the two outputs are compared.  The card name and power limit are
read with nvidia-smi in the same run and printed with the numbers.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import scipy.ndimage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "scene2pset_b200")
REF = os.path.join(ROOT, "oracle", "_ref", "scene2pset")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def write_scene(name, tmp):
    """Reconstructs every view of BASELINE scene `name` with the engine and writes the scene directory."""
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    maps, _ = sc.reconstruct(st, list(range(s.n_views)), want=("depth",))
    sc.close()
    synth.write_mve_scene(s, tmp)
    n_px = 0
    for v, m in enumerate(maps):
        vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
        d = np.ascontiguousarray(m["depth"], np.float32)
        synth.write_mvei(os.path.join(vd, "depth-L%d.mvei" % s.scale), d)
        sil = scipy.ndimage.binary_dilation(scipy.ndimage.binary_fill_holes(d > 0), iterations=8)
        synth.write_mvei(os.path.join(vd, "mask.mvei"), np.where(sil, 255, 0).astype(np.uint8))
        n_px += d.size
    return s, n_px


def timed(exe, args, scene_dir, out, env):
    t0 = time.perf_counter()
    r = subprocess.run([exe] + args + [scene_dir, out], capture_output=True, text=True, env=env)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        raise RuntimeError(r.stdout + r.stderr)
    n = int(re.findall(r"Writing final point set \((\d+) points\)", r.stdout)[-1])
    return dt, n, r.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    for exe in (CLI, REF):
        if not os.path.exists(exe):
            sys.exit("%s not built (python -c 'import __graft_entry__ as g; g.build()')" % exe)
    rows = [dict(card(), host_threads=os.cpu_count())]
    print(json.dumps(rows[0]), flush=True)
    for name in a.scenes.split(","):
        with tempfile.TemporaryDirectory(prefix="pset_bench_") as tmp:
            s, n_px = write_scene(name, tmp)
            base = ["-n", "-c", "-s", "-d", "depth-L%d" % s.scale] + (["-i", "none"] if s.scale else [])
            for masked in (False, True):
                args = base + (["-m", "mask"] if masked else [])
                env_ref = {k: v for k, v in os.environ.items() if k != "OMP_NUM_THREADS"}
                t_ref, n_ref, _ = timed(REF, args, tmp, os.path.join(tmp, "ref.ply"), env_ref)
                t_gpu, n_gpu, out = timed(CLI, args, tmp, os.path.join(tmp, "gpu.ply"), dict(os.environ, B200MVS_PSET_STATS="1"))
                st = re.search(r"peak device bytes (\d+), device ms: pointset ([\d.e+-]+), filter ([\d.e+-]+), mask ([\d.e+-]+)", out)
                row = dict(scene=name, views=s.n_views, map_px=n_px, masks=masked, points_ref=n_ref, points_gpu=n_gpu,
                           ref_s=round(t_ref, 3), gpu_cli_s=round(t_gpu, 3), speedup=round(t_ref / t_gpu, 2),
                           peak_device_bytes=int(st.group(1)), device_ms_pointset=float(st.group(2)),
                           device_ms_filter=float(st.group(3)), device_ms_mask=float(st.group(4)))
                print(json.dumps(row), flush=True)
                rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
