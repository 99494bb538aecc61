"""Reconstruction masks on an object scene: what the background costs when it is reconstructed and then clipped, against
never reconstructing it.

    python tools/recon_mask_bench.py [--scene C5] [--reps 3] [--out FILE]

The scene (C5: 128 views of 1280x960, a textured sphere in front of a flat grey background, scale 0) is made and uploaded
once; every view gets its silhouette at the photo's size (synth.silhouette, the `valid` of the render).  In one process,
after one warm-up of each:
  maps:      Scene.reconstruct of every view, unmasked and with Scene.set_view_mask, alternating, --reps times each;
  point set: Scene.reconstruct_pointset unmasked with the silhouettes as scene2pset -m clip masks (masks=), against
             set_view_mask and no clip, alternating, --reps times each (-F option set).
Printed per run: wall time of the call (it returns after the device has finished), n_opt, n_sample_sets, n_rounds,
n_filled, n_seeds_processed, and for point sets the number of points.  The masked maps must fill no background pixel.
The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OPTIONS = dict(with_normals=True, with_conf=True, with_scale=True)
COUNTERS = ("n_opt", "n_sample_sets", "n_rounds", "n_filled", "n_seeds_processed", "n_seeds_success")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="C5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from mve_b200 import dmrecon, synth
    if not torch.cuda.is_available():
        raise SystemExit("recon_mask_bench needs a CUDA device")
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    s = synth.make_scene(a.scene, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    sil = {v: synth.silhouette(s, v, device="cuda") for v in refs}
    clip = [dict(mask=sil[v], camera=dict(flen=s.flen[v], paspect=s.paspect[v], ppoint=s.ppoint[v], rot=s.rot[v],
                                          trans=s.trans[v])) for v in refs]
    sc = dmrecon.Scene.from_synth(s)
    fg = float(np.mean([(m > 0).mean() for m in sil.values()]))
    rows.append(dict(scene=a.scene, views=s.n_views, width=s.width, height=s.height, scale=s.scale, foreground_fraction=round(fg, 4)))
    print(json.dumps(rows[-1]), flush=True)

    def masks(on):
        for v in refs:
            sc.set_view_mask(v, sil[v] if on else None)

    def maps_run(masked):
        masks(masked)
        t0 = time.perf_counter()
        maps, stats = sc.reconstruct(st, refs, want=("depth",))
        dt = time.perf_counter() - t0
        if masked:
            for j, v in enumerate(refs):
                assert not (maps[j]["depth"][sil[v] == 0] > 0).any(), v        # scale 0: the mask has the map's size
        return dict(kind="maps", masked=masked, wall_s=round(dt, 4), **{k: int(getattr(stats, k)) for k in COUNTERS})

    def pset_run(masked):
        masks(masked)
        t0 = time.perf_counter()
        r, stats = sc.reconstruct_pointset(st, refs, OPTIONS, None if masked else clip)
        dt = time.perf_counter() - t0
        return dict(kind="pointset", masked=masked, clip_masks=not masked, wall_s=round(dt, 4), points=int(len(r["vertices"])),
                    num_filtered=int(r["num_filtered"]), **{k: int(getattr(stats, k)) for k in COUNTERS})

    for fn in (maps_run, pset_run):
        fn(False)
        fn(True)                                     # warm-up of both
        for _ in range(a.reps):
            for masked in (False, True):
                rows.append(fn(masked))
                print(json.dumps(rows[-1]), flush=True)
    for kind in ("maps", "pointset"):
        for masked in (False, True):
            t = [r["wall_s"] for r in rows if r.get("kind") == kind and r["masked"] == masked]
            rows.append(dict(summary=kind, masked=masked, wall_s_median=float(np.median(t)), wall_s_min=min(t), wall_s_max=max(t)))
            print(json.dumps(rows[-1]), flush=True)
    sc.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
