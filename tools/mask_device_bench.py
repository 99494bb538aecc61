"""Masks that are already CUDA tensors: copied to the host and set as host masks, against set in device memory.

    python tools/mask_device_bench.py [--scene C5] [--reps 3] [--out FILE]

The scene (C5: 128 views of 1280x960, scale 0) is made and uploaded once; every view's silhouette at the photo's size
(synth.silhouette) is put on the device as a torch.uint8 tensor, as a segmentation network would leave it.  In one
process, after one warm-up of each, alternating, --reps times each:
  reconstruction: Scene.set_view_mask(t) of every view (the tensor goes through .cpu()) + reconstruct(on_device=True),
                  against set_view_mask(t, on_device=True) + the same reconstruction;
  clip:           the silhouette clip of a device-resident point set of the scene's maps (made before the timed part,
                  one per run) with the tensors' .cpu() copies (b200mvs_pset_clip_masks), against the tensors in place
                  (b200mvs_pset_clip_masks_device).
Printed per run: wall time of the timed part (it ends with a device synchronise), and for the clip the handle's ms_mask.
Each pair of outputs is checked equal: the maps byte for byte, the clipped points and num_filtered.  The card name and
power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon, synth
    if not torch.cuda.is_available():
        raise SystemExit("mask_device_bench needs a CUDA device")
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    s = synth.make_scene(a.scene, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    sil = {v: torch.from_numpy(np.ascontiguousarray(synth.silhouette(s, v, device="cuda"))).cuda() for v in refs}
    sc = dmrecon.Scene.from_synth(s)
    rows.append(dict(scene=a.scene, views=s.n_views, width=s.width, height=s.height, scale=s.scale,
                     mask_bytes=int(sum(t.numel() for t in sil.values()))))
    print(json.dumps(rows[-1]), flush=True)

    def recon(on_device):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for v in refs:
            sc.set_view_mask(v, sil[v], on_device=on_device)
        maps, _ = sc.reconstruct(st, refs, want=("depth", "conf"), on_device=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dict(kind="reconstruction", device_masks=on_device, wall_s=round(dt, 4)), maps

    # the scene's maps, once, for the point sets of the clip runs
    for v in refs:
        sc.set_view_mask(v, None)
    maps, _ = sc.reconstruct(st, refs, want=("depth",), on_device=True)
    cams = [dict(flen=s.flen[v], paspect=s.paspect[v], ppoint=s.ppoint[v], rot=s.rot[v], trans=s.trans[v]) for v in refs]
    masks = [dict(mask=sil[v], camera=cams[j]) for j, v in enumerate(refs)]
    L = D._pset_lib()
    _, opt = D._options(None)

    def clip(on_device):
        h = D._create(L, 0, opt, True)
        try:
            for j, v in enumerate(refs):
                D._add_device_view(L, h, dict(id=v, depth=maps[j]["depth"], camera=cams[j]))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if on_device:
                nf = D._clip_device_masks(L, h, masks, 0)
            else:
                host = [np.ascontiguousarray(m["mask"].cpu().numpy()) for m in masks]
                ptrs = (C.c_void_p * len(host))(*[m.ctypes.data for m in host])
                ws = np.array([m.shape[1] for m in host], np.int32)
                hs = np.array([m.shape[0] for m in host], np.int32)
                pc = (D._PsetCamera * len(host))(*[D._camera(c) for c in cams])
                n = C.c_uint64(0)
                D._check(L.b200mvs_pset_clip_masks(h, len(host), ptrs, D._p(ws), D._p(hs), pc, C.byref(n)))
                nf = int(n.value)
            dt = time.perf_counter() - t0
            r = D._finish(L, h, D._options(None)[0], None, [], 0)
            torch.cuda.synchronize()
            row = dict(kind="clip", device_masks=on_device, wall_s=round(dt, 4), ms_mask=round(r["info"]["ms_mask"], 3),
                       num_filtered=nf, points=int(r["vertices"].shape[0]))
            return row, r["vertices"]
        finally:
            L.b200mvs_pset_destroy(h)

    for fn in (recon, clip):
        fn(False)
        fn(True)                                     # warm-up of both
        for _ in range(a.reps):
            out = {}
            for on_device in (False, True):
                row, out[on_device] = fn(on_device)
                rows.append(row)
                print(json.dumps(row), flush=True)
            if fn is recon:
                for j in range(len(refs)):
                    for k in ("depth", "conf"):
                        assert torch.equal(out[False][j][k], out[True][j][k]), (j, k)
            else:
                assert torch.equal(out[False], out[True]) and rows[-1]["num_filtered"] == rows[-2]["num_filtered"]
    for kind in ("reconstruction", "clip"):
        for on_device in (False, True):
            t = [r["wall_s"] for r in rows if r.get("kind") == kind and r["device_masks"] == on_device]
            rows.append(dict(summary=kind, device_masks=on_device, wall_s_median=float(np.median(t)), wall_s_min=min(t),
                             wall_s_max=max(t)))
            print(json.dumps(rows[-1]), flush=True)
    sc.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
