"""The point set of a reconstruction as CUDA tensors: through a host-resident set against a device-resident one.

    python tools/pset_resident_bench.py [--scenes C2,C5] [--runs N] [--out FILE]

For each BASELINE scene (C2 runs at its scale 1, C5 at scale 0), with `-n -c -s`, without and with masks (each view's own
silhouette, made from its map as tools/pset_bench.py makes it: filled pixels, holes closed, grown by 8 pixels):
  route host:   Scene.reconstruct_pointset (b200mvs_pset_create handle), then torch.from_numpy(a).cuda() of every array;
  route device: Scene.reconstruct_pointset(on_device=True) (b200mvs_pset_create_on_device handle, read with
                b200mvs_pset_read_device).
Each route runs in a fresh process of its own (so its peak RSS is its own): the scene is made and uploaded, the maps for
the silhouettes are made, the route runs once to warm up and then `runs` times timed, each ending in a device
synchronise.  Printed per route: the median and spread of the wall time to CUDA tensors, the bytes over PCIe that the
point set moves (computed from the shapes: a host-resident set comes down view by view and goes up again as tensors, and
its mask clip sends every point's vertex up and a byte per point down; the masks go up on both routes), the process' peak
RSS, the handle's peak_device_bytes, the context's b200mvs_memory peak and ms_mask.  The point sets of the two routes must
be byte-identical.  The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the
host is reconfigured."""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OPTIONS = dict(with_normals=True, with_conf=True, with_scale=True)
ARRAYS = ("vertices", "normals", "colors", "values", "confidences")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def silhouettes(sc, s, st, refs):
    import scipy.ndimage
    maps, _ = sc.reconstruct(st, refs, want=("depth",))
    out = []
    for j, v in enumerate(refs):
        d = maps[j]["depth"]
        sil = scipy.ndimage.binary_dilation(scipy.ndimage.binary_fill_holes(d > 0), iterations=8)
        out.append(dict(mask=np.where(sil, 255, 0).astype(np.uint8),
                        camera=dict(flen=s.flen[v], paspect=s.paspect[v], ppoint=s.ppoint[v], rot=s.rot[v], trans=s.trans[v])))
    return out


def run(sc, st, refs, masks, route):
    """One route to CUDA tensors; returns (tensors, result dict, PCIe bytes of the set)."""
    import torch
    r, _ = sc.reconstruct_pointset(st, refs, OPTIONS, masks, on_device=route == "device")
    pcie = sum(m["mask"].nbytes for m in masks or [])
    if route == "host":
        set_bytes = sum(r[k].nbytes for k in ARRAYS if r[k] is not None)
        pcie += 2 * set_bytes                                            # down view by view, up as tensors
        if masks:
            pcie += (len(r["vertices"]) + r["num_filtered"]) * 13         # clip: each vertex up, one flag byte down
        t = {k: torch.from_numpy(r[k]).cuda() for k in ARRAYS if r[k] is not None}
    else:
        t = {k: r[k] for k in ARRAYS if r[k] is not None}
    torch.cuda.synchronize()
    return t, r, pcie


def child(name, route, masked, runs, out):
    import torch
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    refs = list(range(s.n_views))
    masks = silhouettes(sc, s, st, refs) if masked == "1" else None
    run(sc, st, refs, masks, route)                                      # warm-up
    walls = []
    for _ in range(runs):
        t0 = time.perf_counter()
        t, r, pcie = run(sc, st, refs, masks, route)
        walls.append(time.perf_counter() - t0)
        mem = sc.memory_stats()
        np.savez(out, **{k: v.cpu().numpy() for k, v in t.items()})
        del t
        torch.cuda.synchronize()
    sc.close()
    print(json.dumps(dict(scene=name, route=route, masks=masked == "1", views=s.n_views, scale=s.scale, runs=runs,
                          points=int(len(r["vertices"])), num_filtered=int(r["num_filtered"]),
                          wall_s_median=round(float(np.median(walls)), 4), wall_s_min=round(min(walls), 4),
                          wall_s_max=round(max(walls), 4), pcie_bytes=int(pcie),
                          peak_rss_mb=round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0, 1),
                          handle_peak_device_bytes=int(r["info"]["peak_device_bytes"]), context_peak_bytes=int(mem.peak),
                          ms_mask=round(r["info"]["ms_mask"], 3))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", nargs=5, metavar=("SCENE", "ROUTE", "MASKED", "RUNS", "NPZ"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child[0], a.child[1], a.child[2], int(a.child[3]), a.child[4])
        return
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    with tempfile.TemporaryDirectory(prefix="pset_resident_bench_") as tmp:
        for name in a.scenes.split(","):
            for masked in ("0", "1"):
                res = {}
                for route in ("host", "device"):
                    npz = os.path.join(tmp, "%s_%s_%s.npz" % (name, route, masked))
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, route, masked, str(a.runs), npz],
                                       capture_output=True, text=True)
                    if p.returncode != 0:
                        raise RuntimeError(p.stdout + p.stderr)
                    rows.append(json.loads(p.stdout.strip().splitlines()[-1]))
                    res[route] = np.load(npz)
                    print(json.dumps(rows[-1]), flush=True)
                equal = sorted(res["host"].files) == sorted(res["device"].files) and \
                    all(res["host"][k].tobytes() == res["device"][k].tobytes() for k in res["host"].files)
                rows.append(dict(scene=name, masks=masked == "1", point_sets_equal=bool(equal)))
                print(json.dumps(rows[-1]), flush=True)
                if not equal:
                    raise SystemExit("the host-resident and device-resident sets differ on %s" % name)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
