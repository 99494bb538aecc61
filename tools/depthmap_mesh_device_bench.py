"""Triangulating the depth maps of a reconstruction that stay on the GPU: through host memory, map by map, against the
batched device entry point.

    python tools/depthmap_mesh_device_bench.py [--scenes C2,C5] [--reps 5] [--out FILE]

Per scene the maps and level images come from Scene.reconstruct(on_device=True) and Scene.level(on_device=True), made
once and cleaned on the device (depthmap_confidence_clean_maps, then depthmap_cleanup_maps with threshold 100).  Each map
gets its view's inverse calibration and camera-to-world matrix.  Both routes compute the per-view work of scene2pset
(vertex ids, vertices, colours, faces, normals, confidences over 4 rings, scale values) of every map:
  host:   per map .cpu().numpy() of the depth map and the level image, the host entry point (b200mvs_depthmap_pointset),
          and every output back with .cuda();
  device: depthmap_pointset_maps: two library calls for the whole batch (b200mvs_depthmap_pointset_device), one that
          counts and one that fills exactly sized tensors.
After one warm-up of each, the routes alternate --reps times; printed per route: wall time median and min-max (each route
ends in a device synchronise), the PCIe bytes the route moves (computed from the shapes), and whether the outputs of the
two routes are byte-identical.  A separate pass under torch.profiler gives the kernel time of the device route.  The
card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KERNELS = ("k_tri_codes", "k_tri_counts", "k_tri_totals", "k_tri_clear", "k_tri_vertices", "k_tri_faces", "k_vertex_attributes",
           "k_conf_ring", "k_conf_write", "DeviceScan")
KEYS = ("vertex_ids", "vertices", "colors", "faces", "normals", "confidences", "scales")
OPTS = dict(with_normals=True, conf_iterations=4, scale_factor=2.5)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def camera(s, v, w, h):
    """The inverse calibration of view v for a w x h map (CameraInfo::fill_inverse_calibration) and its camera-to-world
    matrix (CameraInfo::fill_cam_to_world)."""
    f32 = np.float32
    flen, pa = f32(s.flen[v]), f32(s.paspect[v])
    ppx, ppy = (f32(x) for x in np.asarray(s.ppoint[v], f32))
    W, H = f32(w), f32(h)
    if (W / H) * pa < f32(1.0):
        ax, ay = flen * H / pa, flen * H
    else:
        ax, ay = flen * W, flen * W * pa
    ip = np.array([f32(1) / ax, 0, -W * ppx / ax, 0, f32(1) / ay, -H * ppy / ay, 0, 0, 1], f32)
    r, t = np.asarray(s.rot[v], f32).reshape(3, 3), np.asarray(s.trans[v], f32)
    ctw = np.eye(4, dtype=f32)
    ctw[:3, :3] = r.T
    ctw[:3, 3] = -(r.T @ t)
    return ip, ctw


def run_scene(name, reps):
    import torch
    from mve_b200 import depthmap as D, dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    refs = list(range(s.n_views))
    try:
        maps, _ = sc.reconstruct(st, refs, want=("depth", "conf"), on_device=True)
        levels = [sc.level(v, st.scale, on_device=True) for v in refs]
    finally:
        sc.close()
    dev = maps[0]["depth"].device
    dms = [m["depth"] for m in maps]
    D.depthmap_confidence_clean_maps(dms, [m["conf"] for m in maps])
    D.depthmap_cleanup_maps(dms, 100, out=dms)
    cams = [camera(s, v, d.shape[1], d.shape[0]) for v, d in zip(refs, dms)]
    del s, maps
    torch.cuda.synchronize(dev)

    def host_route():
        outs = []
        for d, lv, (ip, ctw) in zip(dms, levels, cams):
            r = D.depthmap_pointset(d.cpu().numpy(), ip, cam_to_world=ctw, color=lv.cpu().numpy(), **OPTS)
            outs.append({k: torch.from_numpy(r[k].view(np.int32) if r[k].dtype == np.uint32 else r[k]).to(dev) for k in KEYS})
        torch.cuda.synchronize(dev)
        return outs

    def device_route():
        outs = D.depthmap_pointset_maps(dms, [c[0] for c in cams], levels, [c[1] for c in cams], **OPTS)
        torch.cuda.synchronize(dev)
        return outs

    def as_bytes(t):
        return (t if t.dtype in (torch.float32, torch.int32) else t.view(torch.int32)).cpu().numpy().tobytes()

    routes = dict(host=host_route, device=device_route)
    first = {k: f() for k, f in routes.items()}                     # warm-up, and the outputs to compare
    equal = all(as_bytes(a[k]) == as_bytes(b[k]) for a, b in zip(first["host"], first["device"]) for k in KEYS)
    nv = sum(len(r["vertices"]) for r in first["device"])
    nf = sum(len(r["faces"]) for r in first["device"])
    del first
    times = dict(host=[], device=[])
    for _ in range(reps):
        for k, f in routes.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)

    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        device_route()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA and any(k in e.name for k in KERNELS)]
    per_kernel = {k: round(sum(e.device_time_total for e in ev if k in e.name) / 1000.0, 4) for k in KERNELS}

    px = sum(d.numel() for d in dms)
    blocks = sum((d.numel() + 255) // 256 for d in dms)
    # device route, per call: the map table up (216 B per map, 4 B per 256 pixels; the counts' 8 B per map of device
    # workspace that follows it are not sent) and the counts down (8 B per map)
    # host route: depth (4 B/px) and level (3 B/px) down, up again into the host entry point's staging, its outputs
    # (vertex ids 4 B/px, per vertex 12 + 16 + 12 + 4 + 4 B, per face 12 B) down and up again as tensors
    outputs = 4 * px + 48 * nv + 12 * nf
    row = dict(scene=name, maps=len(dms), pixels=int(px), vertices=int(nv), faces=int(nf), reps=reps, outputs_equal=bool(equal),
               host_pcie_bytes=int(2 * 7 * px + 2 * outputs), device_pcie_bytes=int(2 * ((216 + 8) * len(dms) + 4 * blocks)),
               device_kernel_ms=round(sum(per_kernel.values()), 4), device_kernel_launches=len(ev), kernel_ms=per_kernel)
    for k, v in times.items():
        row[k + "_s_median"] = round(statistics.median(v), 4)
        row[k + "_s_min"], row[k + "_s_max"] = round(min(v), 4), round(max(v), 4)
    del dms, levels
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures on the GPU only")
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    for name in a.scenes.split(","):
        rows.append(run_scene(name, max(a.reps, 3)))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    if not all(r["outputs_equal"] for r in rows[1:]):
        raise SystemExit("the host and device routes differ")


if __name__ == "__main__":
    main()
