"""Cleaning the depth maps of a reconstruction that stay on the GPU: through host memory, map by map, against the batched
device entry points.

    python tools/depthmap_device_bench.py [--scenes C2,C5] [--reps 3] [--thres 100] [--out FILE]

Per scene the maps come from Scene.reconstruct(on_device=True) (depth and conf as CUDA tensors, made once).  Both routes
run depthmap_confidence_clean, then depthmap_cleanup with threshold --thres, on every map:
  host:   per map .cpu().numpy() of depth and conf, the host entry points (b200mvs_depthmap_confidence_clean, then
          b200mvs_depthmap_cleanup), and the result back with .cuda();
  device: a clone of the depth maps, then depthmap_confidence_clean_maps and depthmap_cleanup_maps: two library calls
          for the whole batch (b200mvs_depthmap_confidence_clean_device / b200mvs_depthmap_cleanup_device).
After one warm-up of each, the routes alternate --reps times; printed per route: wall time median and min-max (each route
ends in a device synchronise), the PCIe bytes the route moves (computed from the shapes), and whether the outputs of the
two routes are byte-identical.  A separate pass under torch.profiler gives the kernel time of the device route
(k_conf_clean and k_cc_*).  The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU
or the host is reconfigured."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KERNELS = ("k_conf_clean", "k_cc_init", "k_cc_link", "k_cc_count", "k_cc_erase")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def run_scene(name, reps, thres):
    import torch
    from mve_b200 import depthmap as D, dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    try:
        maps, _ = sc.reconstruct(st, list(range(s.n_views)), want=("depth", "conf"), on_device=True)
    finally:
        sc.close()
    del s
    dev = maps[0]["depth"].device
    depth = [m["depth"] for m in maps]
    conf = [m["conf"] for m in maps]
    torch.cuda.synchronize(dev)

    def host_route():
        outs = []
        for d, c in zip(depth, conf):
            dn, cn = d.cpu().numpy(), c.cpu().numpy()
            D.depthmap_confidence_clean(dn, cn)
            outs.append(torch.from_numpy(D.depthmap_cleanup(dn, thres)).to(dev))
        torch.cuda.synchronize(dev)
        return outs

    def device_route():
        dms = [d.clone() for d in depth]
        D.depthmap_confidence_clean_maps(dms, conf)
        outs = D.depthmap_cleanup_maps(dms, thres, out=dms)
        torch.cuda.synchronize(dev)
        return outs

    routes = dict(host=host_route, device=device_route)
    first = {k: f() for k, f in routes.items()}                     # warm-up, and the outputs to compare
    equal = all(a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() for a, b in zip(first["host"], first["device"]))
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

    px = sum(d.numel() for d in depth)
    # host route per pixel: depth and conf down, the confidence_clean staging (8 B up, 4 B down), the cleanup staging
    # (4 B up, 4 B down), the result up
    row = dict(scene=name, maps=len(depth), pixels=int(px), thres=thres, reps=reps, outputs_equal=bool(equal),
               host_pcie_bytes=int(32 * px), device_pcie_bytes=0,
               device_kernel_ms=round(sum(per_kernel.values()), 4), device_kernel_launches=len(ev), kernel_ms=per_kernel)
    for k, v in times.items():
        row[k + "_s_median"] = round(statistics.median(v), 4)
        row[k + "_s_min"], row[k + "_s_max"] = round(min(v), 4), round(max(v), 4)
    del maps, depth, conf
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--thres", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures on the GPU only")
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    for name in a.scenes.split(","):
        rows.append(run_scene(name, max(a.reps, 3), a.thres))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    if not all(r["outputs_equal"] for r in rows[1:]):
        raise SystemExit("the host and device routes differ")


if __name__ == "__main__":
    main()
