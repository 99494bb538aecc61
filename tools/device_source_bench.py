"""Images that are already CUDA tensors, given to a reconstruction through a host image source or a device image source.

    python tools/device_source_bench.py [--scenes C2,C5] [--runs N] [--out FILE]

The scene's images are first made resident as CUDA tensors (packed HWC, and a planar CHW copy).  Three routes then
alternate in one process, each reconstruction on a fresh context whose images are all fetched through its source:
  host: Scene.set_image_source(lambda v: hwc[v].cpu().numpy()) - every fetch comes down to the host and goes back up
        through the library's pinned staging;
  hwc:  Scene.set_image_source(lambda v: hwc[v], on_device=True) - the pyramid is built from the tensor in place;
  chw:  the same with layout="chw" over the planar copies.
C5 (128 views of 1280x960, scale 0) runs under a budget of fixed + max(largest single-view working set, working set of
all views / 4), from b200mvs_working_set, so that its groups evict pyramids and fetch views again; C2 (16 views of
1920x1080, scale 1) runs without a budget of its own (budget_bytes = 0: 90 % of the free device memory), one fetch per
view.  The maps go to CUDA tensors (reconstruct(on_device=True)).  After one warm-up of each route, `runs` rounds of the
three routes are timed, each reconstruction ending in a device synchronise.  Printed per route: the median and min-max wall
time, n_loads and n_evictions, and the image bytes over PCIe computed from the shapes (2 x bytes_loaded on the host route:
down by .cpu(), up from staging; 0 on the device routes); and whether every map of every route is bit-identical to the
host route's.  The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is
reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ROUTES = ("host", "hwc", "chw")
MAPS = ("depth", "conf", "dz", "normal", "view_ids")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def budget_for(s, st, refs, budgeted):
    """0 (no budget of its own) or fixed + max(largest single working set, working set of all views / 4)."""
    from mve_b200 import dmrecon
    if not budgeted:
        return 0, None
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    single = max(sc.working_set(st, [r]) for r in refs)
    total = sc.working_set(st, refs)
    sc.close()
    return fixed + max(single, total // 4), dict(fixed=fixed, largest_single=single, all_views=total)


def run(s, st, refs, budget, route, hwc, chw):
    """One reconstruction on a fresh context: (wall seconds of the reconstruct call, maps, b200mvs_memory dict)."""
    import torch
    from mve_b200 import dmrecon
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    if route == "host":
        sc.set_image_source(lambda v: hwc[v].cpu().numpy(), budget)
    elif route == "hwc":
        sc.set_image_source(lambda v: hwc[v], budget, on_device=True)
    else:
        sc.set_image_source(lambda v: chw[v], budget, on_device=True, layout="chw")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    maps, _ = sc.reconstruct(st, refs, on_device=True)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    mem = sc.memory_stats().as_dict()
    sc.close()
    return wall, maps, mem


def same_maps(a, b):
    import torch
    for x, y in zip(a, b):
        for k in MAPS:
            if not torch.equal(x[k].view(torch.int32), y[k].view(torch.int32)):
                return False
    return len(a) == len(b)


def bench(name, runs):
    import torch
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    budget, sizes = budget_for(s, st, refs, name == "C5")
    hwc = [torch.from_numpy(np.ascontiguousarray(img)).cuda() for img in s.images]
    chw = [t.permute(2, 0, 1).contiguous() for t in hwc]
    torch.cuda.synchronize()
    walls = {r: [] for r in ROUTES}
    mems, last = {}, {}
    for r in ROUTES:                                                         # warm-up
        run(s, st, refs, budget, r, hwc, chw)
    for _ in range(runs):
        for r in ROUTES:
            wall, maps, mems[r] = run(s, st, refs, budget, r, hwc, chw)
            walls[r].append(wall)
            last[r] = maps
    rows = []
    for r in ROUTES:
        m = mems[r]
        rows.append(dict(scene=name, route=r, views=s.n_views, size="%dx%d" % s.size(0), scale=s.scale,
                         budget=int(m["budget"]) if budget else "none (90 % of free)", budget_sizes=sizes, runs=runs,
                         wall_s_median=round(float(np.median(walls[r])), 4), wall_s_min=round(min(walls[r]), 4),
                         wall_s_max=round(max(walls[r]), 4), n_groups=int(m["n_groups"]), n_loads=int(m["n_loads"]),
                         n_evictions=int(m["n_evictions"]), peak=int(m["peak"]),
                         pcie_image_bytes=int(2 * m["bytes_loaded"]) if r == "host" else 0,
                         maps_equal_host=bool(same_maps(last[r], last["host"])),
                         memory_equal_host=all(m[k] == mems["host"][k] for k in ("n_groups", "n_loads", "n_evictions", "peak"))))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    for name in a.scenes.split(","):
        rows += bench(name, a.runs)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    if not all(r.get("maps_equal_host", True) and r.get("memory_equal_host", True) for r in rows):
        raise SystemExit("a device route differs from the host route")


if __name__ == "__main__":
    main()
