"""One reconstruction call with a pyramid level per entry against one call per level.

    python tools/levels_bench.py [--workloads mixed,multi,budget] [--runs N] [--out FILE]

Two routes alternate in one process over the same entries (reference view, level):
  levels:    one Scene.reconstruct(..., scales=levels) (b200mvs_reconstruct_levels);
  per-level: one Scene.reconstruct at settings.scale = l for each distinct level l, over that level's entries, in turn.
Workloads:
  mixed:  C2's configuration with views alternating 1920x1080 and 960x540; the levels of apps/dmrecon --max-pixels=1500000
          (1 and 0, so every map is 960x540).  Images resident, no budget.
  multi:  all 16 C2 views at levels 1 and 2 (32 entries).  Images resident, no budget.
  budget: C5 (128 views of 1280x960) at levels 0 and 1 (256 entries) on a fresh context per route and round (the
          per-level route's two calls share it) whose images are fetched through a host image source under a budget of
          fixed + max(largest single-entry working set, working set of all entries / 4) (b200mvs_working_set_levels), the
          rule of DESIGN.md section 8.
The maps (depth, conf, dz) go to CUDA tensors (reconstruct(on_device=True)).  After one warm-up of each route, `runs`
rounds of the two routes are timed, each ending in a device synchronise.  Printed per route: the median and min-max wall
time, ms_patch_kernel, n_rounds, n_loads and n_groups (summed over the calls of the per-level route), and whether every
map of the levels route is bit-identical to the per-level route's.  The card name and power limit are read with nvidia-smi
in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MAPS = ("depth", "conf", "dz")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def max_pixels_level(w, h, max_pixels=1500000):
    """apps/dmrecon get_scale_from_max_pixels (dmrecon.cc:89-111)."""
    if w * h <= max_pixels:
        return 0
    return max(0, int(math.ceil(math.log(np.float32(w * h) / np.float32(max_pixels)) / math.log(4.0))))


def workload(name):
    """(scene, settings, views, levels, budgeted)"""
    from mve_b200 import dmrecon, synth
    if name == "mixed":
        sizes = [(1920, 1080) if v % 2 == 0 else (960, 540) for v in range(16)]
        s = synth.make_scene("C2", device="cuda", sizes=sizes)
        views = list(range(s.n_views))
        levels = [max_pixels_level(*s.size(v)) for v in views]
        budgeted = False
    elif name == "multi":
        s = synth.make_scene("C2", device="cuda")
        views = [v for v in range(s.n_views) for _ in (1, 2)]
        levels = [1 + (k % 2) for k in range(len(views))]
        budgeted = False
    else:
        s = synth.make_scene("C5", device="cuda")
        views = [v for v in range(s.n_views) for _ in (0, 1)]
        levels = [k % 2 for k in range(len(views))]
        budgeted = True
    st = dmrecon.Settings(scale=0, nr_recon_neighbors=s.nr_recon_neighbors)
    return s, st, views, levels, budgeted


def budget_for(s, st, views, levels):
    from mve_b200 import dmrecon
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    single = max(sc.working_set(st, [v], scales=[l]) for v, l in zip(views, levels))
    total = sc.working_set(st, views, scales=levels)
    sc.close()
    return fixed + max(single, total // 4), dict(fixed=fixed, largest_single=single, all_entries=total)


def run(sc, s, st, views, levels, route):
    """One route on context sc: (wall seconds, maps in entry order, dict of counters summed over the route's calls)."""
    import torch
    calls = [(list(range(len(views))), levels)] if route == "levels" else \
        [([j for j in range(len(views)) if levels[j] == l], None) for l in sorted(set(levels))]
    maps = [None] * len(views)
    tot = dict(ms_patch_kernel=0.0, n_rounds=0, n_loads=0, n_groups=0)
    loads0 = sc.memory_stats().n_loads
    groups = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for idx, lv in calls:
        if lv is None:
            st_l = type(st).from_buffer_copy(st)
            st_l.scale = levels[idx[0]]
            got, stt = sc.reconstruct(st_l, [views[j] for j in idx], want=MAPS, on_device=True)
        else:
            got, stt = sc.reconstruct(st, views, want=MAPS, on_device=True, scales=lv)
        groups += sc.memory_stats().n_groups
        for j, m in zip(idx, got):
            maps[j] = m
        tot["ms_patch_kernel"] += stt.ms_patch_kernel
        tot["n_rounds"] += stt.n_rounds
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    tot["n_loads"] = sc.memory_stats().n_loads - loads0
    tot["n_groups"] = groups
    return wall, maps, tot


def same_maps(a, b):
    import torch
    return all(torch.equal(x[k].view(torch.int32), y[k].view(torch.int32)) for x, y in zip(a, b) for k in MAPS)


def bench(name, runs):
    from mve_b200 import dmrecon
    s, st, views, levels, budgeted = workload(name)
    row = dict(workload=name, entries=len(views), levels=sorted(set(levels)))
    if budgeted:
        budget, parts = budget_for(s, st, views, levels)
        row.update(budget=budget, **parts)

        def sc_of():
            sc = dmrecon.Scene.from_synth(s, lazy=True)
            sc.set_image_source(lambda v: s.images[v], budget)
            return sc
    else:
        shared = dmrecon.Scene.from_synth(s)

        def sc_of():
            return shared
    walls = {"levels": [], "per-level": []}
    last = {}
    equal = True
    for k in range(runs + 1):
        out = {}
        for route in ("levels", "per-level"):
            sc = sc_of()
            wall, maps, tot = run(sc, s, st, views, levels, route)
            out[route] = maps
            if budgeted:
                sc.close()
            if k > 0:                                # round 0 warms up both routes
                walls[route].append(wall)
                last[route] = tot
        equal = equal and same_maps(out["levels"], out["per-level"])
        del out
    for route in walls:
        w = sorted(walls[route])
        row[route] = dict(wall_s_median=round(float(np.median(w)), 4), wall_s_min=round(w[0], 4), wall_s_max=round(w[-1], 4),
                          ms_patch_kernel=round(last[route]["ms_patch_kernel"], 1), n_rounds=int(last[route]["n_rounds"]),
                          n_loads=int(last[route]["n_loads"]), n_groups=int(last[route]["n_groups"]))
    row["maps_equal"] = "yes" if equal else "no"
    if not budgeted:
        shared.close()
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mixed,multi,budget")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    for name in a.workloads.split(","):
        rows.append(bench(name, a.runs))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
