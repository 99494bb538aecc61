"""Frontier capacity: what the frontier actually holds, and what a smaller initial capacity buys within a device budget.

    python tools/frontier_capacity.py [--out FILE] [--capacities 2,0.5,0.25] [--budget-gib 16]

1. Peak frontier entries per reference pixel (stats.n_entries_peak / pixels of level `scale`) of single-view launches,
   three views of every BASELINE scene (C2 to C5), default capacity.
2. C3, C4 and C5 (all views, lazy scene, images fetched through the image source) within the budget, once per capacity
   (entries per pixel, floor 65536): planned groups, launches, resumes, initial / final capacity, the call time (host clock
   around the synchronised call) and whether the maps equal those of the first capacity.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def peaks(name, views=3):
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    plan = dmrecon.Scene.from_synth(s, lazy=True)
    rows = []
    for v in [round(k * (s.n_views - 1) / max(1, views - 1)) for k in range(views)]:
        sc = dmrecon.Scene.from_synth(s, views=sorted(set(plan.global_view_selection(st, v)) | {v}))
        maps, stats = sc.reconstruct(st, [v], want=("depth",))
        px = maps[0]["depth"].size
        rows.append(dict(scene=name, view=v, pixels=px, peak_entries=int(stats.n_entries_peak),
                         peak_per_px=round(stats.n_entries_peak / px, 4), rounds=int(stats.n_rounds)))
        print(json.dumps(rows[-1]), flush=True)
        sc.close()
    plan.close()
    return rows


def budgeted(name, capacities, budget):
    import hashlib
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    rows, first = [], None
    for f in capacities:
        sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget)
        sc.set_frontier_capacity(f, 1 << 16)
        row = dict(scene=name, budget=budget, entries_per_px=f, working_set_1view=sc.working_set(st, [0]),
                   planned_groups=sc.plan_batches(st, refs, budget - sc.memory_stats().fixed)[0])
        try:
            t0 = time.perf_counter()
            maps, stats = sc.reconstruct(st, refs, want=("depth", "conf"))
            row["call_s"] = round(time.perf_counter() - t0, 2)
            info, m = sc.frontier_info(), sc.memory_stats()
            row.update(groups=int(m.n_groups), launches=int(stats.n_patch_launches), resumes=info["resumes"],
                       initial_entries=info["initial"], final_entries=info["final"], peak_bytes=int(m.peak),
                       kernel_ms=round(stats.ms_patch_kernel, 1), rounds=int(stats.n_rounds), filled=int(stats.n_filled))
            h = hashlib.sha256()
            for mp in maps:
                h.update(mp["depth"].tobytes())
                h.update(mp["conf"].tobytes())
            digest = h.hexdigest()
            first = first or digest
            row["maps_equal_first"] = digest == first
        except dmrecon.B200MVSError as e:            # the outcome is the measurement
            row["error"] = str(e)
        print(json.dumps(row), flush=True)
        rows.append(row)
        sc.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--capacities", default="2,0.5,0.25")
    ap.add_argument("--budget-gib", type=float, default=16.0)
    ap.add_argument("--scenes", default="C3,C4,C5")
    a = ap.parse_args()
    import torch
    props = torch.cuda.get_device_properties(0)
    rows = [dict(gpu=props.name, total_bytes=props.total_memory)]
    for name in ("C2", "C3", "C4", "C5"):
        rows += peaks(name)
    caps = [float(x) for x in a.capacities.split(",")]
    for name in a.scenes.split(","):
        rows += budgeted(name, caps, int(a.budget_gib * (1 << 30)))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
