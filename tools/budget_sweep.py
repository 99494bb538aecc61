"""Device-budget sweep: one b200mvs_reconstruct of a whole scene at budgets that split it into a given number of launches.

    python tools/budget_sweep.py [--out FILE]

C2 (16 views) at budgets that give 1, 2, 4 and 16 groups, and C4 (32 views) at 16 GiB.  Every run uses a lazy scene (cameras
registered, images fetched through the image source) and reports the call time (host clock around the synchronised call),
groups, image loads, bytes loaded, evictions and the peak of the accounted device bytes.  Splitting costs one region-growing
tail per launch (DESIGN.md section 7), plus re-fetching images a later group needs again.
With --parent C4, the same C4 call is made once without a source (the unbounded path) and its outcome is reported.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _budget_for(sc, st, refs, groups):
    """Smallest budget (in MiB steps above the largest single view) that plans into at most `groups` launches."""
    fixed = sc.memory_stats().fixed
    total = sc.working_set(st, refs)
    single = max(sc.working_set(st, [r]) for r in refs)
    if groups == 1:
        return fixed + total
    if groups >= len(refs):
        return fixed + single
    lo, hi = single, total
    while hi - lo > (1 << 20):
        mid = (lo + hi) // 2
        if sc.plan_batches(st, refs, mid)[0] <= groups:
            hi = mid
        else:
            lo = mid
    return fixed + hi


def run(name, budgets, device="cuda"):
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device=device)
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    out = []
    for tag, want_groups, budget in budgets:
        sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget or (16 << 30))
        if budget is None:
            budget = _budget_for(sc, st, refs, want_groups)
            sc.set_image_source(lambda v: s.images[v], budget)
        t0 = time.perf_counter()
        _, stats = sc.reconstruct(st, refs)
        ms = (time.perf_counter() - t0) * 1e3
        m = sc.memory_stats()
        row = dict(scene=name, tag=tag, budget=budget, working_set=sc.working_set(st, refs), fixed=m.fixed,
                   groups=m.n_groups, loads=m.n_loads, bytes_loaded=m.bytes_loaded, evictions=m.n_evictions, peak=m.peak,
                   call_ms=round(ms, 1), kernel_ms=round(stats.ms_patch_kernel, 1), rounds=int(stats.n_rounds),
                   filled=int(stats.n_filled))
        print(json.dumps(row), flush=True)
        out.append(row)
        sc.close()
    return out


def parent_c4(device="cuda"):
    """C4 with all 32 views in one call without a source: every pyramid resident and one launch whatever its size."""
    from mve_b200 import dmrecon, synth
    s = synth.make_scene("C4", device=device)
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    row = dict(scene="C4", tag="no source")
    try:
        sc = dmrecon.Scene.from_synth(s)
        row["working_set"] = sc.working_set(st, list(range(s.n_views)))
        t0 = time.perf_counter()
        sc.reconstruct(st, list(range(s.n_views)))
        row.update(ok=True, call_ms=round((time.perf_counter() - t0) * 1e3, 1), peak=sc.memory_stats().peak)
        sc.close()
    except Exception as e:                      # the outcome is the measurement
        row.update(ok=False, error=str(e))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--parent", action="store_true", help="also run C4 without a source")
    a = ap.parse_args()
    import torch
    props = torch.cuda.get_device_properties(0)
    rows = [dict(gpu=props.name, total_bytes=props.total_memory)]
    rows += run("C2", [("1 group", 1, None), ("2 groups", 2, None), ("4 groups", 4, None), ("16 groups", 16, None)])
    rows += run("C4", [("16 GiB", 0, 16 << 30)])
    if a.parent:
        rows.append(parent_c4())
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
