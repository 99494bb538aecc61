"""The planning phase of a one-call reconstruction (analyzeFeatures, globalViewSelection, seed lists): on host threads
against on the device.

    python tools/plan_bench.py [--scenes C2,C3,C5] [--reps 2] [--out FILE]

For each scene (images rendered on the GPU) every view is reconstructed in one call, in two routes that alternate in one
process after a warm-up call of each:
  host:   Scene.plan_views on B200MVS_HOST_THREADS = the host's cores, then Scene.reconstruct of the prepared plans;
  device: Scene.reconstruct alone, which plans its views on the device.
Per route it prints the planning wall time (host: the plan_views call; device: plan_info's ms_plan), the planning
kernels' CUDA-event time (ms_device), the wall time of the whole call (host: plan_views + reconstruct) and whether the
depth maps and view ids of the two routes are byte-identical.  The card name and power limit are read with nvidia-smi in
the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C3,C5")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from mve_b200 import dmrecon, synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures on the GPU only")
    os.environ["B200MVS_HOST_THREADS"] = str(os.cpu_count())
    rows = [dict(card(), host_threads=os.cpu_count())]
    print(json.dumps(rows[0]), flush=True)
    for name in a.scenes.split(","):
        s = synth.make_scene(name, device="cuda")
        st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
        sc = dmrecon.Scene.from_synth(s)
        refs = list(range(s.n_views))
        want = ("depth", "view_ids")

        def host():
            t0 = time.perf_counter()
            sc.plan_views(st, refs)
            t1 = time.perf_counter()
            maps, _ = sc.reconstruct(st, refs, want=want)
            t2 = time.perf_counter()
            return maps, dict(ms_plan=(t1 - t0) * 1e3, ms_device=0.0, ms_call=(t2 - t0) * 1e3, info=sc.plan_info())

        def device():
            t0 = time.perf_counter()
            maps, _ = sc.reconstruct(st, refs, want=want)
            t1 = time.perf_counter()
            info = sc.plan_info()
            return maps, dict(ms_plan=info["ms_plan"], ms_device=info["ms_device"], ms_call=(t1 - t0) * 1e3, info=info)

        host(), device()                                   # warm-up: modules, scene uploads, the factor table
        res = {"host": [], "device": []}
        equal = True
        for _ in range(a.reps):
            mh, rh = host()
            md, rd = device()
            equal &= all(x[k].tobytes() == y[k].tobytes() for x, y in zip(mh, md) for k in want)
            res["host"].append(rh)
            res["device"].append(rd)
        for route, rs in res.items():
            best = min(rs, key=lambda r: r["ms_call"])
            row = dict(scene=name, views=s.n_views, route=route, ms_plan=round(best["ms_plan"], 1),
                       ms_device=round(best["ms_device"], 2), ms_call=round(best["ms_call"], 1),
                       ms_call_all=[round(r["ms_call"], 1) for r in rs], n_device=best["info"]["n_device"],
                       n_prepared=best["info"]["n_prepared"], peak_bytes=best["info"]["peak_bytes"], maps_equal=equal)
            rows.append(row)
            print(json.dumps(row), flush=True)
        sc.close()
        del s
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
