"""Coarse to fine with prior state (depth, dz and view ids) against depth-only priors and a plain reconstruction.

    python tools/prior_state_bench.py [--workloads C2,C5] [--runs N] [--out FILE]

Routes, alternating in one process over every view of the workload, the maps going to CUDA tensors:
  plain:        Scene.reconstruct at level 1, as it runs today (SfM features only);
  c2f-depth-S:  level 2 first (timed on its own), then level 1 with each view's level-2 depth map as its prior
                (Scene.set_view_prior(on_device=True)) at stride S = 4 and 8;
  c2f-state-S:  the same with the level-2 depth, dz and view_ids maps as the prior (b200mvs_set_view_prior_state_device),
                so a prior seed starts from the coarser map's scaled dz and, when it has exactly nr_recon_neighbors of
                them in the level-1 global selection, its local views.
The priors are cleared before every route.  After one warm-up of each route, `runs` rounds are timed, each ending in a
device synchronise.  Printed per route: the median and min-max wall time (for c2f: the whole sequence, and level 2
alone), n_rounds, n_opt, seeds processed and successful, ms_patch_kernel, the fill of the level-1 maps and the median and
p95 relative depth error of the filled pixels against synth.depth; for the state routes the share of prior seeds that
carried local views (counted on the host from the level-2 maps by the rule of include/b200mvs.h); then the device time
of k_prior_seeds from a separate torch.profiler pass of each c2f route.  The card name and power limit are read with
nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FINE, COARSE = 1, 2


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def settings(s, level):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=level, nr_recon_neighbors=s.nr_recon_neighbors)


def run_route(sc, s, views, stride, state):
    """One timed pass: (level-2 maps or None, maps at level 1, stats of level 1, wall ms, wall ms of level 2 or None)."""
    import torch
    for v in views:
        sc.set_view_prior(v, None, 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t_coarse = coarse = None
    if stride:
        want = ("depth", "dz", "view_ids") if state else ("depth",)
        coarse, _ = sc.reconstruct(settings(s, COARSE), views, on_device=True, want=want)
        torch.cuda.synchronize()
        t_coarse = (time.perf_counter() - t0) * 1e3
        for v, m in zip(views, coarse):
            if state:
                sc.set_view_prior(v, m["depth"], stride, on_device=True, dz=m["dz"], view_ids=m["view_ids"])
            else:
                sc.set_view_prior(v, m["depth"], stride, on_device=True)
    maps, st = sc.reconstruct(settings(s, FINE), views, on_device=True, want=("depth",))
    torch.cuda.synchronize()
    return coarse, maps, st, (time.perf_counter() - t0) * 1e3, t_coarse


def quality(s, views, maps, truth):
    fill, err = [], []
    for v, m in zip(views, maps):
        d = m["depth"]
        t = truth[v]
        ok = (d > 0) & (t > 0)
        fill.append((d > 0).float().mean().item())
        err.append(((d[ok] - t[ok]).abs() / t[ok]).cpu().numpy())
    e = np.concatenate(err)
    return dict(fill=float(np.mean(fill)), err_median=float(np.median(e)), err_p95=float(np.percentile(e, 95)))


def local_share(sc, s, views, coarse, sizes, stride):
    """Of the prior seeds the level-2 maps make at level 1 (no masks), the share whose ids give exactly N local views."""
    n_seeds = n_local = 0
    N = s.nr_recon_neighbors
    for v, m in zip(views, coarse):
        depth = m["depth"].cpu().numpy()
        ids = m["view_ids"].cpu().numpy()
        h, w = depth.shape
        W, H = sizes[v]
        if W < 5 or H < 5:
            continue
        xs = np.arange(2, W - 2, stride)
        ys = np.arange(2, H - 2, stride)
        px = (2 * xs + 1) * w // (2 * W)
        py = (2 * ys + 1) * h // (2 * H)
        d = depth[np.ix_(py, px)]
        seed = np.isfinite(d) & (d > 0)
        g = np.array(sc.global_view_selection(settings(s, FINE), v), np.int32)
        q = ids[np.ix_(py, px)][seed]                             # n x 4
        q = np.sort(np.where(np.isin(q, g) & (q >= 0), q, -1), axis=1)
        inside = q >= 0
        distinct = inside.sum(1) - (inside[:, 1:] & (q[:, 1:] == q[:, :-1])).sum(1)
        n_seeds += int(seed.sum())
        n_local += int((distinct == N).sum())
    return n_local / max(1, n_seeds)


def prior_kernel_ms(sc, s, views, stride, state):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_route(sc, s, views, stride, state)
    events = [e for e in prof.events() if "k_prior_seeds" in e.name]
    return dict(launches=len(events), ms=sum(e.device_time_total for e in events) / 1e3)


def bench(name, runs):
    import torch
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    views = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    truth, sizes = {}, {}
    for v in views:
        w, h = sc.level(v, FINE, on_device=True).shape[1::-1]
        sizes[v] = (w, h)
        truth[v] = torch.from_numpy(synth.depth(s, v, w, h, device="cuda")).cuda()
    routes = {"plain": (0, False), "c2f-depth-4": (4, False), "c2f-state-4": (4, True), "c2f-depth-8": (8, False),
              "c2f-state-8": (8, True)}
    for stride, state in routes.values():
        run_route(sc, s, views, stride, state)
    rec = {k: dict(wall=[], coarse=[]) for k in routes}
    for _ in range(runs):
        for k, (stride, state) in routes.items():
            coarse, maps, st, ms, mc = run_route(sc, s, views, stride, state)
            rec[k]["wall"].append(ms)
            if mc is not None:
                rec[k]["coarse"].append(mc)
            rec[k]["stats"] = dict(n_rounds=st.n_rounds, n_opt=st.n_opt, n_seeds_processed=st.n_seeds_processed,
                                   n_seeds_success=st.n_seeds_success, ms_patch_kernel=round(st.ms_patch_kernel, 1))
            rec[k]["quality"] = quality(s, views, maps, truth)
            if state:
                rec[k]["local_share"] = round(local_share(sc, s, views, coarse, sizes, stride), 4)
    out = dict(workload=name, views=len(views), fine_level=FINE, coarse_level=COARSE, runs=runs, **card())
    for k, (stride, state) in routes.items():
        r = rec[k]
        row = dict(wall_ms_median=round(float(np.median(r["wall"])), 1), wall_ms_min=round(min(r["wall"]), 1),
                   wall_ms_max=round(max(r["wall"]), 1), **r["stats"], **r["quality"])
        if "local_share" in r:
            row["local_share"] = r["local_share"]
        if r["coarse"]:
            row.update(coarse_ms_median=round(float(np.median(r["coarse"])), 1), coarse_ms_min=round(min(r["coarse"]), 1),
                       coarse_ms_max=round(max(r["coarse"]), 1),
                       k_prior_seeds=prior_kernel_ms(sc, s, views, stride, state))
        out[k] = row
    sc.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C2,C5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prior_state_bench.py measures on a GPU; none is visible")
    results = [bench(w, a.runs) for w in a.workloads.split(",")]
    for r in results:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
