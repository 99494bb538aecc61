"""Relative priors: the device fit and install against a host route, and what an aligned monocular prior does to a
reconstruction.

    python tools/prior_align_bench.py [--workloads C2,C5] [--runs N] [--stride S] [--out FILE]

The prior of every view is synth.monocular: the planar disparity of synth.depth at 1/4 of the photo's size under a
seeded affine transform, with 2 % multiplicative noise and 5 % of the pixels in outlier discs, held as a CUDA tensor.
  (a) install, over every view of the workload:
      device: Scene.set_view_prior_relative(v, tensor) - observations, fit and apply on the GPU (b200mvs_set_view_prior_
              relative_device);
      host:   tensor.cpu(), the NumPy fit and apply of tests/prior_align_reference.py (each view's feature positions
              gathered beforehand, as a caller holds them), then Scene.set_view_prior(on_device=True) of the result.
  (b) reconstruction at level 1, maps to CUDA tensors:
      plain:  no prior (SfM features only);
      mono:   the aligned monocular prior at stride S;
      depth:  synth.depth at the map's size as the prior at stride S, the best a prior can be.
The routes of each part alternate in one process: one warm-up of each, then `runs` rounds, each route ending in a device
synchronise.  Printed per route: the median and min-max wall time; for (b) n_rounds, the fill of the maps and the median
and p95 relative depth error of the filled pixels against synth.depth; for (a) the largest difference between the two
routes' s and t.  The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host
is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LEVEL = 1


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def spread(ms):
    return dict(ms_median=round(float(np.median(ms)), 2), ms_min=round(min(ms), 2), ms_max=round(max(ms), 2))


def install_device(sc, views, mono):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fits = [sc.set_view_prior_relative(v, mono[v], 4) for v in views]
    torch.cuda.synchronize()
    return fits, (time.perf_counter() - t0) * 1e3


def install_host(sc, views, mono, cams, feats):
    import torch
    from tests import prior_align_reference as ref
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fits = []
    for v in views:
        values = mono[v].cpu().numpy()
        d, y, _, _ = ref.observations(cams[v], feats[v], values, ref.DISPARITY)
        f = ref.fit(d, y, ref.DISPARITY)
        depth = ref.apply(cams[v], values, ref.DISPARITY, f["scale"], f["shift"])
        sc.set_view_prior(v, torch.from_numpy(depth).cuda(), 4, on_device=True)
        fits.append(f)
    torch.cuda.synchronize()
    return fits, (time.perf_counter() - t0) * 1e3


def reconstruct(sc, s, views, prior, stride, mono, exact):
    import torch
    from mve_b200 import dmrecon
    for v in views:
        if prior == "mono":
            sc.set_view_prior_relative(v, mono[v], stride)
        elif prior == "depth":
            sc.set_view_prior(v, exact[v], stride, on_device=True)
        else:
            sc.set_view_prior(v, None, stride)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    maps, st = sc.reconstruct(dmrecon.Settings(scale=LEVEL, nr_recon_neighbors=s.nr_recon_neighbors), views,
                              on_device=True, want=("depth",))
    torch.cuda.synchronize()
    return maps, st, (time.perf_counter() - t0) * 1e3


def quality(views, maps, truth):
    fill, err = [], []
    for v, m in zip(views, maps):
        d, t = m["depth"], truth[v]
        ok = (d > 0) & (t > 0)
        fill.append((d > 0).float().mean().item())
        err.append(((d[ok] - t[ok]).abs() / t[ok]).cpu().numpy())
    e = np.concatenate(err)
    return dict(fill=round(float(np.mean(fill)), 4), err_median=float(np.median(e)), err_p95=float(np.percentile(e, 95)))


def bench(name, runs, stride):
    import torch
    from mve_b200 import dmrecon, synth
    from tests import prior_align_reference as ref
    s = synth.make_scene(name, device="cuda")
    views = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    mono, exact, truth, cams, feats = {}, {}, {}, {}, {}
    for v in views:
        W0, H0 = s.size(v)
        mono[v] = torch.from_numpy(synth.monocular(s, v, W0 // 4, H0 // 4, seed=v)).cuda()
        w, h = sc.level(v, LEVEL, on_device=True).shape[1::-1]
        exact[v] = torch.from_numpy(synth.depth(s, v, w, h, device="cuda")).cuda()
        truth[v] = exact[v]
        cams[v] = ref.camera(s, v)
        feats[v] = ref.view_features(s, v)
    n_features = sum(len(f) for f in feats.values())
    # (a) install
    install_device(sc, views, mono)
    install_host(sc, views, mono, cams, feats)
    a = dict(device=[], host=[])
    for _ in range(runs):
        fd, ms = install_device(sc, views, mono)
        a["device"].append(ms)
        fh, ms = install_host(sc, views, mono, cams, feats)
        a["host"].append(ms)
    diff = max(max(abs(x["scale"] - y["scale"]) / y["scale"], abs(x["shift"] - y["shift"]) / y["scale"])
               for x, y in zip(fd, fh))
    # (b) reconstruction
    routes = ("plain", "mono", "depth")
    for r in routes:
        reconstruct(sc, s, views, r, stride, mono, exact)
    b = {r: dict(wall=[]) for r in routes}
    for _ in range(runs):
        for r in routes:
            maps, st, ms = reconstruct(sc, s, views, r, stride, mono, exact)
            b[r]["wall"].append(ms)
            b[r]["n_rounds"] = st.n_rounds
            b[r]["quality"] = quality(views, maps, truth)
    out = dict(workload=name, views=len(views), features_per_view=round(n_features / len(views), 1), level=LEVEL,
               stride=stride, runs=runs, **card())
    out["install"] = dict(device=spread(a["device"]), host=spread(a["host"]), max_rel_diff_s_t=diff,
                          inliers=[f["n_inliers"] for f in fd], obs=[f["n_obs"] for f in fd])
    for r in routes:
        out[r] = dict(**spread(b[r]["wall"]), n_rounds=b[r]["n_rounds"], **b[r]["quality"])
    sc.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C2,C5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--stride", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prior_align_bench.py measures on a GPU; none is visible")
    results = [bench(w, a.runs, a.stride) for w in a.workloads.split(",")]
    for r in results:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
