"""Depth maps for a PyTorch caller on the GPU: through host memory against Scene.reconstruct(on_device=True).

    python tools/device_maps_bench.py [--scene C2] [--reps 5] [--out FILE]

One process, one scene (C2: 16 views of 1920x1080 at scale 1), every map (depth, conf, dz, normal, view_ids):
  host:   Scene.reconstruct into pinned host arrays, then every map to the GPU (.cuda(non_blocking=True), synchronised);
  device: Scene.reconstruct(on_device=True) (b200mvs_reconstruct_device), the maps written straight into CUDA tensors.
Both routes run once to warm up, then alternate `reps` times; the best wall time of each is printed with the bytes the
route moves over PCIe (computed from the map shapes: down after dmrecon, up again), and the maps of the two routes must be
byte-identical.  A separate pass under torch.profiler gives the kernel time of k_slots_to_ids (the library launches it on
its own stream, so caller-side CUDA events cannot bracket it alone).  The card name and power limit are read with
nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MAPS = ("depth", "conf", "dz", "normal", "view_ids")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="C2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from mve_b200 import dmrecon, synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures on the GPU only")
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    s = synth.make_scene(a.scene, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    refs = list(range(s.n_views))
    dev = torch.device("cuda:%d" % sc.device)

    # pinned host arrays for the host route, allocated once
    shapes = []
    for r in refs:
        h, w = sc.level(r, st.scale).shape[:2]
        shapes.append(dict(depth=(h, w), conf=(h, w), dz=(h, w, 2), normal=(h, w, 3), view_ids=(h, w, 4)))
    pinned = [{k: torch.empty(sh[k], dtype=torch.int32 if k == "view_ids" else torch.float32, pin_memory=True) for k in MAPS}
              for sh in shapes]
    pcie = 2 * sum(t.numel() * t.element_size() for d in pinned for t in d.values())

    def host_route():
        sc.reconstruct(st, refs, out=[{k: t.numpy() for k, t in d.items()} for d in pinned])
        maps = [{k: t.to(dev, non_blocking=True) for k, t in d.items()} for d in pinned]
        torch.cuda.synchronize(dev)
        return maps

    def device_route():
        maps, _ = sc.reconstruct(st, refs, on_device=True)
        torch.cuda.synchronize(dev)
        return maps

    routes = dict(host=host_route, device=device_route)
    results = {k: f() for k, f in routes.items()}                  # warm-up, and the maps to compare
    equal = all(results["host"][j][k].cpu().numpy().tobytes() == results["device"][j][k].cpu().numpy().tobytes()
                for j in range(len(refs)) for k in MAPS)
    del results
    best = dict(host=float("inf"), device=float("inf"))
    for _ in range(a.reps):
        for name, f in routes.items():
            t0 = time.perf_counter()
            f()
            best[name] = min(best[name], time.perf_counter() - t0)

    from torch.profiler import ProfilerActivity, profile
    from torch.autograd import DeviceType
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        device_route()
    slots = [e for e in prof.events() if "k_slots_to_ids" in e.name and e.device_type == DeviceType.CUDA]
    slots_ms = sum(e.device_time_total for e in slots) / 1000.0

    px = sum(sh["depth"][0] * sh["depth"][1] for sh in shapes)
    rows.append(dict(scene=a.scene, views=s.n_views, scale=s.scale, pixels=int(px), reps=a.reps,
                     host_s=round(best["host"], 4), device_s=round(best["device"], 4),
                     host_pcie_bytes=int(pcie), device_pcie_bytes=0, maps_equal=bool(equal),
                     k_slots_to_ids_launches=len(slots), k_slots_to_ids_ms=round(slots_ms, 4),
                     view_ids_bytes_written=int(16 * px)))
    print(json.dumps(rows[-1]), flush=True)
    sc.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    if not equal:
        raise SystemExit("the host and device routes differ")


if __name__ == "__main__":
    main()
