"""dmrecon + scene2pset through host memory against the one-call path that keeps the maps on the device.

    python tools/recon_pset_bench.py [--scenes C2,C5] [--out FILE]

For each BASELINE scene (C2 runs at its scale 1, C5 at scale 0), with the -F option set (normals, confidences, scale values
and colours from the level image):
  route a: Scene.reconstruct with host maps (depth only), Scene.level for every view's level-`scale` colour image, then
           depthmap.scene_pointset of the maps with those images and the registered cameras;
  route b: Scene.reconstruct_pointset (b200mvs_pset_add_reconstruction).
Each route runs in a fresh process of its own (so its peak RSS is its own): the scene is made and uploaded, the route runs
once to warm up and once timed.  Printed per route: wall time of the timed run, bytes over PCIe that the route itself moves
(computed from the shapes: maps and level images down, maps and colours up again, the points down), the process' peak RSS
and its RSS just before the timed run (the scene's images are in both).  The point sets of a and b must be byte-identical.
The card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OPTIONS = dict(with_normals=True, with_conf=True, with_scale=True)
ARRAYS = ("vertices", "normals", "colors", "values", "confidences")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def rss_now_mb():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) / 1024.0
    return float("nan")


def route_a(sc, s, st, refs):
    from mve_b200 import depthmap as D
    maps, _ = sc.reconstruct(st, refs, want=("depth",))
    views, pcie = [], 0
    for j, v in enumerate(refs):
        img = sc.level(v, st.scale)
        d = maps[j]["depth"]
        views.append(dict(id=v, depth=d, color=img, camera=dict(flen=s.flen[v], paspect=s.paspect[v], ppoint=s.ppoint[v],
                                                                 rot=s.rot[v], trans=s.trans[v])))
        pcie += 2 * (d.nbytes + img.nbytes)          # down after dmrecon, up again for scene2pset
    r = D.scene_pointset(views, OPTIONS)
    return r, pcie


def route_b(sc, s, st, refs):
    r, _ = sc.reconstruct_pointset(st, refs, OPTIONS)
    return r, 0


def child(name, route, out):
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(name, device="cuda")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    sc = dmrecon.Scene.from_synth(s)
    refs = list(range(s.n_views))
    fn = route_a if route == "a" else route_b
    fn(sc, s, st, refs)                                  # warm-up
    rss0 = rss_now_mb()
    t0 = time.perf_counter()
    r, pcie = fn(sc, s, st, refs)
    dt = time.perf_counter() - t0
    pcie += sum(r[k].nbytes for k in ARRAYS if r[k] is not None)
    np.savez(out, **{k: r[k] for k in ARRAYS if r[k] is not None})
    sc.close()
    print(json.dumps(dict(scene=name, route=route, views=s.n_views, scale=s.scale, points=int(len(r["vertices"])),
                          wall_s=round(dt, 4), pcie_bytes=int(pcie), rss_before_mb=round(rss0, 1),
                          peak_rss_mb=round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C2,C5")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", nargs=3, metavar=("SCENE", "ROUTE", "NPZ"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(*a.child)
        return
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    with tempfile.TemporaryDirectory(prefix="recon_pset_bench_") as tmp:
        for name in a.scenes.split(","):
            res = {}
            for route in ("a", "b"):
                npz = os.path.join(tmp, "%s_%s.npz" % (name, route))
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, route, npz],
                                   capture_output=True, text=True)
                if p.returncode != 0:
                    raise RuntimeError(p.stdout + p.stderr)
                row = json.loads(p.stdout.strip().splitlines()[-1])
                res[route] = np.load(npz)
                rows.append(row)
                print(json.dumps(row), flush=True)
            equal = sorted(res["a"].files) == sorted(res["b"].files) and \
                all(res["a"][k].tobytes() == res["b"][k].tobytes() for k in res["a"].files)
            rows.append(dict(scene=name, point_sets_equal=bool(equal)))
            print(json.dumps(rows[-1]), flush=True)
            if not equal:
                raise SystemExit("route a and route b differ on %s" % name)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
