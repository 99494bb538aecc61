"""Views built from their original photos: the cost of undistorting on the device, against the reference on the host.

    python tools/undistort_bench.py [--sets 16x1920x1080,32x4096x3072] [--runs N] [--out FILE]

For each set of seeded 3-channel photos (typical coefficients: k2 in [-0.08, 0.08], k4 in [-0.01, 0.01], flen 0.9-1.3):
  pyramid:   CUDA-event time of every view's pyramid build (Scene.set_view_device from photos already in device memory, so
             the events bracket k_undistort_k2k4 or k_import_rgb, the half-size levels and the quads only), with and
             without the coefficients, `runs` times after a warm-up; the median total over the set;
  upload:    wall time of Scene.set_view (host photo -> pinned staging -> device -> pyramid) per view, ending in a device
             synchronise, with and without the coefficients;
  reference: oracle/_ref/undistort_harness over the same photos and coefficients on all host threads, the time of
             the undistortion alone (read from MVEI files first), when that binary was built.
Level 0 of the first view of each set is checked against tests/undistort_reference.py.  The
card name and power limit are read with nvidia-smi in the same run.  Nothing on the GPU or the host is reconfigured."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HARNESS = os.path.join(ROOT, "oracle", "_ref", "undistort_harness")
CAM = dict(paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3, dtype=np.float32), trans=np.zeros(3, np.float32))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else ("unknown", "unknown")
    return dict(gpu=name, power_limit=power)


def photos(n, w, h, seed):
    rng = np.random.default_rng(seed)
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for _ in range(n)]
    coef = [(float(np.float32(rng.uniform(-0.08, 0.08))), float(np.float32(rng.uniform(-0.01, 0.01))),
             float(np.float32(rng.uniform(0.9, 1.3)))) for _ in range(n)]
    return imgs, coef


def pyramid_ms(sc, dev, coef, w, h, runs, undistort):
    import torch
    stream = torch.cuda.current_stream()
    for v, (k2, k4, flen) in enumerate(coef):
        sc.set_view_distortion(v, k2 if undistort else 0.0, k4 if undistort else 0.0)
        sc.set_view_device(v, dev[v].data_ptr(), w, h, flen, stream=stream.cuda_stream, **CAM)     # warm-up + allocation
    totals = []
    for _ in range(runs):
        t = 0.0
        for v, (k2, k4, flen) in enumerate(coef):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            sc.set_view_device(v, dev[v].data_ptr(), w, h, flen, stream=stream.cuda_stream, **CAM)
            b.record(stream)
            b.synchronize()
            t += a.elapsed_time(b)
        totals.append(t)
    return totals


def upload_s(sc, imgs, coef, runs, undistort):
    import torch
    for v, (k2, k4, flen) in enumerate(coef):
        sc.set_view_distortion(v, k2 if undistort else 0.0, k4 if undistort else 0.0)
        sc.set_view(v, imgs[v], flen, **CAM)
    torch.cuda.synchronize()
    per_view = []
    for _ in range(runs):
        for v, (k2, k4, flen) in enumerate(coef):
            t0 = time.perf_counter()
            sc.set_view(v, imgs[v], flen, **CAM)
            torch.cuda.synchronize()
            per_view.append(time.perf_counter() - t0)
    return per_view


def reference_s(imgs, coef):
    if not os.path.exists(HARNESS):
        return None
    from mve_b200 import synth
    with tempfile.TemporaryDirectory(prefix="undistort_bench_") as tmp:
        args = []
        for v, (k2, k4, flen) in enumerate(coef):
            p = os.path.join(tmp, "p%d.mvei" % v)
            synth.write_mvei(p, imgs[v])
            args += [p, "-", repr(flen), repr(k2), repr(k4)]
        r = subprocess.run([HARNESS] + args, capture_output=True, text=True, check=True)
        return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", default="16x1920x1080,32x4096x3072")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from mve_b200 import dmrecon
    from tests import undistort_reference as UR
    res = dict(card(), host_threads=os.cpu_count(), sets=[])
    for k, spec in enumerate(a.sets.split(",")):
        n, w, h = (int(x) for x in spec.split("x"))
        imgs, coef = photos(n, w, h, 100 + k)
        sc = dmrecon.Scene(n)
        dev = [torch.from_numpy(im).cuda() for im in imgs]
        plain = pyramid_ms(sc, dev, coef, w, h, a.runs, False)
        und = pyramid_ms(sc, dev, coef, w, h, a.runs, True)
        k2, k4, flen = coef[0]
        ok = sc.level(0, 0).tobytes() == UR.undistort_k2k4(imgs[0], flen, k2, k4).tobytes()
        del dev
        up_plain = upload_s(sc, imgs, coef, a.runs, False)
        up_und = upload_s(sc, imgs, coef, a.runs, True)
        sc.close()
        ref = reference_s(imgs, coef)
        row = dict(views=n, width=w, height=h, level0_equals_restatement=ok,
                   pyramid_ms_plain=float(np.median(plain)), pyramid_ms_undistort=float(np.median(und)),
                   pyramid_ms_spread=[float(min(und)), float(max(und))],
                   undistort_extra_ms_per_view=float((np.median(und) - np.median(plain)) / n),
                   upload_view_ms_plain=1e3 * float(np.median(up_plain)), upload_view_ms_undistort=1e3 * float(np.median(up_und)),
                   reference=ref)
        res["sets"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
