"""Kernel-variant bench (runs on the GPU box): one C2 step (pyramids resident) per library variant.

    python tools/kbench.py [--steps 3] lib_a.so lib_b.so ...     # each in its own process through B200MVS_LIB
    python tools/kbench.py --build "256 2" "192 2" ...            # cross-compile variants into build_variants/ (here, no GPU)
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VAR = os.path.join(ROOT, "build_variants")


def build(cfgs):
    os.makedirs(VAR, exist_ok=True)
    for cfg in cfgs:
        parts = cfg.split()
        tpb, minb = parts[0], parts[1]
        extra = parts[2:]
        out = os.path.join(VAR, "lib_%s_%s%s.so" % (tpb, minb, "".join("_" + e.replace("-D", "").replace("=", "") for e in extra)))
        cmd = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
               "-shared", "-DOPT_TPB=" + tpb, "-DOPT_MIN_BLOCKS=" + minb] + extra + ["-o", out, os.path.join(ROOT, "mve_b200", "csrc", "b200mvs.cu"), os.path.join(ROOT, "mve_b200", "csrc", "depthmap.cu")]
        subprocess.check_call(cmd)
        print(out)


def run_one(steps, workload, nviews=16):
    import torch
    from mve_b200 import dmrecon, synth
    s = synth.make_scene(workload, device="cuda")
    g = dmrecon.Scene.from_synth(s)
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(min(nviews, s.n_views)))
    g.reconstruct(st, refs, download=False)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ms, opt, filled, thr, srt = [], [], 0, [], []
    for _ in range(steps):
        flush.zero_()
        torch.cuda.synchronize()
        _, stt = g.reconstruct(st, refs, download=False)
        ms.append(stt.ms_total_device); opt.append(stt.ms_optimise_phases); filled = int(stt.n_filled)
        thr.append(stt.ms_optimise_thread_phases); srt.append(stt.ms_sort_phases)
    out = dict(lib=os.environ.get("B200MVS_LIB", "default"), ms=min(ms), ms_all=ms, optimise_ms=min(opt), optimise_thread_ms=min(thr), sort_ms=min(srt), filled=filled,
               rounds=int(stt.n_rounds), n_opt=int(stt.n_opt), sets=int(stt.n_sample_sets))
    print(json.dumps(out), flush=True)


def main():
    a = sys.argv[1:]
    if a and a[0] == "--build":
        return build(a[1:])
    if a and a[0] == "--one":
        return run_one(int(a[1]), a[2], int(a[3]) if len(a) > 3 else 16)
    steps, workload, nviews = 3, "C2", 16
    while a and a[0].startswith("--"):
        if a[0] == "--steps":
            steps = int(a[1]); a = a[2:]
        elif a[0] == "--workload":
            workload = a[1]; a = a[2:]
        elif a[0] == "--views":
            nviews = int(a[1]); a = a[2:]
        else:
            raise SystemExit("unknown option " + a[0])
    for lib in a or ["default"]:
        env = dict(os.environ)
        if lib != "default":
            env["B200MVS_LIB"] = os.path.abspath(lib)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", str(steps), workload, str(nviews)], env=env, capture_output=True, text=True)
        print(r.stdout.strip() or r.stderr[-800:], flush=True)


if __name__ == "__main__":
    main()
