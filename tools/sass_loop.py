"""SASS report of the thread-per-patch sample loop of k_frontier (sm_90a, no GPU needed).

    python tools/sass_loop.py                      # compile mve_b200/csrc/b200mvs.cu of this tree for sm_90a
    python tools/sass_loop.py --cu OTHER/b200mvs.cu -DFOO   # another tree / extra nvcc flags
    python tools/sass_loop.py --cubin lib.cubin    # an existing cubin (no ptxas spill figures)
    python tools/sass_loop.py --json               # one JSON line instead of the table

Prints the registers, spill bytes and stack frame of k_frontier and, for the sample loop, the SASS instruction count and
its mix.  The sample loop is the smallest loop (a backward branch and the code from its target up to it) that holds at least
one 128-bit global load - the quad texel of a sample - and 15 shared-memory loads per such load - the table look-ups.
One quad load per sample, so samples per iteration = 128-bit global loads in the loop body.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
KERNEL = "k_frontier"
# the device-code flags of mve_b200/build.py (the host-side -shared / -fPIC do not change the cubin)
NVCC_DEVICE_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17"]

INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);")
MOVES = ("MOV", "IMAD.MOV", "IMAD.MOV.U32")      # register-to-register copies of the vector datapath
CONTROL = ("BRA", "BSSY", "BSYNC", "BREAK", "BRX", "JMP", "JMX", "CALL", "RET", "EXIT", "WARPSYNC", "BPT")


def compile_cubin(cu, extra, out_dir):
    cubin = os.path.join(out_dir, "b200mvs.cubin")
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + NVCC_DEVICE_FLAGS + ["-cubin", "-Xptxas", "-v"] + extra + ["-o", cubin, cu]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise SystemExit("nvcc failed")
    return cubin, res.stderr


def ptxas_usage(log, kernel):
    """registers, spill stores, spill loads, stack frame of `kernel` from `-Xptxas -v` output"""
    lines = log.splitlines()
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and kernel in ln:
            block = "\n".join(lines[i:i + 4])
            st = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
            rg = re.search(r"Used (\d+) registers", block)
            return dict(registers=int(rg.group(1)), stack_frame=int(st.group(1)), spill_stores=int(st.group(2)),
                        spill_loads=int(st.group(3)))
    raise SystemExit("no ptxas record for " + kernel)


def res_usage(cubin, kernel):
    out = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", cubin], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    for i, ln in enumerate(lines):
        if ln.strip().startswith("Function") and kernel in ln:
            rg = re.search(r"REG:(\d+)", lines[i + 1])
            st = re.search(r"STACK:(\d+)", lines[i + 1])
            return dict(registers=int(rg.group(1)), stack_frame=int(st.group(1)), spill_stores=None, spill_loads=None)
    raise SystemExit("no resource record for " + kernel)


def kernel_sass(cubin, kernel):
    out = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], capture_output=True, text=True, check=True).stdout
    insns, inside = [], False
    for ln in out.splitlines():
        if ln.strip().startswith("Function :"):
            inside = kernel in ln
            continue
        if inside:
            m = INSN.search(ln)
            if m:
                insns.append((int(m.group(1), 16), m.group(2) or "", m.group(3), m.group(4).strip()))
    if not insns:
        raise SystemExit("no SASS for " + kernel)
    return insns


def op_base(op):
    return op.split(".")[0]


def is_quad_load(op):
    return op_base(op) == "LDG" and ".128" in op


def sample_loop(insns):
    """(first index, last index) of the smallest loop whose body holds >= 1 quad load and 15 LDS per quad load"""
    addr = {a: i for i, (a, _, _, _) in enumerate(insns)}
    best = None
    for j, (a, _, op, args) in enumerate(insns):
        if op_base(op) != "BRA":
            continue
        m = re.match(r"`?\(?(0x[0-9a-f]+)", args.strip())
        if not m:
            continue
        t = int(m.group(1), 16)
        if t > a or t not in addr:
            continue
        i = addr[t]
        body = insns[i:j + 1]
        nq = sum(is_quad_load(o) for _, _, o, _ in body)
        nlds = sum(op_base(o) == "LDS" for _, _, o, _ in body)
        if nq >= 1 and nlds >= 15 * nq and (best is None or j - i < best[1] - best[0]):
            best = (i, j)
    if best is None:
        raise SystemExit("sample loop not found")
    return best


def report(usage, insns):
    i, j = sample_loop(insns)
    body = insns[i:j + 1]
    n = len(body)
    samples = sum(is_quad_load(o) for _, _, o, _ in body)
    count = lambda pred: sum(1 for _, _, o, _ in body if pred(o))
    moves = count(lambda o: o in MOVES or o.startswith("IMAD.MOV"))
    control = [(a, p.strip(), o) for a, p, o, _ in body if op_base(o) in CONTROL]
    mix = {}
    for _, _, o, _ in body:
        mix[op_base(o)] = mix.get(op_base(o), 0) + 1
    return dict(kernel=KERNEL, **usage, loop_start=hex(body[0][0]), loop_end=hex(body[-1][0]), samples_per_iteration=samples,
                instructions=n, instructions_per_sample=n / samples, moves=moves, moves_per_sample=moves / samples,
                control=len(control), control_per_sample=len(control) / samples,
                lds=count(lambda o: op_base(o) == "LDS"), ldg=count(lambda o: op_base(o) == "LDG"),
                ffma=mix.get("FFMA", 0), fadd=mix.get("FADD", 0), fmul=mix.get("FMUL", 0), prmt=mix.get("PRMT", 0),
                control_list=["%s %s %s" % (hex(a), p, o) for a, p, o in control],
                mix=dict(sorted(mix.items(), key=lambda kv: -kv[1])))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cu", default=os.path.join(ROOT, "mve_b200", "csrc", "b200mvs.cu"))
    ap.add_argument("--cubin")
    ap.add_argument("--json", action="store_true")
    args, extra = ap.parse_known_args()
    with tempfile.TemporaryDirectory() as tmp:
        if args.cubin:
            cubin, usage = args.cubin, res_usage(args.cubin, KERNEL)
        else:
            cubin, log = compile_cubin(args.cu, extra, tmp)
            usage = ptxas_usage(log, KERNEL)
        r = report(usage, kernel_sass(cubin, KERNEL))
    if args.json:
        print(json.dumps(r))
        return
    sp = lambda v: "n/a" if v is None else v
    print("%s: %d registers, %s bytes spill stores, %s bytes spill loads, %d bytes stack frame"
          % (KERNEL, r["registers"], sp(r["spill_stores"]), sp(r["spill_loads"]), r["stack_frame"]))
    print("sample loop %s-%s: %d samples per iteration, %d instructions (%.1f per sample)"
          % (r["loop_start"], r["loop_end"], r["samples_per_iteration"], r["instructions"], r["instructions_per_sample"]))
    print("  moves %d (%.1f per sample), control %d (%.1f per sample), LDS %d, LDG %d, FFMA %d, FADD %d, FMUL %d, PRMT %d"
          % (r["moves"], r["moves_per_sample"], r["control"], r["control_per_sample"], r["lds"], r["ldg"], r["ffma"], r["fadd"],
             r["fmul"], r["prmt"]))
    print("  control:", ", ".join(r["control_list"]))
    print("  mix:", " ".join("%s %d" % kv for kv in r["mix"].items()))


if __name__ == "__main__":
    main()
