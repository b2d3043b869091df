#!/usr/bin/env python3
"""Cycles per arithmetic-coded decision of the device token decoder (k_tokens<1>).

k_tokens<1> is one serial chain of decisions per frame, so its time per frame over the frame's decisions is the
chain's latency per decision.  This tool counts every frame's decisions on the host -- the kernel's own code,
tokens_core.cuh, compiled with g++ and a counter on lr_decide (tools/tokens_chain_count.cc) -- for the frames
tools/tokens_bench.py times (default: the first 30 frames of each GOP of bench.py's 1080p workload), and
joins the counts with the kernel times of a tokens_bench.py --json file:

    python tools/tokens_bench.py --json tb.json        # on the GPU
    python tools/tokens_chain.py --times tb.json --sm-mhz 1980

Without --times it prints the decision counts alone (no GPU needed).  --sass FILE (an object or library built
with -gencode arch=compute_90a,code=sm_90a) adds the instruction mix of k_tokens<1>: instructions, branches,
FLO (one per decision) and multiplies.  Cycles are at --sm-mhz, which should be the SM clock the kernel ran at
(nvidia-smi --query-gpu=clocks.max.sm)."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def counter_lib():
    d = tempfile.mkdtemp(prefix="tokens_chain_")
    so = os.path.join(d, "tokens_chain_count.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC",
                           os.path.join(ROOT, "tools", "tokens_chain_count.cc"),
                           os.path.join(ROOT, "alfalfa_b200", "csrc", "parser.cc"), "-o", so])
    L = C.CDLL(so)
    L.tc_new.restype = C.c_void_p
    L.tc_new.argtypes = [C.c_int, C.c_int]
    L.tc_free.argtypes = [C.c_void_p]
    L.tc_frame.restype = C.c_int
    L.tc_frame.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_ulonglong)]
    return L


def bench_gops(frames):
    """(label, frames) as tools/tokens_bench.py builds them by default"""
    import bench
    w, h, inst = bench.load_instances(bench.WORKLOADS["1080p"], per_clip=0)
    return w, h, [("gop%d" % k, g[:frames]) for k, g in enumerate(inst)]


def sass_mix(path):
    """instruction mix of k_tokens<1> in a cubin-bearing file"""
    out = subprocess.run([os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), "-sass", path],
                         capture_output=True, text=True, check=True).stdout
    body, on = [], False
    for line in out.splitlines():
        if "Function :" in line:
            on = "k_tokensILi1E" in line
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if on and m:
            body.append(m.group(2))
    ops = [b.split(".")[0] for b in body]
    mix = {k: ops.count(k) for k in ("FLO", "BRA", "BSSY", "IMAD", "SHF", "LDS", "SEL", "ISETP")}
    mix["instructions"] = len(ops)
    return mix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--times", default=None, help="tools/tokens_bench.py --json output (same frames)")
    ap.add_argument("--sm-mhz", type=float, default=1980.0)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--sass", default=None, help="object or library with k_tokens<1> (sm_90a)")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    L = counter_lib()
    w, h, gops = bench_gops(a.frames)
    times = json.load(open(a.times)) if a.times else None
    if times:
        print("timed on: %s" % times.get("device"))
    res, tot_d, tot_ms = [], 0, 0.0
    for g, (name, frames) in enumerate(gops):
        H = L.tc_new(w, h)
        out = (C.c_ulonglong * 2)()
        rows = []
        for i, f in enumerate(frames):
            rc = L.tc_frame(H, f, len(f), out)
            if rc != 0:
                raise SystemExit("%s frame %d: parser code %d" % (name, i, rc))
            r = {"decisions": int(out[0]), "tokens": int(out[1])}
            if times:
                t = times["gops"][g]["frames"][i]
                assert t["tokens"] == r["tokens"], "the timed frames are not these frames"
                r["kernel_ms"] = t["kernel_ms"]
            rows.append(r)
        L.tc_free(H)
        d = sum(r["decisions"] for r in rows)
        line = "%-6s %3d frames  %10d decisions  %8.2f per token" % (name, len(rows), d, d / max(1, sum(r["tokens"] for r in rows)))
        if times and all(r.get("kernel_ms") is not None for r in rows):
            ms = sum(r["kernel_ms"] for r in rows)
            big = max(rows, key=lambda r: r["decisions"])
            line += "  %6.1f ns/decision = %5.1f cycles  (largest frame: %d decisions, %.2f ms, %.1f cycles)" % (
                ms * 1e6 / d, ms * 1e3 * a.sm_mhz / d, big["decisions"], big["kernel_ms"],
                big["kernel_ms"] * 1e3 * a.sm_mhz / big["decisions"])
            tot_ms += ms
        tot_d += d
        print(line)
        res.append({"gop": name, "frames": rows})
    summary = {"decisions": tot_d}
    if tot_ms:
        summary.update(kernel_ms=tot_ms, ns_per_decision=tot_ms * 1e6 / tot_d, cycles_per_decision=tot_ms * 1e3 * a.sm_mhz / tot_d,
                       sm_mhz=a.sm_mhz)
        print("all: %d decisions, %.1f ms of k_tokens, %.2f ns = %.1f cycles per decision at %.0f MHz" % (
            tot_d, tot_ms, summary["ns_per_decision"], summary["cycles_per_decision"], a.sm_mhz))
    if a.sass:
        summary["sass"] = sass_mix(a.sass)
        print("k_tokens<1> SASS: %s" % summary["sass"])
    if a.json:
        json.dump({"summary": summary, "gops": res}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
