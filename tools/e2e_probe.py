#!/usr/bin/env python3
"""GPU-box tool: sweep the host-side knobs of vp8gpu_decode_ivf on the bench workload (output left on the device)
and print Mpix/s, the host time accounting and -- with --trace (VP8GPU_TRACE=1) -- the per-batch device times of every
dispatcher and, per worker, the distribution of its chunks' latency from "staged" to "head frame ready" and to "ready" (k_tokens).
The bench shape: --configs 64:4:5 --streams 258.
usage: tools/e2e_probe.py [--configs "threads:dispatchers:nice,..."] [--steps N] [--trace]"""
import argparse
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="64:4:5,64:4:0,64:2:5,64:1:5,64:8:5,32:2:5,128:4:5,128:8:5")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--streams", type=int, default=258)
    ap.add_argument("--trace", action="store_true", help="VP8GPU_TRACE=1: per-batch and per-chunk device times on stderr")
    a = ap.parse_args()
    if a.trace:
        os.environ["VP8GPU_TRACE"] = "1"
    import bench
    from alfalfa_b200 import Context, capi
    w, h, instances = bench.load_instances(bench.WORKLOADS["1080p"], per_clip=0)
    L = capi.lib()
    all_frames = []
    for r in range(-(-a.streams // len(instances))):
        for inst in instances:
            all_frames.extend(inst)
    big = bench.make_ivf(w, h, all_frames)
    n = len(all_frames)
    ctx = Context(w, h, device=0, max_frames=128 * 102 + 64)
    ctx.set_device_tokens(True)
    nd, ns = C.c_uint32(0), C.c_uint32(0)
    for cfg in a.configs.split(","):
        threads, disp, nice = [int(x) for x in cfg.split(":")]
        os.environ["VP8GPU_DISPATCHERS"] = str(disp)
        os.environ["VP8GPU_WORKER_NICE"] = str(nice)
        best = 1e9
        for it in range(a.steps + 1):
            t0 = time.perf_counter()
            capi.check(L.vp8gpu_decode_ivf(ctx.h, big, len(big), threads, None, 0, C.byref(nd), C.byref(ns)), ctx.h, "decode_ivf")
            capi.check(L.vp8gpu_ctx_sync(ctx.h), ctx.h, "sync")
            dt = time.perf_counter() - t0
            if it:
                best = min(best, dt)
        st = (C.c_double * 8)()
        L.vp8gpu_decode_ivf_stats(ctx.h, st)
        print("threads %3d dispatchers %d nice %d: %7.0f Mpix/s (%d frames in %.3f s) | parse %.2f wait_dispatch %.2f wait_dma %.2f "
              "submit %.2f idle %.2f batches %d" % (threads, disp, nice, n * w * h / 1e6 / best, n, best, st[0], st[1], st[2], st[3],
                                                      st[5], int(st[6])), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
