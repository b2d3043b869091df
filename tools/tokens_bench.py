#!/usr/bin/env python3
"""Latency of the device-side token decoder for single frames.

Default: every frame of the six GOPs of bench.py's 1080p workload goes through vp8gpu_parse_frame_device
(first partition on the host, H2D, k_tokens with ONE frame, records back), one frame per launch, under
torch.profiler: the table gives each frame's k_tokens kernel time next to its DCT partition bytes, DCT
partitions and tokens, so it reads as ns per token and per byte.  The host columns time the whole
device path and the all-host front end (vp8gpu_parse_frame) around the same frame.
usage: python tools/tokens_bench.py [ivf ...] [--frames N] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


class _Bool:
    """RFC 6386 section 7 boolean decoder, enough to read a frame header's first fields"""

    def __init__(self, data):
        self.d, self.pos = data, 2
        self.value = (data[0] << 8) | data[1] if len(data) >= 2 else 0
        self.range, self.count = 255, 0

    def bit(self, prob):
        split = 1 + (((self.range - 1) * prob) >> 8)
        big = split << 8
        if self.value >= big:
            b, self.range, self.value = 1, self.range - split, self.value - big
        else:
            b, self.range = 0, split
        while self.range < 128:
            self.value, self.range = (self.value << 1) & 0xFFFF, self.range << 1
            self.count += 1
            if self.count == 8:
                self.count = 0
                if self.pos < len(self.d):
                    self.value |= self.d[self.pos]
                self.pos += 1
        return b

    def lit(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | self.bit(128)
        return v


def partition_layout(f):
    """(DCT partitions, their bytes incl. the partition-size table) from a frame's tag and header (RFC 6386 9.2-9.5)"""
    key = not (f[0] & 1)
    first = ((f[0] | (f[1] << 8) | (f[2] << 16)) >> 5) & 0x7FFFF
    hdr = 10 if key else 3
    b = _Bool(f[hdr:hdr + first])
    if key:
        b.lit(2)  # colour space, clamping
    if b.lit(1):  # segmentation
        upd_map, upd_data = b.lit(1), b.lit(1)
        if upd_data:
            b.lit(1)
            for bits in [7] * 4 + [6] * 4:
                if b.lit(1):
                    b.lit(bits + 1)
        if upd_map:
            for _ in range(3):
                if b.lit(1):
                    b.lit(8)
    b.lit(1 + 6 + 3)  # filter type, level, sharpness
    if b.lit(1) and b.lit(1):  # loop-filter deltas and their update
        for _ in range(8):
            if b.lit(1):
                b.lit(7)
    return 1 << b.lit(2), len(f) - hdr - first


def kernel_times_us(prof):
    """k_tokens kernel durations in launch order"""
    ev = [e for e in prof.events() if "k_tokens" in e.name and str(e.device_type).endswith("CUDA")]
    ev.sort(key=lambda e: e.time_range.start)
    return [e.time_range.elapsed_us() for e in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("ivf", nargs="*", help="default: the GOPs of bench.py's 1080p workload")
    ap.add_argument("--frames", type=int, default=30, help="frames per GOP")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from alfalfa_b200 import Context, capi
    from alfalfa_b200.decoder import read_ivf
    if a.ivf:
        gops = []
        for p in a.ivf:
            w, h, frames = read_ivf(open(p, "rb").read())
            gops.append((os.path.basename(p), frames[:a.frames]))
    else:
        names = bench.WORKLOADS["1080p"]
        w, h, inst = bench.load_instances(names, per_clip=0)
        # instance -> clip: load_instances keeps the clips' order, a clip's GOPs one after another
        labels = []
        for n in names:
            _, _, fr = read_ivf(open(bench.clip_path(n), "rb").read())
            nk = sum(1 for f in fr if not (f[0] & 1))
            labels += ["%s#%d" % (n[:-4], k) if nk > 1 else n[:-4] for k in range(nk)]
        gops = [(labels[k] if k < len(labels) else "gop%d" % k, g[:a.frames]) for k, g in enumerate(inst)]
    torch.cuda.init()
    L = capi.lib()
    ctx = Context(w, h, max_frames=4)
    pf = C.c_void_p()
    capi.check(L.vp8gpu_parsed_create(C.byref(pf)))

    def run_gop(frames, timed):
        st_h, st_d = C.c_void_p(), C.c_void_p()
        capi.check(L.vp8gpu_state_create(w, h, C.byref(st_h)))
        capi.check(L.vp8gpu_state_create(w, h, C.byref(st_d)))
        rows = []
        for f in frames:
            t0 = time.perf_counter()
            capi.check(L.vp8gpu_parse_frame(st_h, f, len(f), pf), ctx.h, "parse")
            t1 = time.perf_counter()
            capi.check(L.vp8gpu_parse_frame_device(ctx.h, st_d, f, len(f), pf), ctx.h, "parse_device")
            t2 = time.perf_counter()
            d = L.vp8gpu_parsed_desc(pf).contents
            nparts, tbytes = partition_layout(f)
            rows.append({"key": not (f[0] & 1), "bytes": len(f), "part_bytes": tbytes, "nparts": nparts,
                         "tokens": int(d.n_tokens), "host_ms": (t1 - t0) * 1e3, "device_path_ms": (t2 - t1) * 1e3})
        L.vp8gpu_state_destroy(st_h)
        L.vp8gpu_state_destroy(st_d)
        return rows

    run_gop(gops[0][1][:4], False)  # warm-up: module load, scratch ring
    props = torch.cuda.get_device_properties(0)
    print("device: %s, %d SMs" % (props.name, props.multi_processor_count))
    out = []
    for name, frames in gops:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            rows = run_gop(frames, True)
        kt = kernel_times_us(prof)
        for i, r in enumerate(rows):
            r["kernel_ms"] = kt[i] / 1e3 if len(kt) == len(rows) else None
        print("== %s: %d frames" % (name, len(rows)))
        print("frame key  bytes  part_B parts  tokens  k_tokens_ms  ns/token  ns/byte  device_path_ms  host_ms")
        for i, r in enumerate(rows):
            k = r["kernel_ms"]
            ks = ("%11.3f %9.1f %8.1f" % (k, k * 1e6 / max(r["tokens"], 1), k * 1e6 / max(r["part_bytes"], 1))
                  if k is not None else "%11s %9s %8s" % ("n/a", "", ""))
            print("%5d %3s %7d %7d %5d %7d %s %15.3f %8.3f" % (i, "K" if r["key"] else "", r["bytes"], r["part_bytes"], r["nparts"],
                                                            r["tokens"], ks, r["device_path_ms"], r["host_ms"]))
        ks = [r["kernel_ms"] for r in rows if r["kernel_ms"] is not None]
        if ks:
            print("   k_tokens: max %.3f ms, mean %.3f ms, sum %.3f ms over %d frames; %.1f ns per token overall" % (
                max(ks), sum(ks) / len(ks), sum(ks), len(ks), sum(ks) * 1e6 / max(sum(r["tokens"] for r in rows), 1)))
        out.append({"gop": name, "frames": rows})
        sys.stdout.flush()
    L.vp8gpu_parsed_destroy(pf)
    ctx.close()
    if a.json:
        json.dump({"device": props.name, "gops": out}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
