#!/usr/bin/env python3
"""GPU-box tool: where does a macroblock step of the wavefront kernels spend its cycles?
Uses the -DVP8_PROFILE build of the library (alfalfa_b200/csrc/build.sh prof), decodes frames of the
bench clip through the HBM-resident batch API and prints average clock64() cycles per phase per MB.  The loop filter's
phases are k_loopfilter_band's (the default) unless VP8GPU_WAVEFRONT selects another kernel pair.
usage: tools/phase_profile.py [--g N]"""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["VP8GPU_LIB"] = os.path.join(ROOT, "alfalfa_b200", "libvp8gpu_prof.so")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import oracle_lib as O  # noqa: E402
from alfalfa_b200 import Context, capi  # noqa: E402

INTRA = ["load_mb", "build_residuals", "wait_row", "edge loads", "predict+add", "store+next", "publish", "loop overhead"]
LF = ["load_mb", "wait_row", "top/left loads+smem", "filter", "write back", "publish", "-", "loop overhead"]
LF_BAND = ["load_mb", "wait in band", "wait between bands", "top/left loads+smem", "filter", "ring back-pressure",
           "write back+publish", "loop overhead"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=1)
    a = ap.parse_args()
    lf_labels = LF if os.environ.get("VP8GPU_WAVEFRONT") in ("legacy", "ll", "intra-ll", "lf-ll") else LF_BAND
    L = capi.lib()
    prof = C.CDLL(os.environ["VP8GPU_LIB"]).vp8gpu_debug_profile
    data = open(os.path.join(ROOT, "bench_data", "synth1080p_medium_q90.ivf"), "rb").read()
    w, h, frames = O.read_ivf(data)
    n_mbs = ((w + 15) // 16) * ((h + 15) // 16)
    ctx = Context(w, h, max_frames=a.g * 4 + 8)
    st, pf = C.c_void_p(), C.c_void_p()
    capi.check(L.vp8gpu_state_create(w, h, C.byref(st)))
    capi.check(L.vp8gpu_parsed_create(C.byref(pf)))
    buf = (C.c_ulonglong * 32)()
    refs = [None] * a.g
    for fi, f in enumerate(frames[30:34]):  # key frame with loop filter on, then inter frames
        capi.check(L.vp8gpu_parse_frame(st, f, len(f), pf))
        d = capi.FrameDesc.from_buffer_copy(bytes(L.vp8gpu_parsed_desc(pf).contents))
        mbs = np.frombuffer(C.string_at(L.vp8gpu_parsed_mbs(pf), n_mbs * 32), dtype=capi.MB_DTYPE).copy()
        tok = np.frombuffer(C.string_at(L.vp8gpu_parsed_tokens(pf), max(d.n_tokens, 1) * 4), dtype="<u4").copy()
        sp = np.frombuffer(C.string_at(L.vp8gpu_parsed_split(pf), max(d.n_split, 1) * 64), dtype="u1").copy()
        jobs = (capi.Job * a.g)()
        outs = []
        for g in range(a.g):
            out = ctx.alloc_frame()
            outs.append(out)
            jobs[g].desc = C.pointer(d)
            jobs[g].mbs, jobs[g].tokens, jobs[g].split = mbs.ctypes.data, tok.ctypes.data, sp.ctypes.data
            jobs[g].refs[:] = [-1] * 3 if d.key_frame else [refs[g].id] * 3
            jobs[g].out = out.id
        b = C.c_void_p()
        capi.check(L.vp8gpu_batch_upload(ctx.h, jobs, a.g, C.byref(b)), ctx.h, "upload")
        ms3 = (C.c_float * 3)()
        capi.check(L.vp8gpu_batch_run_timed(ctx.h, 0, b, ms3), ctx.h, "warm")
        prof(buf, 1)
        capi.check(L.vp8gpu_batch_run_timed(ctx.h, 0, b, ms3), ctx.h, "run")
        prof(buf, 1)
        v = list(buf)
        n_intra = int((mbs["ref_frame"] == 0).sum())
        print("frame %d (%s) x%d: k_inter %.3f ms  k_intra %.3f ms  k_loopfilter %.3f ms | intra MBs %d bpred %d filtered %d"
              % (30 + fi, "key" if d.key_frame else "inter", a.g, ms3[0], ms3[1], ms3[2], n_intra,
                 int((mbs["y_mode"] == 4).sum()), int((mbs["lf_level"] > 0).sum())))
        for name, base, labels in (("k_intra", 0, INTRA), ("k_loopfilter", 16, lf_labels)):
            n = v[base + 8]
            if not n:
                continue
            tot = sum(v[base:base + 8])
            print("  %s: %d MB steps, %.0f cycles/MB total" % (name, n, tot / n))
            for i, lab in enumerate(labels):
                if v[base + i]:
                    print("     %-22s %8.0f cycles/MB  %4.1f%%" % (lab, v[base + i] / n, 100.0 * v[base + i] / tot))
        L.vp8gpu_batch_free(ctx.h, b)
        for r in refs:
            if r is not None:
                r.release()
        refs = outs
    ctx.close()


if __name__ == "__main__":
    main()
