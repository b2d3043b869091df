#!/usr/bin/env python
"""Frames / s of re-encoding many 1080p chunks at once (alfalfa_b200.reencode_chunks: the update_residues frames of every
chunk at a frame position in one vp8gpu_encoder_update_residues_batch call) next to the same chunks through a loop of
single Encoder.reencode calls, alternating in one process, at n = 1, 2, 4, 8, 16, 32 chunks; the emitted frames of both
arms must be byte-identical.  Also the per-phase timeline of the last batch call (where the time of a batch goes) and
the unmodified reference's Encoder::reencode (oracle/_ref/ref_reencode) on the same chunks, one process per chunk on
all usable host cores.  Prints one JSON line.

A chunk is a bench clip (tools/reencode_bench.py's bench_inputs: 12 frames, extra-frame chunk, kf_q_weight 0.75, targets
= the clip's own decoded pictures); its receiver state is another bench clip after k frames.  Clip and k vary so that
the chunks of a batch really differ."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

BD = os.path.join(ROOT, "bench_data")
CHUNKS = ["synth1080p_medium_q90.ivf", "synth1080p_medium_q110_s21.ivf", "synth1080p_hard_q60_s7.ivf", "synth1080p_easy_q60_s5.ivf"]
STATES = [("synth1080p_easy_q40.ivf", 8), ("synth1080p_medium_q70_s33.ivf", 5), ("synth1080p_easy_q60_s5.ivf", 3),
          ("synth1080p_hard_q60_s7.ivf", 10), ("synth1080p_medium_q90.ivf", 6), ("synth1080p_easy_q40.ivf", 2),
          ("synth1080p_medium_q110_s21.ivf", 4), ("synth1080p_medium_q70_s33.ivf", 11)]
KF_Q_WEIGHT = 0.75


def gpu_card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable: " + r.stderr[-200:]


def make_chunks(ctx, n):
    """n (state, prediction chunk bytes, prediction frames, targets): chunk clip i % 4 against state (i // 4) % 8"""
    from alfalfa_b200 import Decoder
    from alfalfa_b200.decoder import read_ivf
    import reencode_bench as B
    clips, states = {}, {}
    out = []
    for i in range(n):
        clip, (prev, k) = CHUNKS[i % len(CHUNKS)], STATES[(i // len(CHUNKS)) % len(STATES)]
        if clip not in clips:
            _, chunk, pfs, targets = B.bench_inputs(ctx, os.path.join(BD, prev), os.path.join(BD, clip))
            clips[clip] = (chunk, pfs, targets)
        if (prev, k) not in states:
            d = Decoder(ctx)
            for c in read_ivf(open(os.path.join(BD, prev), "rb").read())[2][:k]:
                _, r = d.get_frame_output(c)
                r.release()
            states[(prev, k)] = d.serialize()
        out.append((states[(prev, k)],) + clips[clip])
    return out


def encoders(ctx, chunks):
    from alfalfa_b200 import Decoder, Encoder
    return [Encoder.from_decoder(ctx, Decoder.deserialize(ctx, s)) for s, _, _, _ in chunks]


def run_batch(ctx, chunks):
    from alfalfa_b200 import reencode_chunks
    encs = encoders(ctx, chunks)
    t0 = time.perf_counter()
    frames = reencode_chunks(encs, [t for _, _, _, t in chunks], [p for _, _, p, _ in chunks], KF_Q_WEIGHT, True)
    return frames, time.perf_counter() - t0, encs[-1].timeline()


def run_loop(ctx, chunks):
    encs = encoders(ctx, chunks)
    t0 = time.perf_counter()
    frames = [e.reencode(t, p, KF_Q_WEIGHT, True) for e, (_, _, p, t) in zip(encs, chunks)]
    return frames, time.perf_counter() - t0, None


def reference_leg(chunks, frames, w, h):
    """oracle/_ref/ref_reencode, one process per chunk on every usable core: frames / s over the whole set and how many
    of its frames equal the batch's"""
    from alfalfa_b200.decoder import read_ivf, write_ivf
    from bench import effective_cpus
    tool = os.path.join(ROOT, "oracle", "_ref", "ref_reencode")
    if not os.path.exists(tool):
        return {"unavailable": "oracle/_ref/ref_reencode not built"}
    cores = effective_cpus()
    with tempfile.TemporaryDirectory() as tmp:
        jobs = []
        for i, (state, chunk, _, targets) in enumerate(chunks):
            raw, pivf, sbin, oivf = (os.path.join(tmp, "%d.%s" % (i, x)) for x in ("yuv", "p.ivf", "bin", "o.ivf"))
            with open(raw, "wb") as f:
                for planes in targets:
                    for p in planes:
                        f.write(p.tobytes())
            open(pivf, "wb").write(write_ivf(w, h, chunk))
            open(sbin, "wb").write(state)
            jobs.append(([tool, oivf, str(w), str(h), raw, pivf, sbin, repr(KF_Q_WEIGHT), "1"], oivf))
        t0 = time.perf_counter()
        with ThreadPoolExecutor(cores) as pool:
            rcs = list(pool.map(lambda j: subprocess.run(j[0], capture_output=True).returncode, jobs))
        secs = time.perf_counter() - t0
        if any(rcs):
            return {"unavailable": "ref_reencode failed: %s" % rcs}
        ref = [read_ivf(open(o, "rb").read())[2] for _, o in jobs]
    n = sum(len(r) for r in ref)
    return {"fps": n / secs, "cores": cores, "chunks": len(chunks), "frames": n,
            "identical_frames": sum(1 for r, f in zip(ref, frames) for a, b in zip(r, f) if a == b),
            "sample": "oracle/_ref/ref_reencode (unmodified Encoder::reencode, C++ fallback build), one process per chunk; wall time "
                      "of all processes incl. reading the inputs and parsing the chunks"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,2,4,8,16,32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    sizes = [int(x) for x in a.sizes.split(",")]

    from alfalfa_b200 import Context
    w, h = 1920, 1080
    card = gpu_card()
    ctx = Context(w, h, device=a.device, max_frames=16 * max(sizes) + 64)
    chunks = make_chunks(ctx, max(sizes))
    out = {"metric": "re-encode fps @1080p, n chunks of 12 frames (extra-frame chunks): reencode_chunks (batched update_residues) "
                     "vs a loop of Encoder.reencode", "gpu": card, "kf_q_weight": KF_Q_WEIGHT, "results": []}
    last_batch = None
    for n in sizes:
        sub = chunks[:n]
        run_batch(ctx, sub), run_loop(ctx, sub)  # warm-up: allocations, pooled buffers, first launches
        tb, tl, tls = [], [], None
        for _ in range(a.repeats):
            fb, sb, tls = run_batch(ctx, sub)
            fl, sl, _ = run_loop(ctx, sub)
            assert fb == fl, "n=%d: the batch emitted other bytes than the single calls" % n
            tb.append(sb)
            tl.append(sl)
        frames = sum(len(f) for f in fb)
        out["results"].append({"chunks": n, "frames": frames, "batch_fps": frames / statistics.median(tb),
                               "loop_fps": frames / statistics.median(tl), "batch_s": tb, "loop_s": tl,
                               "last_batch_call_ms": {k: round(v, 3) for k, v in tls.items() if v}})
        last_batch = fb
    ctx.close()
    out["reference"] = reference_leg(chunks, last_batch, w, h)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
