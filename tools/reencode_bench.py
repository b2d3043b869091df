#!/usr/bin/env python
"""Frames / s of Encoder::update_residues (SURVEY.md 8 row f3) at 1080p through the public API -- target planes in host
memory in, compressed frame out, every step incl. the H2D of the target, the kernels, the D2H of records and tokens,
the host writer and the decode of the emitted frame that advances the Encoder -- next to the UNMODIFIED reference's
Encoder::reencode (oracle/_ref/ref_reencode, one host core) on the same inputs, and how many emitted frames are
byte-identical.  Run by bench.py in a child process under a timeout; prints one JSON line.

The ExCamera situation: the chunk (a bench clip, coded on its own by the reference encoder) is re-encoded as an
extra-frame chunk against the state another clip leaves behind; targets = the chunk's own decoded pictures."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


PREV = os.path.join(ROOT, "bench_data", "synth1080p_easy_q40.ivf")
CHUNK = os.path.join(ROOT, "bench_data", "synth1080p_medium_q90.ivf")
PREV_FRAMES = 8


def bench_inputs(ctx, prev_path=PREV, chunk_path=CHUNK, frames=12):
    """The inputs of the measured re-encode: the state PREV_FRAMES frames of `prev_path` leave behind (Decoder::
    serialize, the reference's own format, tests/test_state_format.py), the first `frames` frames of `chunk_path`,
    parsed with keep_labels by their own decoder, and their decoded pictures as targets.  ctx: a Context of the
    clips' size.  -> (state, chunk, prediction_frames, targets)"""
    import numpy as np

    from alfalfa_b200 import Decoder
    from alfalfa_b200.decoder import read_ivf

    w, h, prev = read_ivf(open(prev_path, "rb").read())
    w2, h2, chunk = read_ivf(open(chunk_path, "rb").read())
    assert (w, h) == (w2, h2) == (ctx.width, ctx.height)
    chunk = chunk[:frames]
    d = Decoder(ctx)
    for c in prev[:PREV_FRAMES]:
        d.get_frame_output(c)
    state = d.serialize()
    pred_decoder = Decoder(ctx)
    prediction_frames, targets = [], []
    cw, ch = (w + 1) // 2, (h + 1) // 2
    for c in chunk:
        pf = pred_decoder.parse_frame(c, keep_labels=True)
        _, r = pred_decoder.decode_frame(pf)
        b = np.frombuffer(r.display_bytes(), np.uint8)
        targets.append((b[:w * h].reshape(h, w).copy(), b[w * h:w * h + cw * ch].reshape(ch, cw).copy(),
                        b[w * h + cw * ch:].reshape(ch, cw).copy()))
        prediction_frames.append(pf)
    return state, chunk, prediction_frames, targets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--prev", default=PREV)
    ap.add_argument("--chunk", default=CHUNK)
    ap.add_argument("--kf-q-weight", type=float, default=0.75)
    a = ap.parse_args()

    from alfalfa_b200 import Context, Decoder, Encoder
    from alfalfa_b200.decoder import read_ivf, write_ivf

    w, h = read_ivf(open(a.chunk, "rb").read())[:2]
    ctx = Context(w, h, device=a.device, max_frames=32)
    state, chunk, prediction_frames, targets = bench_inputs(ctx, a.prev, a.chunk, a.frames)

    def run():
        enc = Encoder.from_decoder(ctx, Decoder.deserialize(ctx, state))
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        frames = enc.reencode(targets, prediction_frames, a.kf_q_weight, True)
        return frames, time.perf_counter() - t0, ctx.launch_count() - l0

    run()  # warm-up (allocations, first launches)
    frames, secs, launches = min((run() for _ in range(3)), key=lambda x: x[1])
    n = len(frames)
    out = {"metric": "Encoder::reencode (update_residues) fps @1080p, extra-frame chunk", "frames": n, "fps": n / secs,
           "ms_per_frame": 1e3 * secs / n, "bytes_per_frame": sum(len(f) for f in frames) / n, "gpu_launches": int(launches),
           "api": "vp8gpu_encoder_update_residues: host target planes -> compressed frame, incl. the decode that advances the Encoder",
           "chunk": os.path.basename(a.chunk), "state_after": os.path.basename(a.prev)}
    ctx.close()
    tool = os.path.join(ROOT, "oracle", "_ref", "ref_reencode")
    if os.path.exists(tool):
        with tempfile.TemporaryDirectory() as tmp:
            raw, pivf, sbin, oivf = (os.path.join(tmp, x) for x in ("t.yuv", "p.ivf", "s.bin", "o.ivf"))
            with open(raw, "wb") as f:
                for planes in targets:
                    for p in planes:
                        f.write(p.tobytes())
            open(pivf, "wb").write(write_ivf(w, h, chunk))
            open(sbin, "wb").write(state)
            t0 = time.perf_counter()
            r = subprocess.run([tool, oivf, str(w), str(h), raw, pivf, sbin, repr(a.kf_q_weight), "1"], capture_output=True, text=True)
            ref_secs = time.perf_counter() - t0
            if r.returncode == 0:
                ref_frames = read_ivf(open(oivf, "rb").read())[2]
                out["reference"] = {"fps": len(ref_frames) / ref_secs, "cores": 1, "kind": "reference",
                                    "sample": "oracle/_ref/ref_reencode (unmodified Encoder::reencode, C++ fallback build), the same chunk, "
                                              "targets and state; wall time of the process incl. reading the inputs and parsing the chunk",
                                    "identical_frames": sum(1 for x, y in zip(ref_frames, frames) if x == y), "frames": len(ref_frames)}
            else:
                out["reference"] = {"unavailable": r.stderr[-200:]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
