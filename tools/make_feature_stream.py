#!/usr/bin/env python3
"""Synthesise a feature-complete VP8 stream (SURVEY.md 8d, "bitstream B").

No >= 1080p VP8 material exists in the reference tree, and its encoder only produces one partition,
LAST-only prediction and no SPLITMV.  This tool builds frames directly from seeded-random flat
records (include/vp8gpu.h) and writes them with the product's bitstream writer
(vp8gpu_serialize_frame_ex, host only): 1-8 DCT partitions, segmentation (map + absolute / delta
quantiser and loop-filter levels), loop-filter deltas, quantiser deltas, golden / altref prediction
with sign bias, buffer copies and refreshes, hidden frames, persistent probability updates, every
intra mode incl. B_PRED in key and inter frames, SPLITMV with all four layouts, vectors up to +-64 px
in quarter-pel steps, sparse coefficients up to DCT_CAT6.  What the stream decodes to is defined by
the reference decoder: tools/make_bench_streams.sh records its SHA-1 in tests/golden/bench_clips.json.

usage: python tools/make_feature_stream.py OUT.ivf WIDTH HEIGHT FRAMES [SEED]
"""
import ctypes as C
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DC_PRED, V_PRED, H_PRED, TM_PRED, B_PRED, NEARESTMV, NEARMV, ZEROMV, NEWMV, SPLITMV = range(10)
REF_CURRENT, REF_LAST, REF_GOLDEN, REF_ALTREF = range(4)
# modemv_data.cc:252-278: luma sub-blocks of each partition of the four split layouts
SPLIT_LAYOUTS = [
    [0x00FF, 0xFF00],
    [0x3333, 0xCCCC],
    [0x0033, 0x00CC, 0x3300, 0xCC00],
    [1 << i for i in range(16)],
]


def random_value(rng):
    """coefficient magnitudes: mostly 1..2, a tail through every DCT_CAT class"""
    r = rng.random()
    if r < 0.70:
        return 1
    if r < 0.85:
        return 2
    if r < 0.93:
        return int(rng.integers(3, 11))
    if r < 0.98:
        return int(rng.integers(11, 67))
    return int(rng.integers(67, 2048))


def serialize(L, capi, hdr, ft, mbs, tokens, split):
    """one compressed frame from flat records: tokens a list of packed vp8gpu_token, split a list of (16, 2) vectors"""
    tok = np.array(tokens if tokens else [0], dtype="<u4")
    sp = np.stack(split) if split else np.zeros((1, 16, 2), dtype=np.int16)
    sp = np.ascontiguousarray(sp, dtype="<i2")
    cap = 64 + len(mbs) * 96 + len(tokens) * 4
    out = (C.c_uint8 * cap)()
    size = C.c_size_t(0)
    rc = L.vp8gpu_serialize_frame_ex(C.byref(hdr), C.byref(ft), mbs.ctypes.data, tok.ctypes.data, sp.ctypes.data, out, cap,
                                     C.byref(size))
    if rc != 0:
        raise RuntimeError("serialize_frame_ex failed: %d" % rc)
    return bytes(out[:size.value])


def ivf(w, h, chunks):
    """-> IVF bytes (util/ivf.cc:36-82)"""
    out = [struct.pack("<4sHH4sHHIII", b"DKIF", 0, 32, b"VP80", w, h, 30, 1, len(chunks)) + b"\0\0\0\0"]
    for i, c in enumerate(chunks):
        out += [struct.pack("<IQ", len(c), i), c]
    return b"".join(out)   # joined once: the tests build streams of thousands of frames


def make_frame(rng, L, capi, w, h, index, saved_probs, all_bpred=False, segment_maps=True):
    """all_bpred: every intra macroblock uses B_PRED; segment_maps=False: no segmentation (so no segment-map
    update in inter frames, the form re-encoding takes) (the draws are the same either way)"""
    cols, rows = (w + 15) // 16, (h + 15) // 16
    n = cols * rows
    key = index == 0
    hdr = capi.EncodeHeader()
    hdr.width, hdr.height = w, h
    hdr.key_frame = int(key)
    hdr.show_frame = 0 if index % 6 == 4 else 1   # hidden frames: decoded, used as references, not output
    hdr.y_ac_qi = int(rng.integers(10, 100))
    hdr.loop_filter_level = int(rng.integers(0, 48)) if rng.random() < 0.85 else 0
    hdr.sharpness = int(rng.integers(0, 8))
    hdr.optimize_token_probs = int(rng.random() < 0.7)
    ft = capi.EncodeFeatures()
    ft.log2_partitions = (index + 3) % 4   # 8, 1, 2, 4, 8, ... DCT partitions
    ft.refresh_last = 1 if key or rng.random() < 0.85 else 0
    ft.refresh_entropy_probs = int(rng.random() < 0.5)
    ft.saved_coef_probs = saved_probs.ctypes.data
    for name in ("y_dc_delta", "y2_dc_delta", "y2_ac_delta", "uv_dc_delta", "uv_ac_delta"):
        if rng.random() < 0.4:
            setattr(ft, name, int(rng.integers(-15, 16)))
    seg = key or rng.random() < 0.6   # segmentation is sticky state: (re)sent often so that it is exercised
    if seg:
        ft.segmentation_enabled = 1
        ft.update_mb_segmentation_map = int(key or rng.random() < 0.6)
        ft.update_segment_feature_data = int(key or rng.random() < 0.6)
        ft.segment_feature_absolute = int(rng.random() < 0.5)
        for i in range(4):
            if ft.segment_feature_absolute:
                ft.segment_quant[i] = int(rng.integers(0, 128))
                ft.segment_lf[i] = int(rng.integers(0, 64))
            else:
                ft.segment_quant[i] = int(rng.integers(-127, 128))   # negative sums exercise the Unsigned<7> wrap
                ft.segment_lf[i] = int(rng.integers(-63, 64))
        for i in range(3):
            ft.segment_tree_probs[i] = int(rng.integers(1, 255)) if rng.random() < 0.8 else 255
        if not segment_maps:
            ft.segmentation_enabled = ft.update_mb_segmentation_map = ft.update_segment_feature_data = 0
    if rng.random() < 0.6:
        ft.lf_delta_enabled = 1
        ft.lf_delta_update = int(rng.random() < 0.7)
        for i in range(4):
            ft.ref_lf_delta[i] = int(rng.integers(-20, 21)) if rng.random() < 0.7 else 0
            ft.mode_lf_delta[i] = int(rng.integers(-20, 21)) if rng.random() < 0.7 else 0
    if not key:
        ft.refresh_golden = int(rng.random() < 0.25)
        ft.refresh_alternate = int(rng.random() < 0.25)
        ft.copy_to_golden = 0 if ft.refresh_golden else int(rng.integers(0, 3))
        ft.copy_to_alternate = 0 if ft.refresh_alternate else int(rng.integers(0, 3))
        ft.sign_bias_golden = int(rng.random() < 0.4)
        ft.sign_bias_alternate = int(rng.random() < 0.4)

    mbs = np.zeros(n, dtype=capi.MB_DTYPE)
    split = []
    tokens = []
    for i in range(n):
        m = mbs[i]
        m["segment_id"] = int(rng.integers(0, 4))
        intra = key or rng.random() < 0.25
        if intra:
            m["ref_frame"] = REF_CURRENT
            m["y_mode"] = int(rng.integers(0, 5))
            if all_bpred:
                m["y_mode"] = B_PRED
            m["uv_mode"] = int(rng.integers(0, 4))
            if m["y_mode"] == B_PRED:
                m["b_modes"] = int(sum(int(rng.integers(0, 10)) << (4 * k) for k in range(16)))
        else:
            m["ref_frame"] = int(rng.choice([REF_LAST, REF_LAST, REF_GOLDEN, REF_ALTREF]))
            r = rng.random()

            def rand_mv():
                if rng.random() < 0.3:   # whole-pel
                    return int(rng.integers(-64, 65)) * 8, int(rng.integers(-64, 65)) * 8
                return int(rng.integers(-256, 257)) * 2, int(rng.integers(-256, 257)) * 2
            if r < 0.2:
                m["y_mode"] = ZEROMV
            elif r < 0.45 and i > 0 and mbs[i - 1]["ref_frame"] != REF_CURRENT:
                m["y_mode"] = NEWMV      # the writer picks NEAREST / NEAR when the vector allows it
                m["mv_x"], m["mv_y"] = mbs[i - 1]["mv_x"], mbs[i - 1]["mv_y"]
            elif r < 0.8:
                m["y_mode"] = NEWMV
                m["mv_x"], m["mv_y"] = rand_mv()
            else:
                m["y_mode"] = SPLITMV
                layout = SPLIT_LAYOUTS[int(rng.integers(0, 4))]
                mv = np.zeros((16, 2), dtype=np.int16)
                for members in layout:
                    v = (0, 0) if rng.random() < 0.2 else rand_mv()
                    if rng.random() < 0.3:   # small vectors share more sub-block contexts
                        v = (int(rng.integers(-4, 5)) * 2, int(rng.integers(-4, 5)) * 2)
                    for k in range(16):
                        if members >> k & 1:
                            mv[k] = v
                m["split_idx"] = len(split)
                m["mv_x"], m["mv_y"] = int(mv[15, 0]), int(mv[15, 1])
                split.append(mv)
        has_y2 = m["y_mode"] not in (B_PRED, SPLITMV)
        m["flags"] = 1 if has_y2 else 0
        if rng.random() < 0.35:
            continue   # no coefficients: mb_skip_coeff
        first = len(tokens)
        blocks = rng.choice(25 if has_y2 else 24, size=int(rng.integers(1, 7)), replace=False)
        for b in sorted(int(x) for x in blocks):
            lo = 1 if (has_y2 and b < 16) else 0
            for pos in sorted(int(x) for x in rng.choice(np.arange(lo, 16), size=int(rng.integers(1, 4)), replace=False)):
                v = random_value(rng) * (1 if rng.random() < 0.5 else -1)
                tokens.append((v & 0xFFFF) | (pos << 16) | (b << 20))
        m["tok_off"], m["tok_cnt"] = first, len(tokens) - first
    return serialize(L, capi, hdr, ft, mbs, tokens, split)


def make_stream(w, h, frames, seed, all_bpred=False, segment_maps=True):
    """-> IVF bytes"""
    from alfalfa_b200 import capi
    L = capi.lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    return ivf(w, h, [make_frame(rng, L, capi, w, h, i, saved, all_bpred, segment_maps) for i in range(frames)])


if __name__ == "__main__":
    if len(sys.argv) < 5:
        sys.exit(__doc__)
    data = make_stream(int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]) if len(sys.argv) > 5 else 1)
    open(sys.argv[1], "wb").write(data)
    print("%s: %d bytes" % (sys.argv[1], len(data)))
