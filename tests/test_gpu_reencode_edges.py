"""Re-encoding (Encoder::update_residues, reencode_as_interframe) at the edges of its kernels, byte for byte against
the unmodified reference's Encoder::reencode (oracle/_ref/ref_reencode, its stored answers): the bench's 1080p
workload, and the prediction streams of tools/make_edge_stream.py written without segmentation (make_reencodable:
degenerate frame shapes, prediction windows on every side of the plane edges, q index 0 frames, and the saturate
streams: q index 0 throughout, flat or ZEROMV predictors) re-encoded towards the stream's own pictures, saturated
pictures (a 0 / 255 checkerboard of 4 x 4 blocks whose phase flips every frame; uniform noise whose top-left
macroblock codes all 384 coefficients) and, on the saturate streams, the pictures the receiver predicts (every
residue 0) -- each as an extra-frame chunk (options 2 + 4) and as a whole chunk (options 1 + 4:
reencode_as_interframe runs the decision loop at the shape).  On the saturate streams the emitted frames are parsed
and the extremes asserted: a Y2 token near the +-2047 clamp, a macroblock of 384 tokens, no token at all.  The receiver's state comes
from another seed of the same family at the same size, so LAST, GOLDEN and ALTREF differ from the stream's own.

Also run under the SIMT emulator in both thread orders (tests/test_simt_emulation.py), without the 1080p and the
16383-pixel-wide cases."""
import os
import sys

import numpy as np
import pytest

import oracle_lib as O
import reference_answers as R
from test_gpu_reencode import ROOT, _decoded_targets, product_reencode_cases, reference_reencode, state_after

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_edge_stream as E  # noqa: E402

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("VP8GPU_SIMT_EMULATED"))
NAMES = [n for n in E.reencode_names() if not (EMULATED and "16383" in n)]
TARGETS = ("own", "checker", "noise")   # + "zero" on the saturate streams


def checker(w, h, i):
    """0 / 255 in 4 x 4 blocks, the phase flipping with the frame index: against a reference that holds the previous
    frame's checkerboard every residue is +-255"""
    def plane(pw, ph):
        y, x = np.mgrid[0:ph, 0:pw]
        return np.where(((x >> 2) + (y >> 2) + i) & 1, 255, 0).astype(np.uint8)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    return plane(w, h), plane(cw, ch), plane(cw, ch)


def fdct16(d):
    """vp8m::fdct16 (the reference's DCTCoefficients::subtract_dct) on a 4 x 4 residue, raster order"""
    t = [0] * 16
    for i in range(4):
        a1, b1 = (d[4 * i] + d[4 * i + 3]) * 8, (d[4 * i + 1] + d[4 * i + 2]) * 8
        c1, d1 = (d[4 * i + 1] - d[4 * i + 2]) * 8, (d[4 * i] - d[4 * i + 3]) * 8
        t[4 * i:4 * i + 4] = a1 + b1, (c1 * 2217 + d1 * 5352 + 14500) >> 12, a1 - b1, (d1 * 2217 - c1 * 5352 + 7500) >> 12
    o = [0] * 16
    for i in range(4):
        a1, b1, c1, d1 = t[i] + t[i + 12], t[i + 4] + t[i + 8], t[i + 4] - t[i + 8], t[i] - t[i + 12]
        o[i], o[i + 8] = (a1 + b1 + 7) >> 4, (a1 - b1 + 7) >> 4
        o[i + 4] = ((c1 * 2217 + d1 * 5352 + 12000) >> 16) + (d1 != 0)
        o[i + 12] = (d1 * 2217 - c1 * 5352 + 51000) >> 16
    return o


def fwht16(x):
    """vp8m::fwht16 (the reference's wht) of the sixteen luma DCs"""
    t = [0] * 16
    for i in range(4):
        a1, d1 = (x[4 * i] + x[4 * i + 2]) * 4, (x[4 * i + 1] + x[4 * i + 3]) * 4
        c1, b1 = (x[4 * i + 1] - x[4 * i + 3]) * 4, (x[4 * i] - x[4 * i + 2]) * 4
        t[4 * i:4 * i + 4] = a1 + d1 + (a1 != 0), b1 + c1, b1 - c1, a1 - d1
    o = [0] * 16
    for i in range(4):
        a1, d1, c1, b1 = t[i] + t[i + 8], t[i + 4] + t[i + 12], t[i + 4] - t[i + 12], t[i] - t[i + 8]
        for k, v in enumerate((a1 + d1, b1 + c1, b1 - c1, a1 - d1)):
            o[i + 4 * k] = (v + (v < 0) + 3) >> 3
    return o


def _dense_block(rng, first):
    """uniform noise over a 4 x 4 block whose residue against 128 has |coefficient| >= 4 (q index 0: a token) at
    every position from `first` on"""
    while True:
        b = rng.integers(0, 256, size=16)
        c = fdct16([int(v) - 128 for v in b])
        if all(abs(v) >= 4 for v in c[first:]):
            return b.reshape(4, 4), c[0]


def noise(w, h, i):
    """uniform noise over 0..255; the top-left macroblock (whose predictor is flat 128 in the saturate streams'
    inter frames) is drawn again until every one of its 384 coefficients at q index 0 is a token: 15 AC per luma
    block, 16 Y2 (|value| >= 8), 16 per chroma block"""
    rng = np.random.default_rng(700 + i)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    y, u, v = (rng.integers(0, 256, size=s, dtype=np.uint8) for s in ((h, w), (ch, cw), (ch, cw)))
    if w >= 16 and h >= 16:
        blocks = [_dense_block(rng, 1) for _ in range(16)]
        while not all(abs(c) >= 8 for c in fwht16([dc for _, dc in blocks])):
            blocks[int(rng.integers(0, 16))] = _dense_block(rng, 1)
        for k, (b, _) in enumerate(blocks):
            y[4 * (k >> 2):4 * (k >> 2) + 4, 4 * (k & 3):4 * (k & 3) + 4] = b
        for plane in (u, v):
            for k in range(4):
                plane[4 * (k >> 1):4 * (k >> 1) + 4, 4 * (k & 1):4 * (k & 1) + 4] = _dense_block(rng, 0)[0]
    return y, u, v


def zero_residue(w, h, chunks, state):
    """what a receiver in `state` decodes from the inter frames of a stream without coefficients and without loop
    filter: the prediction of every macroblock, so that re-encoding them as an extra-frame chunk leaves every
    residue 0.  (The key frame is not re-encoded there; its target is the first inter frame's.)"""
    from alfalfa_b200 import Context, Decoder
    ctx = Context(w, h, max_frames=16)
    d = Decoder.deserialize(ctx, state)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    out = []
    for c in chunks[1:]:
        _, r = d.get_frame_output(c)
        b = np.frombuffer(r.display_bytes(), np.uint8)
        out.append((b[:w * h].reshape(h, w).copy(), b[w * h:w * h + cw * ch].reshape(ch, cw).copy(),
                    b[w * h + cw * ch:].reshape(ch, cw).copy()))
        r.release()
    del d
    ctx.close()
    return out[:1] + out


def targets_of(kind, w, h, chunks, state):
    if kind == "own":
        return _decoded_targets(w, h, chunks)
    if kind == "zero":
        return zero_residue(w, h, chunks, state)
    return [(checker if kind == "checker" else noise)(w, h, i) for i in range(len(chunks))]


def emitted_tokens(w, h, state, frames):
    """per emitted frame: (tokens per macroblock, values of its Y2 tokens), parsed by a receiver in `state`"""
    from alfalfa_b200 import Context, Decoder
    ctx = Context(w, h, max_frames=16)
    d = Decoder.deserialize(ctx, state)
    out = []
    for f in frames:
        p = d.parse_frame(f)
        d.decode_frame(p)
        mbs, tok, _ = p.arrays()
        vals = ((tok.astype(np.int64) & 0xFFFF) ^ 0x8000) - 0x8000
        out.append((mbs["tok_cnt"].astype(int), vals[((tok >> 20) & 31) == 24]))
    del d
    ctx.close()
    return out


def case_inputs(name):
    w, h, chunks = O.read_ivf(E.make_reencodable(name))
    _, _, prev = O.read_ivf(E.make_reencodable(name, previous=True))
    return w, h, chunks, state_after(w, h, prev, len(prev))


def check(w, h, want, got, what):
    assert isinstance(got, tuple), "%s: the product refused the case: %s" % (what, got)
    frames, in_step = got
    assert len(frames) == len(want), what
    for i, (a, b) in enumerate(zip(R.digests(frames), want)):
        assert a == b, "%s frame %d: %d vs %d bytes, or different bytes" % (what, i, a[1], b[1])
    assert in_step, what


def kinds_of(name):
    """the zero-residue target needs a stream without coefficients and loop filter (the saturate family) and a size
    of whole macroblocks (a target only covers the display; beyond it the encoder replicates its last column / row)"""
    w, h = (int(x) for x in name.rsplit("_", 1)[1].split("x"))
    return TARGETS + (("zero",) if name.startswith("saturate") and w % 16 == 0 and h % 16 == 0 else ())


@pytest.mark.parametrize("name", NAMES)
def test_prediction_streams_reencode_like_the_reference(name):
    """every target kind, extra-frame chunk (kf_q_weight 0.75) and whole chunk (0.5), in one child process; on the
    saturate streams, after equality, the extremes the targets are made for: a Y2 token of |value| >= 2000 (checker),
    a macroblock with all 384 coefficients coded (noise), no token at all (zero residue)"""
    w, h, chunks, state = case_inputs(name)
    kinds = [k for k in kinds_of(name) for _ in range(2)]
    cases = [(w, h, targets_of(kind, w, h, chunks, state), chunks, state, kfw, extra)
             for kind in kinds_of(name) for kfw, extra in ((0.75, True), (0.5, False))]
    results = product_reencode_cases(cases)
    for kind, case, got in zip(kinds, cases, results):
        check(w, h, reference_reencode(*case), got, "%s target, %s" % (kind, "extra-frame chunk" if case[6] else "whole chunk"))
    if not name.startswith("saturate"):
        return
    for kind, case, (frames, _) in zip(kinds, cases, results):
        if not case[6]:
            continue   # the whole chunk starts with the decision loop's frame: extremes are asserted on the others
        parsed = emitted_tokens(w, h, state, frames)
        y2 = max(int(np.abs(v).max()) if len(v) else 0 for _, v in parsed)
        densest = max(int(c.max()) for c, _ in parsed)
        print("%s %s target: largest |Y2 token| %d, most tokens in a macroblock %d" % (name, kind, y2, densest))
        if kind == "checker":
            assert y2 >= 2000, y2
        elif kind == "noise":
            assert densest == 384, densest
        elif kind == "zero":
            assert densest == 0, densest


def test_bench_workload_reencodes_like_the_reference():
    """tools/reencode_bench.py's inputs (1080p, 12 frames of one clip against the state 8 frames of another leave
    behind, kf_q_weight 0.75) as an extra-frame chunk, as it measures them, and as a whole chunk"""
    if EMULATED:
        pytest.skip("1080p: on the GPU only")
    import reencode_bench
    from alfalfa_b200 import Context
    w, h = 1920, 1080
    ctx = Context(w, h, max_frames=32)
    state, chunk, _, targets = reencode_bench.bench_inputs(ctx)
    ctx.close()
    cases = [(w, h, targets, chunk, state, 0.75, extra) for extra in (True, False)]
    for case, got in zip(cases, product_reencode_cases(cases, timeout=600)):
        check(w, h, reference_reencode(*case), got, "extra-frame chunk" if case[6] else "whole chunk")
