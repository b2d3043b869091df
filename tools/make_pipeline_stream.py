#!/usr/bin/env python3
"""Pipeline streams: VP8 streams aimed at the whole-stream decoder with device-side tokens (vp8gpu_decode_ivf), written
with the product's bitstream writer like tools/make_edge_stream.py.  Seeded and deterministic:

  density_WxH_pN   as many tokens per partition byte as VP8 allows, on N DCT partitions: every coded block carries a
                   +-1 at every position, with optimised token probabilities, so "not EOB", "non-zero" and "ONE" cost
                   almost nothing and a token costs little more than its sign bit at p = 128.  Key and inter frames,
                   with Y2 (16 x 16 modes) and without (B_PRED, SPLITMV), every macroblock coded or about half of them
                   (there the byte rule of Engine::token_cap_for binds, not the 400 tokens per macroblock)
  densemix_WxH     half-coded density frames among much larger frames (+-2114 everywhere: 20-bit tokens), so that in
                   vp8gpu_decode_ivf a density frame's token piece is sized for itself and neighbours other frames'
  densegop_WxH     one GOP of 56 near-largest frames: more than an arena at its floor holds for a worker with 96 slots
  sizemix_WxH      GOPs of 1, 2, 3, 31, 32, 33, 95, 96, 97 and 200 frames (chunk boundaries, slot-ring wrap, GOPs longer
                   than the ring) mixing runs of near-largest dense frames, mid-size frames, all-skip inter frames of a
                   few bytes and hidden ALTREF frames, so that the token arena of every worker wraps and waits
  largestlast_WxH  GOPs of 30 frames whose last frame is by far the largest (its tokens are decoded last in a k_tokens
  largestfirst_WxH launch), or whose key frame is (decoded last, and the rest of its launch ready long before)
                   (order_names(): a catalogue of their own, checked against the host-token path, not stored answers)

usage: python tools/make_pipeline_stream.py NAME OUT.ivf        (NAME one of names())
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_feature_stream as F  # noqa: E402
from make_feature_stream import B_PRED, NEWMV, REF_ALTREF, REF_CURRENT, REF_GOLDEN, REF_LAST, SPLIT_LAYOUTS, SPLITMV, ZEROMV  # noqa: E402

DENSITY_SIZES = [(16, 16), (176, 144), (640, 368)]
DENSITY_PARTS = [1, 2, 4, 8]
DENSITY_FRAMES = ["key", "y2", "no_y2", "half"]   # what each frame of a density stream codes
DENSITY_1080 = "density_1920x1080_p8"             # one key + inter pair at the bench's size
DENSEMIX_SIZES = [(176, 144)]
DENSEGOP = "densegop_640x368"                     # one GOP of DENSEGOP_FRAMES near-largest frames
DENSEGOP_FRAMES = 56
SIZEMIX_SIZES = [(96, 64), (176, 144)]
GOP_LENGTHS = [1, 2, 3, 31, 32, 33, 95, 96, 97, 200]
MAX_COEF = 2114


def _lib():
    from alfalfa_b200 import capi
    return capi.lib(), capi


def _template(has_y2):
    """pos << 16 | block << 20 of every position of every block of a macroblock, in the writer's order"""
    out = []
    for b in range(25 if has_y2 else 24):
        lo = 1 if (has_y2 and b < 16) else 0
        out += [(pos << 16) | (b << 20) for pos in range(lo, 16)]
    return np.array(out, dtype=np.uint32)


TEMPLATE = {True: _template(True), False: _template(False)}


def _frame(L, capi, rng, w, h, saved, key, log2_parts, pick, show=True, refresh_last=True, refresh_alt=False, value=1):
    """one frame; pick(rng, m) sets macroblock m's modes and returns whether it is coded.  Every coded macroblock
    carries +-value at every position of every block."""
    cols, rows = (w + 15) // 16, (h + 15) // 16
    hdr = capi.EncodeHeader()
    hdr.width, hdr.height = w, h
    hdr.key_frame, hdr.show_frame = int(key), int(show)
    hdr.y_ac_qi, hdr.loop_filter_level, hdr.sharpness = int(rng.integers(4, 100)), int(rng.integers(0, 40)), int(rng.integers(0, 8))
    hdr.optimize_token_probs = 1
    ft = capi.EncodeFeatures()
    ft.log2_partitions = log2_parts
    ft.refresh_last = int(key or refresh_last)
    ft.refresh_alternate = int(refresh_alt and not key)
    ft.refresh_entropy_probs = 1
    ft.saved_coef_probs = saved.ctypes.data
    mbs = np.zeros(cols * rows, dtype=capi.MB_DTYPE)
    split, pieces, n_tok = [], [], 0
    for i in range(cols * rows):
        m = mbs[i]
        coded = pick(rng, m, split)
        has_y2 = m["y_mode"] not in (B_PRED, SPLITMV)
        m["flags"] = 1 if has_y2 else 0
        if not coded:
            continue
        t = TEMPLATE[has_y2]
        signs = rng.integers(0, 2, size=len(t)).astype(bool)
        pieces.append(t | np.where(signs, (-value) & 0xFFFF, value).astype(np.uint32))
        m["tok_off"], m["tok_cnt"] = n_tok, len(t)
        n_tok += len(t)
    tokens = np.concatenate(pieces).tolist() if pieces else []
    return F.serialize(L, capi, hdr, ft, mbs, tokens, split)


def _intra(rng, m, y2):
    m["ref_frame"] = REF_CURRENT
    m["y_mode"] = int(rng.integers(0, 4)) if y2 else B_PRED
    m["uv_mode"] = int(rng.integers(0, 4))
    if m["y_mode"] == B_PRED:
        m["b_modes"] = int(sum(int(rng.integers(0, 10)) << (4 * k) for k in range(16)))


def _inter(rng, m, split, y2, refs=(REF_LAST, REF_GOLDEN, REF_ALTREF)):
    m["ref_frame"] = refs[int(rng.integers(0, len(refs)))]
    if y2:
        m["y_mode"] = NEWMV if rng.random() < 0.6 else ZEROMV
        if m["y_mode"] == NEWMV:
            m["mv_x"], m["mv_y"] = int(rng.integers(-40, 41)) * 2, int(rng.integers(-40, 41)) * 2
        return
    mv = np.zeros((16, 2), dtype=np.int16)
    for members in SPLIT_LAYOUTS[int(rng.integers(0, 4))]:
        v = (int(rng.integers(-24, 25)) * 2, int(rng.integers(-24, 25)) * 2)
        for k in range(16):
            if members >> k & 1:
                mv[k] = v
    m["y_mode"], m["split_idx"] = SPLITMV, len(split)
    m["mv_x"], m["mv_y"] = int(mv[15, 0]), int(mv[15, 1])
    split.append(mv)


def _pick(kind):
    """macroblock chooser of a frame kind: key (intra, both), y2 / no_y2 (inter frame, one kind of block), mixed
    (inter frame, both), half (inter frame, both, about half the macroblocks coded), skip (nothing coded)"""
    def pick(rng, m, split):
        y2 = {"y2": True, "no_y2": False}.get(kind, bool(rng.random() < 0.5))
        if kind == "key":
            _intra(rng, m, y2)
            return True
        if kind == "skip":
            m["ref_frame"], m["y_mode"] = REF_LAST, ZEROMV
            return False
        if rng.random() < 0.25:
            _intra(rng, m, y2)
        else:
            _inter(rng, m, split, y2)
        return kind != "half" or bool(rng.random() < 0.5)
    return pick


# ---------------------------------------------------------------- density
def make_density(w, h, parts, seed, kinds=DENSITY_FRAMES):
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    log2 = parts.bit_length() - 1
    return F.ivf(w, h, [_frame(L, capi, rng, w, h, saved, k == "key", log2, _pick(k)) for k in kinds]), [parts] * len(kinds)


def make_densemix(w, h, seed):
    """key frame and large frames at +-2114, with half-coded density frames between them"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    chunks, nparts = [], []
    for i, kind in enumerate(["key", "mixed", "half", "mixed", "half", "half", "mixed", "half"]):
        value = 1 if kind == "half" else MAX_COEF
        chunks.append(_frame(L, capi, rng, w, h, saved, kind == "key", i % 4, _pick(kind), value=value))
        nparts.append(1 << i % 4)
    return F.ivf(w, h, chunks), nparts


def make_densegop(w, h, seed):
    """one GOP of near-largest frames, enough of them that a worker with 96 slots outruns an arena at its floor (room
    for 50 of them)"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    kinds = ["key"] + ["mixed"] * (DENSEGOP_FRAMES - 1)
    return F.ivf(w, h, [_frame(L, capi, rng, w, h, saved, k == "key", i % 4, _pick(k)) for i, k in enumerate(kinds)]), \
        [1 << i % 4 for i in range(len(kinds))]


# ---------------------------------------------------------------- sizemix
def gop_kinds(length, rng):
    """frame kinds of one GOP: runs of dense frames, all-skip frames, mid-size ones, now and then a hidden ALTREF"""
    kinds = ["key"]
    while len(kinds) < length:
        r = rng.random()
        run = int(rng.integers(1, 13))
        if r < 0.4:
            kinds += ["mixed"] * run
        elif r < 0.65:
            kinds += ["skip"] * run
        elif r < 0.9:
            kinds += ["half"] * run
        else:
            kinds += ["altref"]
    return kinds[:length]


def make_sizemix(w, h, seed):
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    chunks, nparts = [], []
    for g, length in enumerate(GOP_LENGTHS):
        for i, kind in enumerate(gop_kinds(length, rng)):
            log2 = (g + i) % 4
            nparts.append(1 << log2)
            if kind == "altref":   # hidden, becomes ALTREF only
                chunks.append(_frame(L, capi, rng, w, h, saved, False, log2, _pick("half"), show=False, refresh_last=False,
                                     refresh_alt=True))
            else:
                chunks.append(_frame(L, capi, rng, w, h, saved, kind == "key", log2, _pick(kind)))
    return F.ivf(w, h, chunks), nparts


# ---------------------------------------------------------------- largest frame last / first
ORDER_SIZES = [(176, 144)]
ORDER_GOPS, ORDER_GOP_LEN = 4, 30


def make_order(w, h, seed, largest_last):
    """GOPs of small frames (skip and half-coded at +-1) with one frame at +-2114 everywhere: the last or the key frame"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    chunks = []
    for g in range(ORDER_GOPS):
        for i in range(ORDER_GOP_LEN):
            big = i == (ORDER_GOP_LEN - 1 if largest_last else 0)
            kind = "key" if i == 0 else ("mixed" if big else ("skip" if (g + i) % 3 == 0 else "half"))
            chunks.append(_frame(L, capi, rng, w, h, saved, i == 0, (g + i) % 4, _pick(kind), value=MAX_COEF if big else 1))
    return F.ivf(w, h, chunks), [1 << (g + i) % 4 for g in range(ORDER_GOPS) for i in range(ORDER_GOP_LEN)]


# ---------------------------------------------------------------- catalogue
def names():
    return (["density_%dx%d_p%d" % (w, h, p) for w, h in DENSITY_SIZES for p in DENSITY_PARTS] + [DENSITY_1080] +
            ["densemix_%dx%d" % s for s in DENSEMIX_SIZES] + [DENSEGOP] + ["sizemix_%dx%d" % s for s in SIZEMIX_SIZES])


def order_names():
    return ["largest%s_%dx%d" % (o, w, h) for o in ("last", "first") for w, h in ORDER_SIZES]


def make(name):
    """IVF bytes of the pipeline stream `name`"""
    return make_with_partitions(name)[0]


def make_with_partitions(name):
    """(IVF bytes, DCT partitions of every frame) of the pipeline stream `name`"""
    parts = name.split("_")
    w, h = (int(x) for x in parts[1].split("x"))
    if parts[0] == "density":
        p = int(parts[2][1:])
        if (w, h) == (1920, 1080):
            return make_density(w, h, p, 600 + p, kinds=["key", "mixed"])
        return make_density(w, h, p, 600 + w + p)
    if parts[0] == "densemix":
        return make_densemix(w, h, 700 + w)
    if parts[0] == "densegop":
        return make_densegop(w, h, 750 + w)
    if parts[0] == "sizemix":
        return make_sizemix(w, h, 800 + w)
    if parts[0] in ("largestlast", "largestfirst"):
        return make_order(w, h, 900 + w + (parts[0] == "largestfirst"), parts[0] == "largestlast")
    raise KeyError(name)


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__ + "\nnames: " + " ".join(names() + order_names()))
    data = make(sys.argv[1])
    open(sys.argv[2], "wb").write(data)
    print("%s: %d bytes" % (sys.argv[2], len(data)))
