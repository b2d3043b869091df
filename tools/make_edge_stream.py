#!/usr/bin/env python3
"""Edge streams: VP8 streams aimed at the inputs where the decode kernels can go wrong, written with the product's
bitstream writer like tools/make_feature_stream.py.  Three seeded, deterministic families:

  shapes    the feature-stream mix at degenerate frame sizes: 1 x 1, one macroblock, one column, one row, two and
            three columns (B_PRED in every intra macroblock, so that the intra wavefront's lag binds), MB-aligned
            widths of 16 mod 32 (row pitch > width), the format's limits (16383 px = 1024 macroblocks), each also
            at an odd display size
  mv_edges  inter frames whose vectors are chosen per macroblock, not drawn: every prediction window (16 x 16 and
            the 4 x 4 blocks of SPLITMV, luma and the chroma vectors derived from it) is aimed at a boundary class
            of each plane edge (CLASSES) at each filter phase, on LAST, GOLDEN and ALTREF
  coeffs    dense blocks (all 16 positions of all 24 / 25 blocks) at +-2114, the largest DCT_CAT6 value, q indices
            0 and 127 with +-15 deltas and clamping segment overrides, DC-only blocks whose (dc + 4) >> 3 is 0,
            macroblocks with Y2 tokens only and macroblocks whose only tokens dequantise to 0 mod 2^16, loop-filter
            level 63 at every sharpness, deltas that push levels past 0 and 63

The windows are those of k_inter (alfalfa_b200/csrc/kernels.cu): a 16 x 16 window starts 2 pixels before the
vector's full-pixel position when its phase is not 0 and is then 21 pixels wide; a SPLITMV block's window always
starts 2 pixels before and is 9 wide.  In mv_edges only macroblocks at even rows and even columns carry vectors,
the others are intra-coded or ZEROMV, so the writer's vector prediction is 0 and every vector up to +-2046
eighth-pels can be coded as it was chosen.

Each family can also be written without segmentation (segment_maps=False), the form in which
Encoder::update_residues takes it (a prediction frame that updates the segment map is refused, and with segments the
reference's encoder drifts from its receiver, DESIGN.md section 5): make_reencodable() / reencode_names().

usage: python tools/make_edge_stream.py NAME OUT.ivf        (NAME one of names())
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_feature_stream as F  # noqa: E402
from make_feature_stream import (B_PRED, DC_PRED, NEWMV, REF_ALTREF, REF_CURRENT, REF_GOLDEN, REF_LAST, SPLIT_LAYOUTS,  # noqa: E402
                                 SPLITMV, ZEROMV)

# (width, height, all_bpred): 1 MB, 1 column, 1 row, 2 and 3 columns, MB-aligned width 16 mod 32, the format's limits
SHAPES = [(1, 1, False), (16, 16, False), (17, 17, False), (16, 512, False), (15, 511, False), (2048, 16, False),
          (2047, 15, False), (32, 480, True), (31, 479, True), (40, 480, True), (39, 473, True), (48, 48, False),
          (47, 45, False), (80, 32, False), (79, 31, False), (16383, 32, False), (16383, 17, False), (16, 16383, False),
          (15, 16383, False)]
SHAPE_FRAMES = 6   # key frame, inter frames, one hidden frame (index 4)
MV_EDGE_SIZES = [(80, 80), (96, 48)]   # MB-aligned width 16 mod 32 (pitch > width) and 0 mod 32
COEFF_SIZES = [(72, 40), (64, 64)]
MV_LIMIT = 2046   # largest vector component the writer codes as a delta (eighth-pels)

# where a window [X, X + n) lies against a plane [0, P): `far` pixels is "far outside"
CLASSES = ("far_lo", "outside_lo", "straddle_lo", "edge_lo", "inside_lo", "interior", "inside_hi", "edge_hi",
           "straddle_hi", "outside_hi", "far_hi")
FAR = {"Y": 200, "C": 100}   # chroma: the same displacement in the half-size plane
PHASES = {"Y": (0, 2, 4, 6), "C": tuple(range(8))}   # luma vectors are even eighth-pels


def classify(X, n, P, far):
    if X + n <= -far:
        return "far_lo"
    if X + n <= 0:
        return "outside_lo"
    if X < 0:
        return "straddle_lo"
    if X >= P + far:
        return "far_hi"
    if X >= P:
        return "outside_hi"
    if X + n > P:
        return "straddle_hi"
    if X == 0:
        return "edge_lo"
    if X + n == P:
        return "edge_hi"
    if X == 1:
        return "inside_lo"
    if X + n == P - 1:
        return "inside_hi"
    return "interior"


def target_origin(cls, n, P, far):
    return {"far_lo": -n - far, "outside_lo": -n - 1, "straddle_lo": -1, "edge_lo": 0, "inside_lo": 1,
            "interior": (P - n) // 2, "inside_hi": P - n - 1, "edge_hi": P - n, "straddle_hi": P - n + 1,
            "outside_hi": P, "far_hi": P + far}[cls]


def chroma_component(s):
    """chroma vector component from the sum of four luma components (kernels.cu chroma_component)"""
    s = (s + 0x8000 & 0xFFFF) - 0x8000
    return (s + 4) >> 3 if s >= 0 else -((-s + 4) >> 3)


def window(path, plane, base, mv):
    """(first pixel, width) of the window k_inter reads along one axis for a block at `base` with vector `mv`"""
    if path == "split":
        return base + (mv >> 3) - 2, 9
    full = 16 if plane == "Y" else 8
    return base + (mv >> 3) - (2 if mv & 7 else 0), full + (5 if mv & 7 else 0)


def vector_for(path, plane, base, X, phase):
    """the vector (eighth-pels of its plane) whose window along one axis starts at X with the given phase"""
    lead = 2 if (path == "split" or phase) else 0
    return ((X + lead - base) << 3) | phase


def windows_of_frame(desc, mbs, split):
    """every coded inter window of a parsed frame: (path, plane, axis, class, phase) per window and axis"""
    cols, rows = desc.mb_cols, desc.mb_rows
    size = {"Y": (16 * cols, 16 * rows), "C": (8 * cols, 8 * rows)}
    out = []

    def add(path, plane, bx, by, mvx, mvy):
        for axis, base, mv, P in (("x", bx, mvx, size[plane][0]), ("y", by, mvy, size[plane][1])):
            X, n = window(path, plane, base, mv)
            out.append((path, plane, axis, classify(X, n, P, FAR[plane]), mv & 7))
    for i, m in enumerate(mbs):
        if m["ref_frame"] == REF_CURRENT:
            continue
        row, col = divmod(i, cols)
        if m["y_mode"] != SPLITMV:
            mvx, mvy = int(m["mv_x"]), int(m["mv_y"])
            add("16x16", "Y", 16 * col, 16 * row, mvx, mvy)
            add("16x16", "C", 8 * col, 8 * row, chroma_component(4 * mvx), chroma_component(4 * mvy))
            continue
        v = split[m["split_idx"]].astype(int)
        for b in range(16):
            add("split", "Y", 16 * col + 4 * (b & 3), 16 * row + 4 * (b >> 2), v[b, 0], v[b, 1])
        for q in range(4):
            a = (q >> 1) * 8 + (q & 1) * 2
            sx, sy = (int(v[a, k] + v[a + 1, k] + v[a + 4, k] + v[a + 5, k]) for k in (0, 1))
            add("split", "C", 8 * col + 4 * (q & 1), 8 * row + 4 * (q >> 1), chroma_component(sx), chroma_component(sy))
    return out


def all_cells():
    return [(path, plane, axis, cls, ph) for path in ("16x16", "split") for plane in ("Y", "C") for axis in ("x", "y")
            for cls in CLASSES for ph in PHASES[plane]]


def _lib():
    from alfalfa_b200 import capi
    return capi.lib(), capi


def _header(capi, w, h, key, show, qi, lf, sharp):
    hdr = capi.EncodeHeader()
    hdr.width, hdr.height = w, h
    hdr.key_frame, hdr.show_frame = int(key), int(show)
    hdr.y_ac_qi, hdr.loop_filter_level, hdr.sharpness = qi, lf, sharp
    hdr.optimize_token_probs = 1
    return hdr


def _random_intra(rng, m):
    m["ref_frame"] = REF_CURRENT
    m["y_mode"] = int(rng.integers(0, 5))
    m["uv_mode"] = int(rng.integers(0, 4))
    if m["y_mode"] == B_PRED:
        m["b_modes"] = int(sum(int(rng.integers(0, 10)) << (4 * k) for k in range(16)))


def _sparse_tokens(rng, m, tokens):
    has_y2 = m["y_mode"] not in (B_PRED, SPLITMV)
    m["flags"] = 1 if has_y2 else 0
    if rng.random() < 0.4:
        return
    first = len(tokens)
    for b in sorted(int(x) for x in rng.choice(25 if has_y2 else 24, size=int(rng.integers(1, 5)), replace=False)):
        lo = 1 if (has_y2 and b < 16) else 0
        for pos in sorted(int(x) for x in rng.choice(np.arange(lo, 16), size=int(rng.integers(1, 4)), replace=False)):
            v = F.random_value(rng) * (1 if rng.random() < 0.5 else -1)
            tokens.append((v & 0xFFFF) | (pos << 16) | (b << 20))
    m["tok_off"], m["tok_cnt"] = first, len(tokens) - first


# ---------------------------------------------------------------- shapes
def make_shape(w, h, all_bpred, seed, segment_maps=True, frames=SHAPE_FRAMES):
    return F.make_stream(w, h, frames, seed, all_bpred=all_bpred, segment_maps=segment_maps)


# ---------------------------------------------------------------- mv_edges
class _Schedule:
    """the (class, phase) cells of one (path, plane, axis) still to be aimed at; refilled when used up"""

    def __init__(self, plane):
        self.plane = plane
        # the far classes first: only macroblocks near that edge can reach them
        self.full = [(c, p) for c in sorted(CLASSES, key=lambda c: not c.startswith("far")) for p in PHASES[plane]]
        self.todo = list(self.full)

    def take(self, path, base, P, to_luma, rng):
        """first pending cell whose vector the writer can code; -> plane vector"""
        for pool in (self.todo, self.full):
            order = list(pool) if pool is self.todo else [pool[int(k)] for k in rng.permutation(len(pool))]
            for cell in order:
                n = window(path, self.plane, 0, cell[1])[1]
                X = target_origin(cell[0], n, P, FAR[self.plane])
                v = vector_for(path, self.plane, base, X, cell[1])
                if abs(to_luma(v)) <= MV_LIMIT:
                    if pool is self.todo:
                        self.todo.remove(cell)
                        if not self.todo:
                            self.todo = list(self.full)
                    return v
        raise RuntimeError("no codable vector")


def _luma_subs(c, k):
    """four even luma components whose sum the chroma rounding maps to c; k picks the rounding case"""
    sums = [8 * c + d for d in (-4, -2, 0, 2, 4) if chroma_component(8 * c + d) == c]
    S = sums[k % len(sums)]
    base = (S // 8) * 2
    subs = [base + 2 if j < (S - 4 * base) // 2 else base for j in range(4)]
    assert sum(subs) == S and chroma_component(S) == c
    return subs


def make_mv_edges(w, h, frames, seed, segment_maps=True):
    """-> (IVF bytes, intended): intended[i] = {macroblock index: (16, 2) vectors} of every aimed macroblock of frame i.
    segment_maps=False: the key frame without segmentation (the inter frames never use it)"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    cols, rows = (w + 15) // 16, (h + 15) // 16
    PY, PC = (16 * cols, 16 * rows), (8 * cols, 8 * rows)
    sched = {(path, plane, axis): _Schedule(plane) for path in ("16x16", "split") for plane in "YC" for axis in "xy"}
    chunks, intended = [F.make_frame(rng, L, capi, w, h, 0, saved, segment_maps=segment_maps)], [{}]
    refs = [REF_LAST, REF_GOLDEN, REF_ALTREF]
    kinds = ["c16", "y16", "csplit", "c16", "ysplit", "csplit", "y16"]   # 7: every kind reaches every grid position
    nk = nref = nround = 0
    for index in range(1, frames):
        hdr = _header(capi, w, h, False, index % 6 != 4, int(rng.integers(10, 100)), int(rng.integers(0, 40)), index % 8)
        ft = capi.EncodeFeatures()
        ft.log2_partitions = index % 4
        ft.refresh_last = 1
        ft.refresh_golden = int(index % 4 == 1)
        ft.refresh_alternate = int(index % 5 == 2)
        ft.refresh_entropy_probs = 1
        ft.saved_coef_probs = saved.ctypes.data
        mbs = np.zeros(cols * rows, dtype=capi.MB_DTYPE)
        split, tokens, aimed = [], [], {}
        for i in range(cols * rows):
            m = mbs[i]
            row, col = divmod(i, cols)
            if row % 2 or col % 2:
                if rng.random() < 0.5:
                    _random_intra(rng, m)
                else:
                    m["ref_frame"], m["y_mode"] = refs[int(rng.integers(0, 3))], ZEROMV
                _sparse_tokens(rng, m, tokens)
                continue
            m["ref_frame"] = refs[nref % 3]
            nref += 1
            kind = kinds[nk % len(kinds)]
            nk += 1
            mv = np.zeros((16, 2), dtype=np.int16)
            if kind in ("y16", "c16"):
                plane = kind[0].upper()
                sc = 1 if plane == "Y" else 2   # luma vector per plane eighth-pel
                bx, by = (16 * col, 16 * row) if plane == "Y" else (8 * col, 8 * row)
                P = PY if plane == "Y" else PC
                vx = sched[("16x16", plane, "x")].take("16x16", bx, P[0], lambda v: sc * v, rng)
                vy = sched[("16x16", plane, "y")].take("16x16", by, P[1], lambda v: sc * v, rng)
                mv[:] = (sc * vx, sc * vy)
                m["y_mode"], m["mv_x"], m["mv_y"] = NEWMV, sc * vx, sc * vy
            elif kind == "ysplit":
                layout = SPLIT_LAYOUTS[nk // len(kinds) % 4]
                for members in layout:
                    b = (members & -members).bit_length() - 1
                    bx, by = 16 * col + 4 * (b & 3), 16 * row + 4 * (b >> 2)
                    v = (sched[("split", "Y", "x")].take("split", bx, PY[0], int, rng),
                         sched[("split", "Y", "y")].take("split", by, PY[1], int, rng))
                    for k in range(16):
                        if members >> k & 1:
                            mv[k] = v
            else:   # csplit: 16 partitions, each 2 x 2 luma group aimed through the chroma rounding
                for q in range(4):
                    a = (q >> 1) * 8 + (q & 1) * 2
                    cx = sched[("split", "C", "x")].take("split", 8 * col + 4 * (q & 1), PC[0], lambda v: 2 * abs(v) + 4, rng)
                    cy = sched[("split", "C", "y")].take("split", 8 * row + 4 * (q >> 1), PC[1], lambda v: 2 * abs(v) + 4, rng)
                    sx, sy = _luma_subs(cx, nround), _luma_subs(cy, nround + 1)
                    nround += 1
                    for j, b in enumerate((a, a + 1, a + 4, a + 5)):
                        mv[b] = (sx[j], sy[j])
            if kind in ("ysplit", "csplit"):
                m["y_mode"], m["split_idx"] = SPLITMV, len(split)
                m["mv_x"], m["mv_y"] = int(mv[15, 0]), int(mv[15, 1])
                split.append(mv)
            aimed[i] = mv
            _sparse_tokens(rng, m, tokens)
        chunks.append(F.serialize(L, capi, hdr, ft, mbs, tokens, split))
        intended.append(aimed)
    return F.ivf(w, h, chunks), intended


# ---------------------------------------------------------------- coeffs
MAX_COEF = 2114   # 67 + 2^11 - 1: DCT_CAT6
# per frame: base q index, sign of the +-15 deltas, absolute segment q indices (28 / 57: y_ac = 32 / 64, so that
# +-2048 / +-1024 dequantise to 0 mod 2^16) or relative ones that clamp
COEFF_FRAMES = [(127, +1, (0, 127, 28, 57)), (0, -1, (0, 127, 28, 57)), (127, +1, None), (0, -1, None),
                (64, -1, (127, 0, 28, 57)), (127, -1, (0, 127, 28, 57)), (0, +1, None), (90, +1, (0, 127, 57, 28))]
ZERO_TOKEN = {28: 2048, 57: 1024}   # y_ac 32 / 64


def make_coeffs(w, h, seed, segment_maps=True):
    """segment_maps=False: no segmentation (so no segment-map update in the inter frames)"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    cols, rows = (w + 15) // 16, (h + 15) // 16
    chunks = []
    kinds = ["dense_max", "zero_dequant", "dense_mixed", "y2_only", "dc_only_zero", "skip"]
    nk = 0
    for index, (qi, sign, seg_abs) in enumerate(COEFF_FRAMES):
        key = index == 0
        # level 63 at every sharpness over the two coeffs streams (w = 72, 64), other levels between
        hdr = _header(capi, w, h, key, index % 6 != 4, qi, 63 if (index + w) % 3 else int(rng.integers(1, 63)), index % 8)
        ft = capi.EncodeFeatures()
        ft.log2_partitions = index % 4
        ft.refresh_last = 1
        ft.refresh_entropy_probs = 1
        ft.saved_coef_probs = saved.ctypes.data
        for name in ("y_dc_delta", "y2_dc_delta", "y2_ac_delta", "uv_dc_delta", "uv_ac_delta"):
            setattr(ft, name, 15 * sign)
        ft.segmentation_enabled = ft.update_mb_segmentation_map = ft.update_segment_feature_data = 1
        if not segment_maps:
            ft.segmentation_enabled = ft.update_mb_segmentation_map = ft.update_segment_feature_data = 0
        ft.segment_feature_absolute = int(seg_abs is not None)
        for i in range(4):
            ft.segment_quant[i] = seg_abs[i] if seg_abs else (-127, 127, -15, 15)[i]
            ft.segment_lf[i] = (63, 0, 40, 63)[i] if seg_abs else (-63, 63, 20, -20)[i]
        for i in range(3):
            ft.segment_tree_probs[i] = 128
        ft.lf_delta_enabled = ft.lf_delta_update = 1
        for i in range(4):
            ft.ref_lf_delta[i] = (10, -63, 63, -20)[i] * (1 if index % 2 else -1)
            ft.mode_lf_delta[i] = (63, -63, 20, -63)[i] * (1 if index % 2 else -1)
        mbs = np.zeros(cols * rows, dtype=capi.MB_DTYPE)
        tokens = []
        for i in range(cols * rows):
            m = mbs[i]
            kind = kinds[nk % len(kinds)]
            nk += 1
            m["segment_id"] = int(rng.integers(0, 4))
            if kind == "zero_dequant":
                if not seg_abs:
                    kind = "dense_max"
                else:
                    m["segment_id"] = 2 + int(rng.integers(0, 2))
            # y2_only and zero_dequant need a mode with Y2 (inner edges are skipped only there without tokens)
            intra = key or rng.random() < 0.4
            if intra:
                _random_intra(rng, m)
                if kind in ("y2_only", "zero_dequant") and m["y_mode"] == B_PRED:
                    m["y_mode"] = DC_PRED
                if kind == "dc_only_zero" and rng.random() < 0.7:
                    m["y_mode"] = B_PRED
                    m["b_modes"] = int(sum(int(rng.integers(0, 10)) << (4 * k) for k in range(16)))
            else:
                m["ref_frame"] = [REF_LAST, REF_GOLDEN, REF_ALTREF][int(rng.integers(0, 3))]
                m["y_mode"] = NEWMV if rng.random() < 0.5 else ZEROMV
                if m["y_mode"] == NEWMV:
                    m["mv_x"], m["mv_y"] = int(rng.integers(-64, 65)) * 2, int(rng.integers(-64, 65)) * 2
            has_y2 = m["y_mode"] not in (B_PRED, SPLITMV)
            m["flags"] = 1 if has_y2 else 0
            if kind == "skip":
                continue
            first = len(tokens)
            for b in range(25 if has_y2 else 24):
                lo = 1 if (has_y2 and b < 16) else 0
                for pos in range(lo, 16):
                    if kind == "dense_max":
                        v = MAX_COEF * (1 if ((b + pos) % 3 or b % 5 == 0) else -1)
                    elif kind == "dense_mixed":
                        v = int(rng.choice([MAX_COEF, int(rng.integers(1, MAX_COEF + 1))])) * (1 if rng.random() < 0.5 else -1)
                    elif kind == "y2_only":
                        if b != 24:
                            continue
                        v = MAX_COEF * (1 if rng.random() < 0.6 else -1) if rng.random() < 0.8 else int(rng.integers(1, 100))
                    elif kind == "zero_dequant":
                        if b >= 16 or pos == 0 or rng.random() < 0.7:
                            continue
                        v = ZERO_TOKEN[seg_abs[m["segment_id"]]] * (1 if rng.random() < 0.5 else -1)
                    else:   # dc_only_zero: -1 at the smallest DC factor (4) dequantises to -4, (-4 + 4) >> 3 = 0
                        if pos != 0 or rng.random() < 0.3:
                            continue
                        v = -1
                    tokens.append((v & 0xFFFF) | (pos << 16) | (b << 20))
            if len(tokens) > first:
                m["tok_off"], m["tok_cnt"] = first, len(tokens) - first
        chunks.append(F.serialize(L, capi, hdr, ft, mbs, tokens, []))
    return F.ivf(w, h, chunks)


# ---------------------------------------------------------------- catalogue
def names():
    return (["shapes_%dx%d" % (w, h) for w, h, _ in SHAPES] + ["mv_edges_%dx%d" % s for s in MV_EDGE_SIZES] +
            ["coeffs_%dx%d" % s for s in COEFF_SIZES])


MV_EDGE_FRAMES = 36


def make(name):
    """IVF bytes of the edge stream `name` (mv_edges: also the intended vectors, make_mv_edges)"""
    family, size = name.rsplit("_", 1)
    w, h = (int(x) for x in size.split("x"))
    if family == "shapes":
        (k, bp), = [(k, bp) for k, (sw, sh, bp) in enumerate(SHAPES) if (sw, sh) == (w, h)]
        return make_shape(w, h, bp, 300 + k)
    if family == "mv_edges":
        return make_mv_edges(w, h, MV_EDGE_FRAMES, 400 + w)[0]
    if family == "coeffs":
        return make_coeffs(w, h, 500 + w)
    raise KeyError(name)


# ---------------------------------------------------------------- re-encoding
# Prediction streams for Encoder::update_residues / reencode_as_interframe: the families above written with
# segment_maps=False.
# (width, height): 1 MB, 1 column, 1 row (128 columns: four words of k_reenc_intra's intra bitmask), 2 and 3 columns
# (the wavefront's lag is clamped at the last column), an MB-aligned width of 16 mod 32 (row pitch > width), 1024
# columns (the bitmask's limit), each also at an odd display size.  Every intra macroblock uses B_PRED (the
# above-right edge and the lag only matter there; the other families carry the 16 x 16 modes), and 12 frames give
# intra macroblocks of inter frames in the first and the last column of every shape.
REENCODE_SHAPES = [(1, 1), (16, 16), (17, 17), (16, 512), (15, 511), (2048, 16), (2047, 15), (32, 64), (31, 63), (48, 64),
                   (47, 63), (208, 64), (207, 63), (16383, 32), (16383, 17)]
REENCODE_SHAPE_FRAMES = 12
SATURATE_SIZES = [(64, 48), (47, 33)]
SATURATE_FRAMES = 10
PREVIOUS_SEED = 1000   # the previous chunk: the same family at the same size, another seed


# ---------------------------------------------------------------- saturate
def make_saturate(w, h, seed, tokens):
    """q index 0 frames without deltas, loop filter off, one partition.  The key frame is DC_PRED throughout; in
    every inter frame macroblock 0 is DC_PRED (its predictor is flat: 128 in all planes, whatever came before), the
    others cycle through ZEROMV from LAST (with Y2), SPLITMV with zero vectors from LAST, B_PRED and ZEROMV again, and
    LAST is refreshed: a target against which every residue is +-255 or dense is a target that flips against the
    previous frame.  tokens=False: no coefficients at all, so that what a receiver decodes is exactly the prediction
    of every macroblock (the zero-residue targets); tokens=True: sparse coefficients (a picture that is not flat, for
    the previous chunk)."""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    saved = np.zeros(1056, dtype=np.uint8)
    cols, rows = (w + 15) // 16, (h + 15) // 16
    chunks = []
    for index in range(SATURATE_FRAMES):
        key = index == 0
        hdr = _header(capi, w, h, key, True, 0, 0, 0)
        ft = capi.EncodeFeatures()
        ft.refresh_last = 1
        ft.refresh_entropy_probs = 1
        ft.saved_coef_probs = saved.ctypes.data
        mbs = np.zeros(cols * rows, dtype=capi.MB_DTYPE)
        split, toks = [], []
        for i in range(cols * rows):
            m = mbs[i]
            kind = 0 if key or i == 0 else 1 + (i + index) % 4
            if kind == 0:
                m["ref_frame"], m["y_mode"], m["uv_mode"] = REF_CURRENT, DC_PRED, DC_PRED
            elif kind == 3:
                m["ref_frame"], m["y_mode"] = REF_CURRENT, B_PRED
                m["uv_mode"] = int(rng.integers(0, 4))
                m["b_modes"] = int(sum(int(rng.integers(0, 10)) << (4 * k) for k in range(16)))
            else:
                m["ref_frame"], m["y_mode"] = REF_LAST, ZEROMV
                if kind == 2:
                    m["y_mode"], m["split_idx"] = SPLITMV, len(split)
                    split.append(np.zeros((16, 2), dtype=np.int16))
            if tokens:
                _sparse_tokens(rng, m, toks)
            else:
                m["flags"] = 1 if m["y_mode"] not in (B_PRED, SPLITMV) else 0
        chunks.append(F.serialize(L, capi, hdr, ft, mbs, toks, split))
    return F.ivf(w, h, chunks)


def reencode_names():
    return (["shapes_%dx%d" % s for s in REENCODE_SHAPES] + ["mv_edges_%dx%d" % s for s in MV_EDGE_SIZES] +
            ["coeffs_%dx%d" % s for s in COEFF_SIZES] + ["saturate_%dx%d" % s for s in SATURATE_SIZES])


def make_reencodable(name, previous=False):
    """IVF bytes of the re-encoding prediction stream `name` (one of reencode_names()); previous: the stream whose
    state the re-encoded chunk starts from"""
    family, size = name.rsplit("_", 1)
    w, h = (int(x) for x in size.split("x"))
    seed = PREVIOUS_SEED if previous else 0
    if family == "shapes":
        k = REENCODE_SHAPES.index((w, h))
        return make_shape(w, h, True, 600 + k + seed, segment_maps=False, frames=REENCODE_SHAPE_FRAMES)
    if family == "mv_edges":
        return make_mv_edges(w, h, MV_EDGE_FRAMES, 400 + w + seed, segment_maps=False)[0]
    if family == "coeffs":
        return make_coeffs(w, h, 500 + w + seed, segment_maps=False)
    if family == "saturate":
        return make_saturate(w, h, 800 + w + seed, tokens=previous)
    raise KeyError(name)
