"""Designed loop-filter inputs for the decode kernels (TEST INFRASTRUCTURE, CPU only; tests/test_lf_maps.py checks
their coverage, tests/test_gpu_loopfilter.py decodes them on the GPU).

A job is a vp8gpu_frame_desc + vp8gpu_mb records + tokens + split vectors built by hand, so that which macroblocks
the loop filter touches, and at which level, comes from a chosen map instead of a bitstream:
  - inter frames: ZEROMV from LAST (the picture before the loop filter is the uploaded reference, Y2 coded, no
    tokens: inner edges skipped), mixed with SPLITMV of zero vectors (no Y2: inner edges filtered) and ZEROMV with a
    few small tokens;
  - key frames: TM_PRED / DC_PRED intra macroblocks with small random tokens (key-frame hev thresholds).
The reference picture is a smooth base + per-4x4 offsets + noise + saturated patches, so that the filter changes
the lines that k_loopfilter_band hands from row to row (checked in tests/test_lf_maps.py).

band_paths() restates where k_loopfilter_band (alfalfa_b200/csrc/kernels.cu) takes each input of a macroblock
from, so the tests can assert that the maps drive every one of its paths."""
import collections
import ctypes as C

import numpy as np

import oracle_lib as O

LF_BAND, LF_RING = 4, 8  # kernels.cu k_loopfilter_band
WORD = 32                # columns per bitmask word (one __ballot_sync)
LEVELS = (1, 14, 15, 19, 20, 39, 40, 63)  # either side of the hev (15, 20 inter, 40) and interior steps
DC_PRED, TM_PRED, ZEROMV, SPLITMV = 0, 3, 7, 9
REF_CURRENT, REF_LAST = 0, 1
HAS_Y2 = 1
ZIGZAG_RANK = np.argsort([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])  # raster position -> coding order
QUANT = (8, 10, 16, 20, 8, 10)  # y_dc, y_ac, y2_dc, y2_ac, uv_dc, uv_ac


# ---------------------------------------------------------------------------------------------------- maps
def _rows_of(rows, cols, f):
    return np.array([[bool(f(r, c)) for c in range(cols)] for r in range(rows)], dtype=bool).reshape(rows, cols)


def maps(cols, rows, seed):
    """[(name, bool array rows x cols: macroblock filtered)] -- every map of the list at this shape"""
    rng = np.random.default_rng(seed)
    out = [("dense", np.ones((rows, cols), bool)),
           ("none", np.zeros((rows, cols), bool)),
           ("alternating", _rows_of(rows, cols, lambda r, c: (r + c) % 2 == 0))]
    for p in (0.1, 0.5, 0.9):
        out.append(("bernoulli%.1f" % p, rng.random((rows, cols)) < p))
    # stale slot: the row above filters c - 8 (and, in the second map, c - 9), never c or c + 1; the row below
    # filters c, so ring slot c % LF_RING holds the row above's words of an earlier column
    out.append(("stale", _rows_of(rows, cols, lambda r, c: c % 16 == (8 * r) % 16)))
    out.append(("stale2", _rows_of(rows, cols, lambda r, c: (c - 8 * (r % 2)) % 16 in ((0, 1) if r % 2 == 0 else (1,)))))
    # runs and gaps of 9..12 columns: every slot is reused inside a run, the ring drains across a gap
    runs = np.zeros((rows, cols), bool)
    for r in range(rows):
        c, on = -int(rng.integers(0, 12)), bool(r % 2)
        while c < cols:
            n = int(rng.integers(LF_RING + 1, LF_RING + 5))
            if on:
                runs[r, max(c, 0):max(c + n, 0)] = True
            c, on = c + n, not on
    out.append(("runs", runs))
    # around the bitmask word boundaries (columns 31 / 32 / 33 and 63 / 64 / 65): every 3-column window, varied by row
    edge = np.zeros((rows, cols), bool)
    for r in range(rows):
        for b in (32, 64):
            for c in range(b - 3, min(b + 3, cols)):
                edge[r, c] = bool((r * 5 + (c - b + 3) * 3 + b) % 7 < 4) if c >= 0 else False
    out.append(("wordedge", edge))
    # one row without a filtered macroblock at each band position in turn (band b: position b % 4)
    empty = rng.random((rows, cols)) < 0.7
    for r in range(rows):
        if r % LF_BAND == (r // LF_BAND) % LF_BAND:
            empty[r] = False
    out.append(("emptyrows", empty))
    out.append(("firstcol", _rows_of(rows, cols, lambda r, c: c == 0)))
    out.append(("lastcol", _rows_of(rows, cols, lambda r, c: c == cols - 1)))
    return out


# level 1 rarely changes a noisy picture (interior limit 1): drawn less often than the others
LEVEL_P = np.array([0.3] + [1.0] * (len(LEVELS) - 1)) / (0.3 + len(LEVELS) - 1)


def levels_of(mask, rng):
    """per-macroblock lf_level: 0 where the map says unfiltered, else one of LEVELS"""
    return np.where(mask, rng.choice(np.array(LEVELS, np.uint8), size=mask.shape, p=LEVEL_P), 0).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------- records
def reference_picture(cols, rows, seed):
    """(Y, U, V) macroblock-aligned: smooth base + per-4x4 offsets 0..40 + noise +-2 + patches saturated at 0 / 255"""
    rng = np.random.default_rng(seed)
    planes = []
    for sub in (1, 2, 2):
        h, w = 16 * rows // sub, 16 * cols // sub
        yy, xx = np.mgrid[0:h, 0:w]
        base = 110 + 24 * np.sin(0.035 * xx * sub + 0.3 * sub) * np.cos(0.025 * yy * sub)
        bh, bw = (h + 3) // 4, (w + 3) // 4
        # mostly small steps between 4x4 blocks (filtered at every level), some up to 40 (filtered only at high levels)
        off = np.where(rng.random((bh, bw)) < 0.75, rng.integers(0, 5, size=(bh, bw)), rng.integers(0, 41, size=(bh, bw)))
        # noise +-2, mostly +-1, left out of 30 % of the 4x4 blocks (where level 1 with sharpness still filters)
        noisy = np.repeat(np.repeat(rng.random((bh, bw)) < 0.7, 4, 0), 4, 1)[:h, :w]
        noise = rng.choice(np.arange(-2, 3), size=(h, w), p=[0.05, 0.2, 0.5, 0.2, 0.05]) * noisy
        p = base + np.repeat(np.repeat(off, 4, 0), 4, 1)[:h, :w] + noise
        p = np.clip(p, 0, 255)
        for _ in range(max(1, (h * w) // 4096)):  # saturated patches
            y0, x0 = int(rng.integers(0, h)), int(rng.integers(0, w))
            p[y0:y0 + int(rng.integers(4, 24)), x0:x0 + int(rng.integers(4, 24))] = 255 * int(rng.integers(0, 2))
        planes.append(np.ascontiguousarray(p.astype(np.uint8)))
    return tuple(planes)


def _tokens(rng, n_mbs, with_tokens, y2):
    """tok_off, tok_cnt per macroblock and the token stream: 1..10 distinct small coefficients per macroblock with
    tokens, in block order and coding order inside a block like a parsed stream; with Y2 the luma blocks carry no DC"""
    idx = np.nonzero(with_tokens)[0]
    cnt = np.zeros(n_mbs, np.int64)
    if idx.size == 0:
        return np.zeros(n_mbs, np.uint32), cnt.astype(np.uint16), np.zeros(0, np.uint32)
    k = 10
    mb = np.repeat(idx, k)
    blk = rng.integers(0, 25, size=mb.size)
    has_y2 = y2[mb]
    blk = np.where(has_y2, blk, blk % 24)  # no Y2 block without Y2
    pos = rng.integers(0, 16, size=mb.size)
    pos = np.where(has_y2 & (blk < 16) & (pos == 0), 1 + rng.integers(0, 15, size=mb.size), pos)
    keep = rng.random(mb.size) < rng.uniform(0.15, 1.0, size=mb.size)
    keep[::k] = True  # at least one token per macroblock with tokens
    mb, blk, pos = mb[keep], blk[keep], pos[keep]
    key = (mb * 32 + blk) * 16 + ZIGZAG_RANK[pos]
    key, first = np.unique(key, return_index=True)  # distinct (block, position) per macroblock, sorted
    mb, blk, pos = mb[first], blk[first], pos[first]
    val = rng.integers(1, 4, size=mb.size) * rng.choice([-1, 1], size=mb.size)
    toks = ((val.astype(np.int64) & 0xFFFF) | (pos << 16) | (blk << 20)).astype(np.uint32)
    cnt = np.bincount(mb, minlength=n_mbs)
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return off.astype(np.uint32), cnt.astype(np.uint16), toks


class Job:
    """one frame's records (desc: oracle_lib.FrameDesc, mbs: MB_DTYPE, tokens, split) and a name for reports"""

    def __init__(self, desc, mbs, tokens, split, name):
        self.desc, self.mbs, self.tokens, self.split, self.name = desc, mbs, tokens, split, name

    @property
    def lf_map(self):
        return self.mbs["lf_level"].reshape(self.desc.mb_rows, self.desc.mb_cols)


def make_job(cols, rows, lf_level, seed, key_frame=False, sharpness=0, frame_level=40, name=""):
    """records of one frame whose macroblock levels are `lf_level` (rows x cols, uint8)"""
    rng = np.random.default_rng(seed)
    n = cols * rows
    mbs = np.zeros(n, O.MB_DTYPE)
    mbs["lf_level"] = np.asarray(lf_level, np.uint8).reshape(-1)
    split = np.zeros((0, 16, 2), np.int16)
    if key_frame:
        mbs["ref_frame"] = REF_CURRENT
        mbs["y_mode"] = rng.choice([DC_PRED, TM_PRED], size=n)
        mbs["uv_mode"] = rng.choice([DC_PRED, TM_PRED], size=n)
        mbs["flags"] = HAS_Y2
        with_tok = rng.random(n) < 0.95
    else:
        kind = rng.choice(3, size=n, p=[0.5, 0.25, 0.25])  # 0 ZEROMV, 1 SPLITMV of zero vectors, 2 ZEROMV + tokens
        mbs["ref_frame"] = REF_LAST
        mbs["y_mode"] = np.where(kind == 1, SPLITMV, ZEROMV)
        mbs["flags"] = np.where(kind == 1, 0, HAS_Y2)
        ns = int((kind == 1).sum())
        mbs["split_idx"] = np.where(kind == 1, np.cumsum(kind == 1) - 1, 0)
        split = np.zeros((ns, 16, 2), np.int16)
        with_tok = kind == 2
    off, cnt, toks = _tokens(rng, n, with_tok, (mbs["flags"] & HAS_Y2) != 0)
    mbs["tok_off"], mbs["tok_cnt"] = off, cnt
    d = O.FrameDesc()
    d.width, d.height = min(16 * cols, 16383), 16 * rows
    d.mb_cols, d.mb_rows = cols, rows
    d.key_frame, d.show_frame = int(key_frame), 1
    d.loop_filter_level, d.sharpness = frame_level, sharpness
    for s in range(4):
        d.quant[6 * s:6 * s + 6] = QUANT
    d.n_tokens, d.n_split = toks.size, split.shape[0]
    d.refresh_last = 1
    return Job(d, mbs, np.ascontiguousarray(toks, np.uint32), np.ascontiguousarray(split), name)


def batch(cols, rows, seed):
    """one launch's jobs at this shape: each map of maps() with its own levels, sharpness and key / inter flag, and
    one job whose frame level is 0 while its macroblock levels are not (its loop filter must not run)"""
    rng = np.random.default_rng(seed)
    jobs = []
    for i, (name, mask) in enumerate(maps(cols, rows, seed)):
        key = i % 4 == 3
        jobs.append(make_job(cols, rows, levels_of(mask, rng), seed * 100 + i, key_frame=key, sharpness=i % 8,
                             frame_level=int(rng.integers(1, 64)), name="%s/%s/sharp%d" % (name, "key" if key else "inter", i % 8)))
    jobs.append(make_job(cols, rows, levels_of(rng.random((rows, cols)) < 0.5, rng), seed * 100 + 99, frame_level=0,
                         sharpness=3, name="frame-level-0"))
    return jobs


def bench_batch(n_jobs=64, cols=120, rows=68, seed=1080):
    """the bench's shape: n_jobs 1920x1080 frames with different Bernoulli maps in one launch"""
    rng = np.random.default_rng(seed)
    jobs = []
    for i in range(n_jobs):
        p = 0.1 + 0.8 * i / max(n_jobs - 1, 1)
        key = i % 8 == 5
        j = make_job(cols, rows, levels_of(rng.random((rows, cols)) < p, rng), seed + i, key_frame=key, sharpness=i % 8,
                     frame_level=int(rng.integers(1, 64)), name="bernoulli%.2f/%s" % (p, "key" if key else "inter"))
        j.desc.width, j.desc.height = 1920, 1080
        jobs.append(j)
    return jobs


# ---------------------------------------------------------------------------------------------------- oracle
def _new_raster(cols, rows, planes=None):
    L = O.lib()
    r = L.vp8o_raster_new(16 * cols, 16 * rows)
    if planes is not None:
        for dst, src in zip((r.contents.y, r.contents.u, r.contents.v), planes):
            C.memmove(dst, np.ascontiguousarray(src).ctypes.data, src.size)
    return r


def oracle_decode(job, ref_planes, filtered=True, lf_level=None):
    """(Y, U, V) of vp8o_reconstruct (+ vp8o_loopfilter) on the job's records, LAST = GOLDEN = ALTREF = ref_planes;
    lf_level replaces the records' levels for the loop filter only"""
    L = O.lib()
    d = job.desc
    ref = _new_raster(d.mb_cols, d.mb_rows, ref_planes)
    out = _new_raster(d.mb_cols, d.mb_rows)
    tok = job.tokens.ctypes.data if job.tokens.size else None
    sp = job.split.ctypes.data if job.split.size else None
    L.vp8o_reconstruct(C.byref(d), job.mbs.ctypes.data, tok, sp, ref, ref, ref, out)
    if filtered:
        mbs = job.mbs
        if lf_level is not None:
            mbs = mbs.copy()
            mbs["lf_level"] = np.asarray(lf_level, np.uint8).reshape(-1)
        L.vp8o_loopfilter(C.byref(d), mbs.ctypes.data, out)
    planes = O.raster_planes(out)
    L.vp8o_raster_free(ref)
    L.vp8o_raster_free(out)
    return planes


# ---------------------------------------------------------------------------------------------------- model
def band_paths(lf_map):
    """Counter of the paths k_loopfilter_band takes on a frame whose macroblock levels are lf_map (rows x cols; only
    level != 0 matters).  A plain restatement of the kernel (line numbers: alfalfa_b200/csrc/kernels.cu):
      ("band position", k)          a filtered macroblock in a row at band position row % LF_BAND = k  (1316-1318)
      ("abits", a, "have_left", h)  a row with the row above in its CTA (ring_in, 1326): the row above filters
                                    c - 1, c, c + 1 (bits 0, 1, 2; 1393-1401); the left columns come from the previous
                                    macroblock (h = 1) or are fetched (1391, 1431-1446)
      ("top words", L, R)           where the 4 lines above come from (1425-1426): the left words from the ring
                                    (written by c) or the frame; the right word (luma x 12-15, chroma x 4-7) from the
                                    ring written by c + 1, by c (its flush_right, 1504-1517), or from the frame
      ("corner", S)                 the top-left corner of a fetched left edge (1436-1445): ring slot c - 1 as written
                                    by c (its left word, 1492 / 1501), by c - 1 (flush_right), or the frame
      ("stale slot", part)          the ring slot read holds the row above's words of an earlier column (c - 8, c - 7,
                                    ...), so the part must come from the frame: left words, right word, corner
      ("top row reads the frame",)  row > 0 at band position 0: waits on lf_progress, reads every word through L2
                                    (1405, 1426)
      ("gap >= LF_RING",)           a row that feeds the ring (ring_out, 1327) skips LF_RING or more columns: its slot
                                    wait (1476) lands on columns the row below may already have passed
      ("word boundary", side, bit)  abits' neighbour c - 1 / c + 1 lies in the previous / next 32-column word of
                                    above_word (the shuffle at 1398), with that neighbour filtered (bit 1) or not
      ("frame ends at band position", k)   the last row is at band position k: rows past mb_rows return (1318) and
                                    the row above it does not feed the ring (1327)
      ("empty row at band position", k)    a row with nothing to filter (it only publishes, 1353-1354)"""
    m = np.asarray(lf_map) != 0
    rows, cols = m.shape
    seen = collections.Counter()
    seen[("frame ends at band position", (rows - 1) % LF_BAND)] += 1
    for r in range(rows):
        pos = r % LF_BAND
        ring_in = pos > 0
        ring_out = pos < LF_BAND - 1 and r + 1 < rows
        marked = np.nonzero(m[r])[0].tolist()
        if not marked:
            seen[("empty row at band position", pos)] += 1
        if ring_out and any(b - a >= LF_RING for a, b in zip(marked, marked[1:])):
            seen[("gap >= LF_RING",)] += 1
        above = m[r - 1] if r > 0 else None
        # last column whose words the row above has written into each ring slot so far (as the kernel walks c up)
        prev = -2
        for c in marked:
            seen[("band position", pos)] += 1
            have_left = prev == c - 1
            prev = c
            if r > 0 and not ring_in:
                seen[("top row reads the frame",)] += 1
            if not ring_in:
                continue
            a = 0
            for d in (-1, 0, 1):
                if 0 <= c + d < cols and above[c + d]:
                    a |= 1 << (d + 1)
            seen[("abits", a, "have_left", int(have_left))] += 1
            left_src = "ring" if a & 2 else "frame"
            right_src = "ring via c+1" if a & 4 else ("ring via c" if a & 2 else "frame")
            seen[("top words", left_src, right_src)] += 1
            # slot c % LF_RING: written by column x of the row above (its own words if x = c mod 8, its left word as
            # the right word of x - 1 if x = c + 1 mod 8); an earlier such x means stale words
            older = [x for x in range(max(0, c - 2 * LF_RING), c) if above[x] and (x - c) % LF_RING in (0, 1)]
            older_own = [x for x in older if (x - c) % LF_RING == 0]
            if not a & 2 and older_own:
                seen[("stale slot", "left words")] += 1
            if not a & 6 and older:
                seen[("stale slot", "right word")] += 1
            if c > 0 and not have_left:
                corner = "ring via c" if a & 2 else ("ring via c-1" if a & 1 else "frame")
                seen[("corner", corner)] += 1
                stale = [x for x in range(max(0, c - 1 - 2 * LF_RING), c - 1) if above[x] and (x - c + 1) % LF_RING in (0, 1)]
                if not a & 3 and stale:
                    seen[("stale slot", "corner")] += 1
            if c % WORD == 0 and c > 0:
                seen[("word boundary", "c-1 in the word before", int(above[c - 1]))] += 1
            if c % WORD == WORD - 1 and c + 1 < cols:
                seen[("word boundary", "c+1 in the word after", int(above[c + 1]))] += 1
    return seen


def all_classes():
    """every class band_paths can report"""
    out = [("band position", k) for k in range(LF_BAND)]
    out += [("abits", a, "have_left", h) for a in range(8) for h in (0, 1)]
    out += [("top words", "ring", "ring via c+1"), ("top words", "ring", "ring via c"),
            ("top words", "frame", "ring via c+1"), ("top words", "frame", "frame")]
    out += [("corner", s) for s in ("ring via c", "ring via c-1", "frame")]
    out += [("stale slot", p) for p in ("left words", "right word", "corner")]
    out += [("top row reads the frame",), ("gap >= LF_RING",)]
    out += [("word boundary", s, b) for s in ("c-1 in the word before", "c+1 in the word after") for b in (0, 1)]
    out += [("frame ends at band position", k) for k in range(LF_BAND)]
    out += [("empty row at band position", k) for k in range(LF_BAND)]
    return out


# ---------------------------------------------------------------------------------------------------- cases
ROWS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 17)          # every residue mod LF_BAND, one to five bands
COLS = (1, 2, 3, 8, 9, 17, 33, 64, 65, 1024)        # 1024 = kMaxCols: 32 bitmask words, one per lane
SHAPES = [(c, r) for c in COLS for r in ROWS]


def shape_seed(cols, rows):
    return 7919 * cols + rows
