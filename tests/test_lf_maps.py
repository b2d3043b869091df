"""The designed loop-filter cases of tests/lf_maps.py on the CPU (tests/test_gpu_loopfilter.py decodes them on the
GPU): their coverage is asserted, not assumed -- every path of k_loopfilter_band that band_paths() names is taken
by some case, the filter changes the lines that are handed from macroblock to macroblock and from row to row, and a
frame level of 0 leaves the picture as reconstructed whatever the macroblock levels say."""
import collections

import numpy as np

import lf_maps as M


def test_band_paths_cover_every_class(capsys):
    """band_paths() over every job of every shape of tests/test_gpu_loopfilter.py: no class is left empty"""
    seen = collections.Counter()
    for cols, rows in M.SHAPES:
        for j in M.batch(cols, rows, M.shape_seed(cols, rows)):
            if j.desc.loop_filter_level:
                seen.update(M.band_paths(j.lf_map))
    with capsys.disabled():
        print("\nk_loopfilter_band paths over the designed cases (macroblocks, rows or frames):")
        for k in M.all_classes():
            print("  %-60s %d" % (" ".join(str(x) for x in k), seen[k]))
    assert set(seen) <= set(M.all_classes()), set(seen) - set(M.all_classes())
    missing = [k for k in M.all_classes() if not seen[k]]
    assert not missing, missing


def test_band_paths_on_a_hand_checked_map():
    """a 3-row map whose paths are counted by hand: row 1 (band position 1) filters columns 2, 3, 9, 10 and 17 below
    a row 0 that filters columns 1 and 9; row 2 filters nothing"""
    m = np.zeros((3, 20), np.uint8)
    m[0, [1, 9]] = 20
    m[1, [2, 3, 9, 10, 17]] = 20
    got = M.band_paths(m)
    # row 1, column: abits (row 0 filters c-1, c, c+1), left taken over or fetched, top-left corner
    #   2: 0b001 fetched, corner of slot 1 written by column 1     3: 0b000 taken over
    #   9: 0b010 fetched, corner of slot 0 written by column 9     10: 0b001 taken over
    #   17: 0b000 fetched; slot 17 % 8 = 1 and the corner's slot 0 hold row 0's words of column 9: stale
    assert got[("abits", 1, "have_left", 0)] == 1 and got[("abits", 0, "have_left", 1)] == 1
    assert got[("abits", 2, "have_left", 0)] == 1 and got[("abits", 1, "have_left", 1)] == 1
    assert got[("abits", 0, "have_left", 0)] == 1
    assert got[("corner", "ring via c-1")] == 1 and got[("corner", "ring via c")] == 1 and got[("corner", "frame")] == 1
    assert got[("top words", "ring", "ring via c")] == 1 and got[("top words", "frame", "frame")] == 4
    assert got[("stale slot", "left words")] == 1 and got[("stale slot", "right word")] == 1
    assert got[("stale slot", "corner")] == 1
    assert got[("empty row at band position", 2)] == 1 and got[("frame ends at band position", 2)] == 1
    assert got[("gap >= LF_RING",)] == 1  # row 0 (feeds the ring) skips from column 1 to 9
    assert got[("band position", 0)] == 2 and got[("band position", 1)] == 5
    assert not got[("top row reads the frame",)] and not got[("word boundary", "c-1 in the word before", 0)]


def test_filter_changes_the_lines_handed_over():
    """On a 12 x 9 frame of every kind (inter, key) at every sharpness, filtered with the oracle one macroblock at a
    time in raster order: in at least 90 % of the filtered macroblocks that have a left and a top edge, the filter
    has changed the macroblock's bottom 4 lines by the time its row is done (what the ring hands to the row below)
    and its right 4 columns by the time it is done (what the next macroblock takes over).  Otherwise a word taken
    from the wrong place would often hold the right bytes and a wrong hand-over would go unnoticed."""
    cols, rows = 12, 9
    ok = n = 0
    for key in (False, True):
        for sharp in range(8):
            seed = 500 + 10 * sharp + key
            rng = np.random.default_rng(seed)
            lv = M.levels_of(np.ones((rows, cols), bool), rng).reshape(-1)
            j = M.make_job(cols, rows, lv, seed, key_frame=key, sharpness=sharp)
            ref = M.reference_picture(cols, rows, seed)
            state = []  # state[k]: the first k macroblocks filtered
            for k in range(rows * cols + 1):
                part = lv.copy()
                part[k:] = 0
                state.append(M.oracle_decode(j, ref, lf_level=part))
            pre = state[0]
            for r in range(1, rows):
                for c in range(1, cols):
                    row_done, mb_done = state[(r + 1) * cols], state[r * cols + c + 1]
                    bottom = any((row_done[p][s * r + 3 * s // 4:s * (r + 1), s * c:s * (c + 1)] !=
                                  pre[p][s * r + 3 * s // 4:s * (r + 1), s * c:s * (c + 1)]).any() for p, s in ((0, 16), (1, 8), (2, 8)))
                    right = any((mb_done[p][s * r:s * (r + 1), s * c + 3 * s // 4:s * (c + 1)] !=
                                 pre[p][s * r:s * (r + 1), s * c + 3 * s // 4:s * (c + 1)]).any() for p, s in ((0, 16), (1, 8), (2, 8)))
                    ok += bottom and right
                    n += 1
    assert ok >= 0.9 * n, "%d of %d macroblocks" % (ok, n)


def test_frame_level_0_leaves_the_picture_untouched():
    """vp8o_loopfilter with loop_filter_level = 0 in the descriptor does nothing even where macroblock levels are
    non-zero (frame.cc:144); every batch carries such a job, which the kernels must skip (lf_enabled == 0)"""
    for cols, rows in ((9, 5), (33, 6)):
        jobs = M.batch(cols, rows, M.shape_seed(cols, rows))
        off = [j for j in jobs if j.desc.loop_filter_level == 0]
        assert len(off) == 1 and (off[0].lf_map != 0).mean() > 0.3
        ref = M.reference_picture(cols, rows, M.shape_seed(cols, rows))
        filtered, unfiltered = M.oracle_decode(off[0], ref), M.oracle_decode(off[0], ref, filtered=False)
        assert all(np.array_equal(a, b) for a, b in zip(filtered, unfiltered))
        # ... while the same records with the level on are changed by the filter
        on = M.make_job(cols, rows, off[0].lf_map, 0)
        on.mbs, on.tokens, on.split = off[0].mbs, off[0].tokens, off[0].split
        assert not all(np.array_equal(a, b) for a, b in zip(M.oracle_decode(on, ref), unfiltered))


def test_records_are_well_formed():
    """what the decode kernels assume of parsed records: tokens inside the stream, distinct (block, position) per
    macroblock, no luma DC beside a Y2 block, no Y2 block without Y2, split entries for every SPLITMV; and every
    kind of macroblock and level is present"""
    kinds = collections.Counter()
    for cols, rows in ((17, 9), (65, 3)):
        for j in M.batch(cols, rows, M.shape_seed(cols, rows)):
            d, mbs, t = j.desc, j.mbs, j.tokens
            assert d.n_tokens == t.size and d.n_split == j.split.shape[0]
            assert (mbs["tok_off"].astype(np.int64) + mbs["tok_cnt"] <= t.size).all()
            for m in mbs:
                tt = t[m["tok_off"]:m["tok_off"] + m["tok_cnt"]]
                blk, pos = (tt >> 20) & 31, (tt >> 16) & 15
                assert len(set(zip(blk.tolist(), pos.tolist()))) == len(tt)
                y2 = bool(m["flags"] & M.HAS_Y2)
                assert y2 or not (blk == 24).any()
                assert not y2 or not ((blk < 16) & (pos == 0)).any()
                assert (tt & 0xFFFF).all()
                if m["y_mode"] == M.SPLITMV:
                    assert not y2 and m["split_idx"] < d.n_split
                kinds[(int(d.key_frame), int(m["y_mode"]), int(m["tok_cnt"] > 0))] += 1
                kinds[("level", int(m["lf_level"]))] += 1
    for k in [(1, M.DC_PRED, 1), (1, M.TM_PRED, 1), (0, M.ZEROMV, 0), (0, M.ZEROMV, 1), (0, M.SPLITMV, 0)]:
        assert kinds[k], k
    for lv in (0,) + M.LEVELS:
        assert kinds[("level", lv)], lv
