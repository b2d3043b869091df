"""The edge streams of tools/make_edge_stream.py on the CPU (tests/test_gpu_edges.py decodes them on the GPU):
their coverage is asserted, not assumed -- every boundary class and filter phase of the mv_edges windows, every
coefficient extreme of the coeffs streams is counted in the records the oracle parsed -- and what the oracle decodes
them to equals the stored answer of the unmodified reference decoder (tests/reference_answers.py)."""
import collections
import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_edge_stream as E  # noqa: E402


def _parsed_frames(data):
    w, h, frames = O.read_ivf(data)
    od = O.OracleDecoder(w, h)
    for f in frames:
        od.decode(f, want_planes=False)
        yield od.parsed()


@pytest.mark.parametrize("size", E.MV_EDGE_SIZES)
def test_mv_edges_records_carry_the_intended_vectors(size):
    """the writer may code a vector as NEAREST / NEAR; what the decoder parses is the vector that was chosen"""
    data, intended = E.make_mv_edges(size[0], size[1], E.MV_EDGE_FRAMES, 400 + size[0])
    n = 0
    for i, p in enumerate(_parsed_frames(data)):
        for mbi, mv in intended[i].items():
            m = p.mbs[mbi]
            got = p.split[m["split_idx"]] if m["y_mode"] == E.SPLITMV else np.tile([m["mv_x"], m["mv_y"]], (16, 1))
            assert np.array_equal(got, mv), "frame %d macroblock %d" % (i, mbi)
            n += 1
    assert n > 100


def test_mv_edges_cover_every_boundary_class_and_phase(capsys):
    """Every coded window of the mv_edges streams, classified along each axis by where it lies against its plane
    (E.CLASSES) and by its filter phase, with the window formulas of k_inter: 16 x 16 (luma, and chroma from the
    rounded vector) and SPLITMV 4 x 4 blocks (luma, and chroma from the rounded sum of four luma vectors).  Every
    cell path x plane x axis x class x phase must be coded at least once; the counts are printed."""
    seen = collections.Counter()
    rounding = collections.Counter()
    for w, h in E.MV_EDGE_SIZES:
        data = E.make("mv_edges_%dx%d" % (w, h))
        for p in _parsed_frames(data):
            if p.desc.key_frame:
                continue
            seen.update(E.windows_of_frame(p.desc, p.mbs, p.split))
            for m in p.mbs:
                if m["ref_frame"] != E.REF_CURRENT and m["y_mode"] == E.SPLITMV:
                    v = p.split[m["split_idx"]].astype(int)
                    for q in range(4):
                        a = (q >> 1) * 8 + (q & 1) * 2
                        s = int(v[a, 0] + v[a + 1, 0] + v[a + 4, 0] + v[a + 5, 0])
                        rounding[("neg" if s < 0 else "pos", "exact" if s % 8 == 0 else "rounded")] += 1
    with capsys.disabled():
        print("\nmv_edges windows per (path, plane, axis, class): count at each phase")
        for path in ("16x16", "split"):
            for plane in "YC":
                for axis in "xy":
                    for cls in E.CLASSES:
                        print("  %-5s %s %s %-11s %s" % (path, plane, axis, cls,
                                                         " ".join("%d:%d" % (ph, seen[(path, plane, axis, cls, ph)]) for ph in E.PHASES[plane])))
        print("  SPLITMV chroma sums (sign, rounding): %s" % dict(rounding))
    missing = [c for c in E.all_cells() if not seen[c]]
    assert not missing, "cells never coded: %s" % missing
    assert all(rounding[(s, r)] for s in ("neg", "pos") for r in ("exact", "rounded")), dict(rounding)


def test_coeffs_cover_the_coefficient_extremes(capsys):
    """Counted in the parsed records with each segment's dequantisation factors (FrameDesc.quant): dense macroblocks
    (every position of every block coded), the largest DCT_CAT6 magnitude, products that wrap int16, macroblocks
    with tokens that all dequantise to 0 mod 2^16 (filtered inner edges, no residual), Y2-only macroblocks, DC-only
    blocks whose (dc + 4) >> 3 is 0, the smallest and largest factors, loop-filter level 63 at every sharpness and
    macroblock levels clamped to 0 and 63."""
    seen = collections.Counter()
    for name in [n for n in E.names() if n.startswith("coeffs_")]:
        for p in _parsed_frames(E.make(name)):
            d = p.desc
            q = np.array(d.quant, dtype=np.int64).reshape(4, 6)
            if d.loop_filter_level == 63:
                seen["frame level 63, sharpness %d" % d.sharpness] += 1
            seen["factor 4 (q 0)"] += int((q == 4).any())
            seen["factor 284 (q 127)"] += int((q == 284).any())
            for m in p.mbs:
                seen["macroblock level 0"] += int(m["lf_level"] == 0)
                seen["macroblock level 63"] += int(m["lf_level"] == 63)
                if not m["tok_cnt"]:
                    continue
                t = p.tokens[m["tok_off"]:m["tok_off"] + m["tok_cnt"]]
                blk, pos, val = (t >> 20) & 31, (t >> 16) & 15, (t & 0xFFFF).astype(np.int16).astype(np.int64)
                # vp8gpu_quant: y_dc, y_ac, y2_dc, y2_ac, uv_dc, uv_ac (include/vp8gpu.h)
                qs = q[m["segment_id"]]
                fac = np.where(blk < 16, np.where(pos > 0, qs[1], qs[0]),
                               np.where(blk < 24, np.where(pos > 0, qs[5], qs[4]), np.where(pos > 0, qs[3], qs[2])))
                prod = val * fac
                seen["dense macroblock"] += int(len(t) == 384)
                seen["token +-2114"] += int((np.abs(val) == 2114).any())
                seen["product wraps int16"] += int(((prod < -32768) | (prod > 32767)).any())
                seen["tokens all dequantise to 0 mod 2^16 (Y2 mode)"] += int((prod % 65536 == 0).all() and (m["flags"] & 1)
                                                                             and m["lf_level"] > 0)
                seen["Y2 tokens only"] += int((blk == 24).all())
                for b in set(blk.tolist()):
                    sel = blk == b
                    if (pos[sel] == 0).all() and (b >= 16 or not (m["flags"] & 1)):
                        dc = ((prod[sel][0] + 32768) % 65536) - 32768
                        seen["DC-only block, (dc + 4) >> 3 == 0"] += int((dc + 4) >> 3 == 0)
    with capsys.disabled():
        print("\ncoeffs features (count):")
        for k in sorted(seen):
            print("  %-48s %d" % (k, seen[k]))
    want = (["frame level 63, sharpness %d" % s for s in range(8)] +
            ["factor 4 (q 0)", "factor 284 (q 127)", "macroblock level 0", "macroblock level 63", "dense macroblock",
             "token +-2114", "product wraps int16", "tokens all dequantise to 0 mod 2^16 (Y2 mode)", "Y2 tokens only",
             "DC-only block, (dc + 4) >> 3 == 0"])
    assert not [k for k in want if not seen[k]], [k for k in want if not seen[k]]


@pytest.mark.parametrize("name", E.names())
def test_host_front_end_matches_the_oracle_on_edge_streams(name):
    """vp8gpu_parse_frame's records (the host front end every GPU decode starts from) equal the oracle's"""
    from alfalfa_b200 import capi
    L = capi.lib()
    data = E.make(name)
    w, h, frames = O.read_ivf(data)
    od = O.OracleDecoder(w, h)
    st, pf = C.c_void_p(), C.c_void_p()
    capi.check(L.vp8gpu_state_create(w, h, C.byref(st)))
    capi.check(L.vp8gpu_parsed_create(C.byref(pf)))
    for i, f in enumerate(frames):
        od.decode(f, want_planes=False)
        op = od.parsed()
        assert L.vp8gpu_parse_frame(st, f, len(f), pf) == 0
        desc = L.vp8gpu_parsed_desc(pf).contents
        assert bytes(desc) == bytes(op.desc), "frame %d desc" % i
        assert C.string_at(L.vp8gpu_parsed_mbs(pf), desc.mb_cols * desc.mb_rows * 32) == op.mbs.tobytes(), "frame %d mbs" % i
        if desc.n_tokens:
            assert C.string_at(L.vp8gpu_parsed_tokens(pf), desc.n_tokens * 4) == op.tokens.tobytes(), "frame %d tokens" % i
        if desc.n_split:
            assert C.string_at(L.vp8gpu_parsed_split(pf), desc.n_split * 64) == op.split.tobytes(), "frame %d split" % i
    L.vp8gpu_parsed_destroy(pf)
    L.vp8gpu_state_destroy(st)


@pytest.mark.parametrize("name", E.names())
def test_oracle_equals_the_unmodified_reference_decoder_on_edge_streams(name):
    """the oracle's display output of every edge stream equals the reference decoder's (its stored answer)"""
    import reference_answers as R
    data = E.make(name)
    want = R.ask("ref_dump", ["shown", "{s.ivf}"], {"s.ivf": data})["-"]
    assert R.digests([O.decode_ivf_display(data)]) == want
