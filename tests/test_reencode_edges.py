"""The re-encoding prediction streams of tools/make_edge_stream.py (make_reencodable; re-encoded on the GPU by
tests/test_gpu_reencode_edges.py) on the CPU: they are deterministic, carry what they are meant to carry -- counted
in the records the oracle parsed -- and the oracle decodes them to the stored answer of the unmodified reference
decoder (tests/reference_answers.py)."""
import collections
import os
import sys

import pytest

import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_edge_stream as E  # noqa: E402


def _parsed(data):
    w, h, frames = O.read_ivf(data)
    od = O.OracleDecoder(w, h)
    for f in frames:
        od.decode(f, want_planes=False)
        yield od.parsed()


@pytest.mark.parametrize("name", ["shapes_17x17", "mv_edges_96x48", "coeffs_64x64"])
def test_generator_is_deterministic(name):
    assert E.make_reencodable(name) == E.make_reencodable(name)
    assert E.make_reencodable(name, previous=True) == E.make_reencodable(name, previous=True)
    assert E.make_reencodable(name) != E.make_reencodable(name, previous=True)


def test_streams_carry_what_they_are_meant_to(capsys):
    """SPLITMV and 16 x 16 windows in every edge class, luma and chroma; q index 0 frames; on every shape intra
    (B_PRED) macroblocks of inter frames in column 0 and in the last column, and past column 32 (the second word of
    k_reenc_intra's bitmask) wherever there are more than 32 columns"""
    seen = collections.Counter()
    for name in E.reencode_names():
        for p in _parsed(E.make_reencodable(name)):
            d = p.desc
            if name.startswith("coeffs"):
                seen["coeffs: q index 0 frame"] += int(d.quant[1] == 4)   # y_ac factor 4
            if d.key_frame:
                continue
            if name.startswith("mv_edges"):
                for path, plane, _, cls, _ in E.windows_of_frame(d, p.mbs, p.split):
                    seen[("window", path, plane, cls)] += 1
            if name.startswith("shapes"):
                cols = d.mb_cols
                for i, m in enumerate(p.mbs):
                    col = i % cols
                    for where in {"column 0" if col == 0 else None, "last column" if col == cols - 1 else None,
                                  "past column 32" if col >= 32 else None} - {None}:
                        if m["ref_frame"] == E.REF_CURRENT:
                            seen[(name, where, "intra")] += 1
                            seen[(name, where, "B_PRED")] += int(m["y_mode"] == E.B_PRED)
    with capsys.disabled():
        print("\nre-encoding prediction streams (count):")
        for k in sorted(seen, key=str):
            print("  %-70s %d" % (k, seen[k]))
    want = ([("shapes_%dx%d" % s, where, kind) for s in E.REENCODE_SHAPES for where in ("column 0", "last column")
             for kind in ("intra", "B_PRED")] +
            [("shapes_%dx%d" % s, "past column 32", "B_PRED") for s in E.REENCODE_SHAPES if s[0] > 512] +
            [("window", path, plane, cls) for path in ("16x16", "split") for plane in "YC" for cls in E.CLASSES] +
            ["coeffs: q index 0 frame"])
    missing = [k for k in want if not seen[k]]
    assert not missing, missing


@pytest.mark.parametrize("previous", [False, True], ids=["stream", "previous"])
@pytest.mark.parametrize("name", E.reencode_names())
def test_oracle_equals_the_unmodified_reference_decoder(name, previous):
    import reference_answers as R
    data = E.make_reencodable(name, previous)
    want = R.ask("ref_dump", ["shown", "{s.ivf}"], {"s.ivf": data})["-"]
    assert R.digests([O.decode_ivf_display(data)]) == want
