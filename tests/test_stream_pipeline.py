"""The pipeline streams of tools/make_pipeline_stream.py on the CPU (tests/test_gpu_stream_pipeline.py decodes them on
the GPU): they are deterministic, the oracle decodes them to the unmodified reference decoder's stored answers, the
density streams reach the token density the capacity rule of Engine::token_cap_for has to cover (and the rule covers
it), and the sizemix streams drive the token arena of vp8gpu_decode_ivf through its wrap and wait branches
(tests/pipeline_model.py, the allocator restated)."""
import ctypes as C
import os
import sys

import pytest

import oracle_lib as O
import pipeline_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_pipeline_stream as P  # noqa: E402

_cache = {}


def _stream(name):
    if name not in _cache:
        _cache[name] = P.make_with_partitions(name)
    return _cache[name]


@pytest.mark.parametrize("name", [n for n in P.names() if n != P.DENSITY_1080])
def test_generator_is_deterministic(name):
    assert P.make(name) == _stream(name)[0]


@pytest.mark.parametrize("name", P.names())
def test_oracle_equals_the_unmodified_reference_decoder_on_pipeline_streams(name):
    """the oracle's display output of every pipeline stream equals the reference decoder's (its stored answer)"""
    import reference_answers as R
    data = _stream(name)[0]
    want = R.ask("ref_dump", ["shown", "{s.ivf}"], {"s.ivf": data})["-"]
    assert R.digests([O.decode_ivf_display(data)]) == want


def _density_records(name):
    """per frame: (tokens, partition bytes, tokens before the last coded macroblock, macroblocks), from the records of
    the host front end (vp8gpu_parse_frame)"""
    import numpy as np
    from alfalfa_b200 import capi
    L = capi.lib()
    data, nparts = _stream(name)
    w, h, frames = O.read_ivf(data)
    st, pf = C.c_void_p(), C.c_void_p()
    capi.check(L.vp8gpu_state_create(w, h, C.byref(st)))
    capi.check(L.vp8gpu_parsed_create(C.byref(pf)))
    out = []
    try:
        for f, p in zip(frames, nparts):
            assert L.vp8gpu_parse_frame(st, f, len(f), pf) == 0
            desc = L.vp8gpu_parsed_desc(pf).contents
            n_mbs = desc.mb_cols * desc.mb_rows
            mbs = np.frombuffer(C.string_at(L.vp8gpu_parsed_mbs(pf), n_mbs * 32), dtype=capi.MB_DTYPE)
            coded = np.flatnonzero(mbs["tok_cnt"])
            before_last = int(mbs["tok_off"][coded[-1]]) if len(coded) else 0
            out.append((int(desc.n_tokens), M.partition_bytes(f, p), before_last, n_mbs))
    finally:
        L.vp8gpu_parsed_destroy(pf)
        L.vp8gpu_state_destroy(st)
    return out


def test_density_streams_reach_the_densest_tokens_and_the_capacity_rule_covers_them(capsys):
    """k_tokens flags an overflow as soon as a coded macroblock starts with fewer than 400 tokens left of the frame's
    capacity; token_cap_for gives a frame of B partition bytes 9 * (B + 16, rounded up to 256) + 1024 tokens, at most
    400 per macroblock.  The density streams must come close to the format's limit (a token is at least its sign bit
    at p = 128: about 8 per byte), and at every frame the capacity must leave the 400 for its last coded macroblock."""
    best, margins = 0.0, []
    with capsys.disabled():
        print("\npipeline streams: tokens per partition byte (largest), capacity margin (smallest) per stream")
        for name in [n for n in P.names() if n.startswith(("density", "densemix"))]:
            recs = _density_records(name)
            dens = max(t / b for t, b, _, _ in recs if b)
            margin = min(M.token_cap_for(b, n) - (before + 400) for t, b, before, n in recs if t)
            best = max(best, dens)
            margins.append((margin, name))
            print("  %-24s %.3f tokens/byte  margin %d tokens" % (name, dens, margin))
        print("  densest %.3f tokens/byte; smallest margin %d tokens (%s)" % (best, min(margins)[0], min(margins)[1]))
    assert best >= 7.5
    assert min(margins)[0] >= 0, min(margins)


# (stream, slots, arena) cases whose wrap and wait branches the GPU test claims to exercise: arena None = plan()'s
# default for one worker with memory to spare (slots x the largest frame), 0 = VP8GPU_TOK_ARENA=0 (the floor)
SLOTS = [4, 5, 7, 16, 96]
ALLOC_STREAM = "sizemix_96x64"


def model_counters(name, slots, chunk=None, arena=None, copies=1):
    """what VP8GPU_TRACE prints for one worker decoding `copies` copies of the stream: (plan, counters)"""
    data, nparts = _stream(name)
    w, h, frames = O.read_ivf(data)
    n_mbs = ((w + 15) // 16) * ((h + 15) // 16)
    pl = M.plan(slots, max(len(f) for f in frames), n_mbs, chunk=chunk, arena=arena)
    return pl, M.simulate(M.needs_per_gop(frames * copies, nparts * copies, n_mbs), pl[0], pl[1], pl[2])


@pytest.mark.parametrize("name", [n for n in P.names() if n.startswith("sizemix")])
@pytest.mark.parametrize("arena", [None, 0], ids=["default_arena", "floor_arena"])
@pytest.mark.parametrize("slots", SLOTS)
def test_allocator_model_wraps_and_waits(name, slots, arena):
    """every frame takes a piece; the arena wraps to offset 0 in every case, and it waits for the oldest frame's pixel
    kernels in every case but the largest ring at the default size (96 slots x the largest frame: no waits)"""
    (s, chunk, cap, worst), n = model_counters(name, slots, arena=arena)
    _, _, frames = O.read_ivf(_stream(name)[0])
    assert n["takes"] == len(frames)
    assert n["wraps"] > 0
    if slots == 96 and arena is None:
        assert n["waits"] == 0
    else:
        assert n["waits"] > 0
    # the chunk size changes the launches, not the placement
    for c in (1, max(1, slots // 2)):
        assert model_counters(name, slots, chunk=c, arena=arena)[1] == n


def test_allocator_model_restates_the_capacity_rule():
    """token_cap_for at the byte rule, the block rule and the 256-byte steps"""
    assert M.token_cap_for(0, 1000) == 256 * 9 + 1024
    assert M.token_cap_for(240, 1000) == 256 * 9 + 1024
    assert M.token_cap_for(241, 1000) == 512 * 9 + 1024
    assert M.token_cap_for(10 ** 6, 99) == 99 * 400
    # plan(): the floor is half the slots plus two of the largest frame, the default every slot's worth
    s, c, cap, worst = M.plan(16, 5000, 99)
    assert (c, cap) == (5, 16 * worst)
    assert M.plan(16, 5000, 99, arena=0)[2] == 10 * worst
    assert M.plan(16, 5000, 99, arena=12)[2] == 12 * worst
