"""Whole-stream decode with device-side tokens (vp8gpu_decode_ivf) on the pipeline streams of
tools/make_pipeline_stream.py: every shown frame equals the oracle's bit for bit, and the decoder gives back every raster
it took, on
  - the density streams, the densest tokens VP8 allows, through parse_frame_device, a Decoder with device tokens and
    decode_ivf (also with density frames among much larger ones, so that their arena pieces are their own tight ones);
  - the sizemix streams with one worker, where the arena counters VP8GPU_TRACE prints equal the allocator model's
    (tests/pipeline_model.py) for every ring size, chunk size and both arena bounds;
  - the bench's shape with the arena at its floor (VP8GPU_TOK_ARENA=0), and a 1080p bench clip at 96 slots;
  - dispatcher and token-permit knobs, and worker kits reused across calls of different sizes."""
import hashlib
import os
import re
import sys

import numpy as np
import pytest

import oracle_lib as O
import pipeline_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_pipeline_stream as P  # noqa: E402
from test_stream_pipeline import ALLOC_STREAM, SLOTS, model_counters  # noqa: E402

pytestmark = pytest.mark.gpu
KNOBS = ("VP8GPU_TOK_SLOTS", "VP8GPU_TOK_CHUNK", "VP8GPU_TOK_ARENA", "VP8GPU_TOK_INFLIGHT", "VP8GPU_DISPATCHERS",
         "VP8GPU_TRACE")
_cache = {}


def _stream(name):
    if name not in _cache:
        data = P.make(name)
        _cache[name] = (data, O.decode_ivf_display(data))
    return _cache[name]


@pytest.fixture(autouse=True)
def no_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def _decode(ctx, data, want, copies, threads, want_output=True):
    """decode_ivf of `copies` copies of a stream; every copy's output equals `want`; every raster comes back"""
    from alfalfa_b200 import decode_ivf
    base = ctx.L.vp8gpu_frames_in_use(ctx.h)
    w, h, frames = O.read_ivf(data)
    out, n_dec, _ = decode_ivf(ctx, P.F.ivf(w, h, frames * copies), threads=threads, want_output=want_output)
    assert n_dec == len(frames) * copies
    assert ctx.L.vp8gpu_frames_in_use(ctx.h) == base
    if want_output:
        assert len(out) == len(want) * copies
        for c in range(copies):
            got = out[c * len(want):(c + 1) * len(want)]
            if got != want:
                n = ctx.display_bytes
                bad = next(i for i in range(len(want) // n) if got[i * n:(i + 1) * n] != want[i * n:(i + 1) * n])
                pytest.fail("copy %d (GOPs from %d on): shown frame %d differs from the oracle's" % (c, c, bad))


DENSITY = [n for n in P.names() if n.startswith("density")]


@pytest.mark.parametrize("name", DENSITY)
def test_parse_frame_device_equals_parse_frame(name):
    from alfalfa_b200 import Context, Decoder
    data, _ = _stream(name)
    w, h, frames = O.read_ivf(data)
    ctx = Context(w, h, max_frames=16)
    host, dev = Decoder(ctx), Decoder(ctx)
    for i, f in enumerate(frames):
        a, b = host.parse_frame(f), dev.parse_frame_device(f)
        assert bytes(a.desc) == bytes(b.desc), "frame %d" % i
        for x, y in zip(a.arrays(), b.arrays()):
            assert x.tobytes() == y.tobytes(), "frame %d" % i
    del host, dev
    ctx.close()


@pytest.mark.parametrize("name", DENSITY)
def test_decoder_with_device_tokens_matches_oracle(name):
    from alfalfa_b200 import Context, Decoder
    data, _ = _stream(name)
    w, h, frames = O.read_ivf(data)
    ctx = Context(w, h, max_frames=16)
    dec = Decoder(ctx)
    dec.set_device_tokens(True)
    od = O.OracleDecoder(w, h)
    for i, f in enumerate(frames):
        want = od.decode(f)
        shown, raster = dec.get_frame_output(f)
        assert shown == want["shown"]
        for p, (g, w_) in enumerate(zip(raster.planes(), want["planes"])):
            assert np.array_equal(g, w_), "frame %d plane %d" % (i, p)
        raster.release()
    for k, r in enumerate(dec.get_references()):
        for g, w_ in zip(r.planes(), O.raster_planes(od.L.vp8o_decoder_ref(od.d, k))):
            assert np.array_equal(g, w_), "reference %d" % k
        r.release()
    del dec
    ctx.close()


@pytest.mark.parametrize("name", DENSITY + ["densemix_176x144"])
def test_decode_ivf_with_device_tokens_matches_oracle(name):
    """8 copies on 4 workers; densemix: half-coded density frames whose arena pieces lie between those of frames
    several times their size"""
    from alfalfa_b200 import Context
    data, want = _stream(name)
    w, h, _ = O.read_ivf(data)
    copies = 2 if w >= 1920 else 8
    ctx = Context(w, h, max_frames=4 * (96 + 6) + 64)
    ctx.set_device_tokens(True)
    _decode(ctx, data, want, copies, threads=4)
    ctx.close()


def _arena_lines(text):
    return [tuple(int(x) for x in m) for m in
            re.findall(r"decode_ivf arena: worker (\d+) takes (\d+) wraps (\d+) waits (\d+) cap (\d+) slots (\d+) chunk (\d+)", text)]


def _alloc_cases():
    out = []
    for s in SLOTS:
        for c in sorted({1, None, s // 2}, key=lambda c: -1 if c is None else c):
            for a in (None, 0):
                out.append(pytest.param(s, c, a, id="slots%d-chunk%s-%s" % (s, "default" if c is None else c,
                                                                             "default_arena" if a is None else "floor")))
    return out


@pytest.mark.parametrize("slots,chunk,arena", _alloc_cases())
def test_allocator_counters_equal_the_model(slots, chunk, arena, monkeypatch, capfd):
    """one worker: where every frame's token piece goes does not depend on timing, so the takes, wraps and waits it
    counts are the model's exactly, and the output is the oracle's"""
    from alfalfa_b200 import Context
    data, want = _stream(ALLOC_STREAM)
    w, h, _ = O.read_ivf(data)
    monkeypatch.setenv("VP8GPU_TRACE", "1")
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", str(slots))
    if chunk is not None:
        monkeypatch.setenv("VP8GPU_TOK_CHUNK", str(chunk))
    if arena is not None:
        monkeypatch.setenv("VP8GPU_TOK_ARENA", str(arena))
    ctx = Context(w, h, max_frames=slots + 6 + 64)
    ctx.set_device_tokens(True)
    capfd.readouterr()
    _decode(ctx, data, want, 1, threads=1)
    ctx.close()
    lines = _arena_lines(capfd.readouterr().err)
    (s, c, cap, _), n = model_counters(ALLOC_STREAM, slots, chunk=chunk, arena=arena)
    assert lines == [(0, n["takes"], n["wraps"], n["waits"], cap, s, c)]


def test_bench_shape_with_the_arena_at_its_floor(monkeypatch, capfd):
    """64 workers, 96 slots, chunks of 32, 4 dispatchers, the arena at its floor (room for 50 of the largest frames),
    4 copies per worker of a GOP of 56 near-largest 640 x 368 frames: `value` (no output) and then `e2e` on the same
    context, as bench.py runs them, so that the second call reuses the first one's kits.  Whichever GOPs a worker
    got, its counters are the allocator model's for that many copies."""
    from alfalfa_b200 import Context
    data, want = _stream(P.DENSEGOP)
    w, h, frames = O.read_ivf(data)
    for k, v in (("VP8GPU_TRACE", "1"), ("VP8GPU_TOK_SLOTS", "96"), ("VP8GPU_TOK_CHUNK", "32"), ("VP8GPU_TOK_ARENA", "0"),
                 ("VP8GPU_DISPATCHERS", "4")):
        monkeypatch.setenv(k, v)
    threads, copies = 64, 4 * 64
    ctx = Context(w, h, max_frames=threads * (96 + 6) + 64)
    ctx.set_device_tokens(True)
    capfd.readouterr()
    _decode(ctx, data, want, copies, threads, want_output=False)
    _decode(ctx, data, want, copies, threads)
    ctx.close()
    lines = _arena_lines(capfd.readouterr().err)
    assert len(lines) == 2 * threads
    for line in lines:
        k, rest = divmod(line[1], len(frames))
        (s, c, cap, _), n = model_counters(P.DENSEGOP, 96, chunk=32, arena=0, copies=k)
        assert rest == 0 and line[1:] == (n["takes"], n["wraps"], n["waits"], cap, s, c), line
    with capfd.disabled():
        print("\nbench shape, arena at the floor: %d takes, %d wraps, %d waits over two calls of %d workers"
              % (sum(x[1] for x in lines), sum(x[2] for x in lines), sum(x[3] for x in lines), threads))
    assert sum(x[2] for x in lines) > 0 and sum(x[3] for x in lines) > 0


def test_1080p_bench_clip_at_96_slots(monkeypatch, capfd):
    """8 workers x 96 slots on 4 copies of a 1080p bench clip (8 GOPs), each copy against the reference decoder's
    digest of the clip (tests/golden/bench_clips.json), with max_frames sized as bench.py sizes it"""
    import json
    from alfalfa_b200 import Context, decode_ivf
    name = "synth1080p_medium_q90.ivf"
    digest = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_clips.json")))[name]["sha1_of_reference_decode"]
    data = open(os.path.join(ROOT, "bench_data", name), "rb").read()
    w, h, frames = O.read_ivf(data)
    monkeypatch.setenv("VP8GPU_TRACE", "1")
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", "96")
    threads, copies = 8, 4
    ctx = Context(w, h, max_frames=threads * (96 + 6) + 64)
    ctx.set_device_tokens(True)
    base = ctx.L.vp8gpu_frames_in_use(ctx.h)
    capfd.readouterr()
    out, n_dec, _ = decode_ivf(ctx, P.F.ivf(w, h, frames * copies), threads=threads)
    assert n_dec == len(frames) * copies and ctx.L.vp8gpu_frames_in_use(ctx.h) == base
    ctx.close()
    size = len(out) // copies
    for c in range(copies):
        assert hashlib.sha1(out[c * size:(c + 1) * size]).hexdigest() == digest, "copy %d" % c
    lines = _arena_lines(capfd.readouterr().err)
    assert len(lines) == threads and all(line[5] == 96 for line in lines)
    with capfd.disabled():
        print("\n1080p bench clip, 8 workers x 96 slots: %d takes, %d wraps, %d waits"
              % (sum(x[1] for x in lines), sum(x[2] for x in lines), sum(x[3] for x in lines)))


@pytest.mark.parametrize("inflight", [0, 1, 3])
@pytest.mark.parametrize("dispatchers", [1, 2, 3, 4])
@pytest.mark.parametrize("name", [n for n in P.names() if n.startswith("sizemix")])
def test_dispatcher_and_permit_knobs(name, dispatchers, inflight, monkeypatch):
    from alfalfa_b200 import Context
    data, want = _stream(name)
    w, h, _ = O.read_ivf(data)
    monkeypatch.setenv("VP8GPU_DISPATCHERS", str(dispatchers))
    monkeypatch.setenv("VP8GPU_TOK_INFLIGHT", str(inflight))
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", "16")
    threads = max(2, dispatchers)
    ctx = Context(w, h, max_frames=threads * (16 + 6) + 64)
    ctx.set_device_tokens(True)
    _decode(ctx, data, want, 1, threads)
    ctx.close()


def test_worker_kits_reused_across_calls_of_different_sizes(monkeypatch):
    """one context: a small stream on 4 workers, a stream with larger frames on 4 (new kits), the small one on 8 (4 of
    them on the larger kits, whose arenas are larger than its plan), and once more with fewer slots and the arena at
    its floor"""
    from alfalfa_b200 import Context
    small, large = "sizemix_176x144", "densemix_176x144"
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", "16")
    ctx = Context(176, 144, max_frames=8 * (16 + 6) + 64)
    ctx.set_device_tokens(True)
    for name, threads in ((small, 4), (large, 4), (small, 8)):
        _decode(ctx, _stream(name)[0], _stream(name)[1], 2, threads)
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", "7")
    monkeypatch.setenv("VP8GPU_TOK_ARENA", "0")
    _decode(ctx, _stream(small)[0], _stream(small)[1], 2, threads=8)
    ctx.close()
