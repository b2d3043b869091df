"""Whole-stream decode (vp8gpu_decode_ivf) hands a frame to the pixel kernels as soon as k_tokens has published that
frame's ready word, not when its whole k_tokens launch is done.  Every decode here must equal the host-token path
(set_device_tokens(False)) byte for byte:
  - the bench's 1080p clips at VP8GPU_TOK_CHUNK 1, 2, 7 and 32;
  - pipeline streams whose largest frame is the last of its GOP, or the first (tools/make_pipeline_stream.py), at
    several chunk sizes;
  - the token arena at its floor, with small rings (the allocator's limit cases);
  - a second call on the same context, whose pooled worker kits still hold the ready words of the first call's
    frames: an epoch left by an earlier frame must never read as ready.
The publishing code of both token kernels (k_tokens, one warp per frame, and k_tokens_lockstep, one lane per frame)
also runs under the SIMT emulator in both thread orders (the tests without the gpu mark)."""
import hashlib
import os
import sys

import pytest

import oracle_lib as O
from test_simt_emulation import SIMT_DIR, SIMT_LIB, run_gpu_tests_emulated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_pipeline_stream as P  # noqa: E402

KNOBS = ("VP8GPU_TOK_SLOTS", "VP8GPU_TOK_CHUNK", "VP8GPU_TOK_ARENA", "VP8GPU_TOK_INFLIGHT", "VP8GPU_DISPATCHERS",
         "VP8GPU_TRACE")
BENCH_CLIPS = ["synth1080p_medium_q90.ivf", "synth1080p_hard_q60_s7.ivf", "synth1080p_medium_q110_s21.ivf",
               "synth1080p_medium_q70_s33.ivf", "synth1080p_easy_q60_s5.ivf"]
_host = {}


@pytest.fixture(autouse=True)
def no_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def _digest(ctx, data, threads):
    from alfalfa_b200 import decode_ivf
    base = ctx.L.vp8gpu_frames_in_use(ctx.h)
    out, n_dec, n_shown = decode_ivf(ctx, data, threads=threads)
    assert ctx.L.vp8gpu_frames_in_use(ctx.h) == base
    return hashlib.sha1(out).hexdigest(), n_dec, n_shown


def _host_digest(key, data, threads):
    """the host-token path's output (its own context: the host workers need no token rings)"""
    if key not in _host:
        from alfalfa_b200 import Context
        w, h, _ = O.read_ivf(data)
        ctx = Context(w, h, max_frames=8 * threads + 64)
        ctx.set_device_tokens(False)
        _host[key] = _digest(ctx, data, threads)
        ctx.close()
    return _host[key]


def _device_ctx(data, threads):
    from alfalfa_b200 import Context
    w, h, _ = O.read_ivf(data)
    ctx = Context(w, h, max_frames=threads * (96 + 6) + 64)
    ctx.set_device_tokens(True)
    return ctx


def _check(name, data, threads, chunks, monkeypatch, calls=1):
    want = _host_digest(name, data, threads)
    ctx = _device_ctx(data, threads)
    for chunk in chunks:
        if chunk:
            monkeypatch.setenv("VP8GPU_TOK_CHUNK", str(chunk))
        for call in range(calls):
            assert _digest(ctx, data, threads) == want, "%s, chunk %s, call %d: output differs from the host-token path" % (
                name, chunk, call)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("clip", BENCH_CLIPS)
def test_bench_clip_at_every_chunk_size(clip, monkeypatch):
    data = open(os.path.join(ROOT, "bench_data", clip), "rb").read()
    _check(clip, data, 4, [1, 2, 7, 32], monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("name", P.order_names())
def test_largest_frame_last_or_first_in_its_gop(name, monkeypatch):
    _check(name, P.make(name), 2, [None, 1, 4, 30], monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [4, 7, 96])
def test_token_arena_at_its_floor(slots, monkeypatch):
    """densegop: one GOP of near-largest frames, more than an arena at its floor holds; sizemix: GOPs of 1 to 200
    frames of very different sizes; one worker each, so that its arena wraps and waits"""
    monkeypatch.setenv("VP8GPU_TOK_ARENA", "0")
    monkeypatch.setenv("VP8GPU_TOK_SLOTS", str(slots))
    for name in (P.DENSEGOP, "sizemix_176x144"):
        _check(name, P.make(name), 1, [None], monkeypatch)


@pytest.mark.gpu
def test_second_call_on_reused_kits_never_takes_a_stale_epoch(monkeypatch):
    """the same stream twice on one context, then the other order stream: the kits of the first call come back from
    the pool with every slot's ready words holding epochs of frames already decoded"""
    a, b = P.order_names()[:2]
    da, db = P.make(a), P.make(b)
    wa, wb = _host_digest(a, da, 2), _host_digest(b, db, 2)
    ctx = _device_ctx(da, 2)
    for name, data, want in ((a, da, wa), (a, da, wa), (b, db, wb), (a, da, wa)):
        assert _digest(ctx, data, 2) == want, "%s on reused kits: output differs from the host-token path" % name
    ctx.close()


# ---- the publishing code under the SIMT emulator, both token kernels, both thread orders ----------------------------
SIMT_SELECTION = ["tests/test_gpu_frame_ready.py", "-k", "largest_frame or reused_kits or (arena and 7)"]


@pytest.fixture(scope="module")
def simt_lib():
    import shutil
    import subprocess
    if shutil.which("g++") is None or os.uname().machine != "x86_64":
        pytest.skip("the emulator's fiber switch is x86-64 and needs g++")
    r = subprocess.run(["sh", os.path.join(SIMT_DIR, "build.sh")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and os.path.exists(SIMT_LIB), r.stderr[-2000:]
    return SIMT_LIB


@pytest.mark.parametrize("order", ["forward", "reverse"])
@pytest.mark.parametrize("warps", ["1", "32"])
def test_publish_and_acquire_emulated(simt_lib, warps, order):
    """VP8GPU_TOK_WARPS=1: k_tokens publishes from lane 0 of each frame's warp; 32: k_tokens_lockstep from each
    frame's lane, whenever that lane's frame ends.  The emulated pixel kernels check that a job's ready word holds its
    epoch when they acquire it."""
    env = {"VP8GPU_TOK_WARPS": warps}
    if order == "reverse":
        env["SIMT_ORDER"] = "reverse"
    run_gpu_tests_emulated(simt_lib, SIMT_SELECTION, env_extra=env)
