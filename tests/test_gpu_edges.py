"""The decode kernels on the edge streams of tools/make_edge_stream.py (degenerate frame shapes, prediction windows
on every side of every plane edge at every filter phase, extreme coefficients; their coverage is asserted in
tests/test_edge_streams.py): every frame, hidden ones included, and the three references after the last frame equal
the oracle's bit for bit, under each intra / loop-filter kernel pair (VP8GPU_WAVEFRONT) and with the DCT partitions
decoded on the host and on the device.  Also many short streams in one vp8gpu_decode_ivf call, and the lock-step
token kernel on the widest frame the format allows."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_edge_stream as E  # noqa: E402

pytestmark = pytest.mark.gpu
_cache = {}


def _stream(name):
    if name not in _cache:
        _cache[name] = E.make(name)
    return _cache[name]


# unset = the default (k_intra_ll + k_loopfilter_band); legacy = k_intra with progress counters + k_loopfilter;
# intra-ll = k_intra_ll + k_loopfilter; ll = k_intra_ll + k_loopfilter_ll; lf-ll = k_intra + k_loopfilter_ll
# (engine.cu reads it at every context creation)
@pytest.fixture(params=[None, "legacy", "intra-ll", "ll", "lf-ll"], ids=["default", "legacy", "intra-ll", "ll", "lf-ll"])
def wavefront(request, monkeypatch):
    if request.param is None:
        monkeypatch.delenv("VP8GPU_WAVEFRONT", raising=False)
    else:
        monkeypatch.setenv("VP8GPU_WAVEFRONT", request.param)
    return request.param


@pytest.mark.parametrize("device_tokens", [False, True], ids=["host_tokens", "device_tokens"])
@pytest.mark.parametrize("name", E.names())
def test_every_frame_and_reference_matches_oracle(name, device_tokens, wavefront):
    from alfalfa_b200 import Context, Decoder
    w, h, frames = O.read_ivf(_stream(name))
    ctx = Context(w, h, max_frames=16)
    dec = Decoder(ctx)
    dec.set_device_tokens(device_tokens)
    od = O.OracleDecoder(w, h)
    for i, f in enumerate(frames):
        want = od.decode(f)
        shown, raster = dec.get_frame_output(f)
        assert shown == want["shown"]
        for p, (g, w_) in enumerate(zip(raster.planes(), want["planes"])):
            assert np.array_equal(g, w_), "frame %d plane %d: %d pixels differ" % (i, p, int((g != w_).sum()))
        raster.release()
    for k, r in enumerate(dec.get_references()):
        for g, w_ in zip(r.planes(), O.raster_planes(od.L.vp8o_decoder_ref(od.d, k))):
            assert np.array_equal(g, w_), "reference %d" % k
        r.release()
    del dec
    ctx.close()


@pytest.mark.parametrize("device_tokens", [False, True], ids=["host_tokens", "device_tokens"])
@pytest.mark.parametrize("name", ["shapes_16x512", "shapes_1x1", "shapes_16x16"])
def test_many_copies_in_one_stream_decode(name, device_tokens):
    """64 copies of a short stream in one vp8gpu_decode_ivf call: 64 GOPs of one-column or one-macroblock frames
    share the launches"""
    from alfalfa_b200 import Context, decode_ivf
    w, h, frames = O.read_ivf(_stream(name))
    data = E.F.ivf(w, h, frames * 64)
    want = O.decode_ivf_display(_stream(name)) * 64
    ctx = Context(w, h, max_frames=48)
    ctx.set_device_tokens(device_tokens)
    out, n_dec, n_shown = decode_ivf(ctx, data, threads=4)
    ctx.close()
    assert n_dec == len(frames) * 64 and out == want


def test_lockstep_token_kernel_on_the_widest_frame():
    """k_tokens_lockstep (VP8GPU_TOK_WARPS=32, read once per process, hence the subprocess) on 1024 macroblock
    columns: its dynamic shared memory holds one above-context row of kMaxCols = 1024"""
    code = r'''
import os, sys
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests")); sys.path.insert(0, os.path.join(%r, "tools"))
import oracle_lib as O, make_edge_stream as E
from alfalfa_b200 import Context, Decoder, decode_ivf
for name in ("shapes_16383x32", "shapes_16383x17"):
    data = E.make(name)
    w, h, frames = O.read_ivf(data)
    ctx = Context(w, h, max_frames=64)
    host, dev = Decoder(ctx), Decoder(ctx)
    for f in frames:
        a, b = host.parse_frame(f), dev.parse_frame_device(f)
        assert bytes(a.desc) == bytes(b.desc)
        for x, y in zip(a.arrays(), b.arrays()):
            assert x.tobytes() == y.tobytes()
    ctx.set_device_tokens(True)
    out, _, _ = decode_ivf(ctx, data, threads=2)
    assert out == O.decode_ivf_display(data), name
    del host, dev
    ctx.close()
print("ok")
''' % (ROOT, ROOT, ROOT)
    env = dict(os.environ, VP8GPU_TOK_WARPS="32")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout[-500:] + out.stderr[-2000:]
