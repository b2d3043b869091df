"""Re-encoding many chunks at once (vp8gpu_encoder_update_residues_batch, alfalfa_b200.reencode_chunks): every chunk of a
batch must come out exactly as its Encoder produces it alone through the single calls (which tests/test_gpu_reencode.py
and tests/test_gpu_reencode_edges.py pin to the reference's Encoder::reencode), and every Encoder must end in the same
state.  The bench's 1080p chunk is also held against the reference's stored answer.

Also run under the SIMT emulator in both thread orders (tests/test_reencode_batch_emulated.py), without the 1080p, the
16-chunk 640x360 and the 1024-column cases."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
import reference_answers as R
from test_gpu_encoder import ROOT, synth
from test_gpu_reencode import _decoded_targets, _full_name, _golden, reference_reencode

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_edge_stream as E  # noqa: E402
from test_gpu_reencode_edges import checker, noise  # noqa: E402

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("VP8GPU_SIMT_EMULATED"))


def _ctx(w, h, chunks):
    from alfalfa_b200 import Context
    return Context(w, h, max_frames=12 * chunks + 32)


def _encode(ctx, frames, qi):
    """this library's encoder at a fixed quantiser, from a fresh Encoder: a key frame, then inter frames"""
    from alfalfa_b200 import Encoder
    enc = Encoder(ctx)
    return [bytes(enc.encode_with_quantizer(*f, qi)) for f in frames]


def _state(ctx, chunks, n):
    """Decoder::serialize after the first n frames of a stream"""
    from alfalfa_b200 import Decoder
    d = Decoder(ctx)
    for c in chunks[:n]:
        _, r = d.get_frame_output(c)
        r.release()
    return d.serialize()


def _parsed(ctx, chunks):
    """the chunk's frames parsed with keep_labels by its own decoder (xc-enc.cc:254, 284-300)"""
    from alfalfa_b200 import Decoder
    d = Decoder(ctx)
    out = []
    for c in chunks:
        pf = d.parse_frame(c, keep_labels=True)
        d.decode_frame(pf)
        out.append(pf)
    return out


def synth_case(ctx, seed, n, qi_prev, qi_chunk):
    """(state, prediction chunk, targets): the state n frames of one synthetic clip leave behind, a chunk of n frames of
    another clip coded on its own, its source pictures as targets"""
    w, h = ctx.width, ctx.height
    prev = _encode(ctx, [synth(w, h, t, seed=seed) for t in range(n)], qi_prev)
    frames = [synth(w, h, t + 3, seed=seed + 50) for t in range(n)]
    return _state(ctx, prev, n), _encode(ctx, frames, qi_chunk), frames


def _encoder(ctx, state):
    from alfalfa_b200 import Decoder, Encoder
    return Encoder.from_decoder(ctx, Decoder.deserialize(ctx, state))


def alone(ctx, cases, kfw, extra):
    """every chunk through Encoder.reencode on an Encoder of its own: (frames per chunk, the Encoders)"""
    encs = [_encoder(ctx, s) for s, _, _ in cases]
    return [e.reencode(t, _parsed(ctx, p), kfw, extra) for e, (_, p, t) in zip(encs, cases)], encs


def batched(ctx, cases, kfw, extra):
    from alfalfa_b200 import reencode_chunks
    encs = [_encoder(ctx, s) for s, _, _ in cases]
    return reencode_chunks(encs, [t for _, _, t in cases], [_parsed(ctx, p) for _, p, _ in cases], kfw, extra), encs


def assert_same(ctx, cases, kfw, extra, what=""):
    want, enc_a = alone(ctx, cases, kfw, extra)
    got, enc_b = batched(ctx, cases, kfw, extra)
    for c, (a, b) in enumerate(zip(want, got)):
        assert len(a) == len(b), "%s chunk %d" % (what, c)
        for i, (x, y) in enumerate(zip(a, b)):
            assert x == y, "%s chunk %d frame %d: %d vs %d bytes, or different bytes" % (what, c, i, len(x), len(y))
    for c, (a, b) in enumerate(zip(enc_a, enc_b)):
        assert a.export_decoder() == b.export_decoder(), "%s chunk %d: Encoder state" % (what, c)
    return got


def frames_in_use(ctx):
    return ctx.L.vp8gpu_frames_in_use(ctx.h)


BATCHES = [((176, 144), 1), ((176, 144), 2), ((176, 144), 5), ((176, 144), 16), ((640, 360), 2), ((640, 360), 5)]
if not EMULATED:
    BATCHES.append(((640, 360), 16))


@pytest.mark.parametrize("size,n", BATCHES)
@pytest.mark.parametrize("kfw,extra", [(1.0, True), (0.75, False), (0.75, True)])
def test_batch_equals_alone(size, n, kfw, extra):
    """n chunks of distinct clips, states and quantisers: reencode_chunks == a loop of Encoder.reencode"""
    ctx = _ctx(*size, n)
    cases = [synth_case(ctx, 11 + 7 * c, 4, 30 + 9 * (c % 5), 44 + 5 * (c % 7)) for c in range(n)]
    assert_same(ctx, cases, kfw, extra, "%dx%d" % size)
    ctx.close()


def test_encoder_state_after_every_position():
    """Encoder.update_residues_batch position by position: after each, every Encoder's export_decoder() equals that of
    the same chunk's Encoder advanced by single update_residues calls; the per-job bytes are the single call's"""
    from alfalfa_b200 import Encoder
    ctx = _ctx(176, 144, 3)
    cases = [synth_case(ctx, 5 + c, 5, 36 + 4 * c, 50 - 3 * c) for c in range(3)]
    enc_a = [_encoder(ctx, s) for s, _, _ in cases]
    enc_b = [_encoder(ctx, s) for s, _, _ in cases]
    preds = [_parsed(ctx, p) for _, p, _ in cases]
    for i in range(1, 5):
        last = i == 4
        want = [e.update_residues(*t[i], p[i], -1, last) for e, (_, _, t), p in zip(enc_a, cases, preds)]
        got = Encoder.update_residues_batch([(e, *t[i], p[i], -1, last) for e, (_, _, t), p in zip(enc_b, cases, preds)])
        assert got == want, i
        for a, b in zip(enc_a, enc_b):
            assert a.export_decoder() == b.export_decoder(), i
            assert a.minihash() == b.minihash(), i
        tl = enc_b[0].timeline()
        assert tl["total"] > 0 and tl["total"] >= tl["writer"] and tl["estimates_launch"] == 0, tl
    ctx.close()


def test_bench_shape():
    """8 x 1080p bench chunks (tools/reencode_bench.py: 12 frames, extra-frame chunk) against the states of different
    clips after different numbers of frames; the bench's own case also equals the reference's stored answer"""
    if EMULATED:
        pytest.skip("1080p: on the GPU only")
    import reencode_bench as B
    bd = os.path.join(ROOT, "bench_data")
    prevs = [(B.PREV, B.PREV_FRAMES), (os.path.join(bd, "synth1080p_medium_q70_s33.ivf"), 5),
             (os.path.join(bd, "synth1080p_hard_q60_s7.ivf"), 3), (os.path.join(bd, "synth1080p_easy_q60_s5.ivf"), 9)]
    chunks = [B.CHUNK, os.path.join(bd, "synth1080p_medium_q110_s21.ivf")]
    ctx = _ctx(1920, 1080, 8)
    cases = []
    for k in range(8):
        prev, nprev = prevs[k % 4]
        state, _, _, targets = B.bench_inputs(ctx, prev, chunks[k // 4])
        if nprev != B.PREV_FRAMES:
            state = _state(ctx, O.read_ivf(open(prev, "rb").read())[2], nprev)
        chunk = O.read_ivf(open(chunks[k // 4], "rb").read())[2][:12]
        cases.append((state, chunk, targets))
    got = assert_same(ctx, cases, 0.75, True, "1080p")
    assert R.digests(got[0]) == reference_reencode(1920, 1080, cases[0][2], cases[0][1], cases[0][0], 0.75, True)
    ctx.close()


def _vector_case(ctx, prev, this, nframes, nprev):
    w, h, prev_chunks = _golden(_full_name(prev))
    _, _, chunks = _golden(_full_name(this))
    chunks = chunks[:nframes]
    return _state(ctx, prev_chunks, nprev), chunks, _decoded_targets(w, h, chunks)


@pytest.mark.parametrize("prev,this", [("0ccf971d", "353ee97f"), ("04b68b0a642d8285303d2b8884fc374e09d28ae9", "07b5eb1e9741d90027c46166eaaff566c6bf934f")])
def test_libvpx_prediction_streams_in_one_batch(prev, this):
    """libvpx vectors as prediction streams (SPLITMV, golden / altref with sign bias, intra macroblocks in inter frames,
    loop-filter deltas), one chunk per receiver state and of different lengths, so that last_frame is set on some jobs
    of a batch only"""
    w, h, _ = _golden(_full_name(this))
    ctx = _ctx(w, h, 3)
    n = 8 if EMULATED else 13
    cases = [_vector_case(ctx, prev, this, n - 2 * k, 1 + 3 * k) for k in range(3)]
    assert_same(ctx, cases, 0.75, True)
    ctx.close()


def test_mixed_batches():
    """in one batch: a still clip (no intra macroblock in its inter frames), a clip with a cut at every frame (mostly
    intra), a chunk with a key frame in the middle (kept by write_frame), a shorter chunk"""
    w, h = 176, 144
    ctx = _ctx(w, h, 4)
    s = [synth_case(ctx, 90 + c, 3, 40, 40)[0] for c in range(4)]
    still = [synth(w, h, 0, seed=3)] * 6
    cuts = [synth(w, h, t, seed=200 + 17 * t) for t in range(6)]
    midkey = [synth(w, h, t, seed=4) for t in range(6)]
    cases = [(s[0], _encode(ctx, still, 50), still), (s[1], _encode(ctx, cuts, 50), cuts),
             (s[2], _encode(ctx, midkey[:3], 46) + _encode(ctx, midkey[3:], 46), midkey), (s[3], _encode(ctx, cuts[:3], 60), cuts[:3])]
    for kfw, extra in ((0.75, True), (0.5, False)):
        assert_same(ctx, cases, kfw, extra)
    ctx.close()


def test_shared_rasters_and_interleaved_calls():
    """clones of one Encoder and Encoders made from one Decoder share their reference rasters inside a batch; batch and
    single calls alternate on the same Encoders within a chunk"""
    from alfalfa_b200 import Decoder, Encoder
    ctx = _ctx(176, 144, 6)
    state, pred, targets = synth_case(ctx, 21, 6, 40, 52)
    preds = _parsed(ctx, pred)
    d = Decoder.deserialize(ctx, state)
    base = Encoder.from_decoder(ctx, d)
    group = [base, base.copy(), Encoder.from_decoder(ctx, d), base.copy()]
    solo = [_encoder(ctx, state) for _ in group]
    qis = [-1, 30, 50, 70]
    start = frames_in_use(ctx)
    for i in range(1, 6):
        last = i == 5
        want = [e.update_residues(*targets[i], preds[i], q, last) for e, q in zip(solo, qis)]
        if i % 2:
            got = Encoder.update_residues_batch([(e, *targets[i], preds[i], q, last) for e, q in zip(group, qis)])
        else:
            got = [e.update_residues(*targets[i], preds[i], q, last) for e, q in zip(group, qis)]
        assert got == want, i
    for a, b in zip(solo, group):
        assert a.export_decoder() == b.export_decoder()
    # the last frame refreshed every reference: each Encoder holds one raster of its own (the solo Encoders' states
    # went with their old references; the shared one is still the Decoder's)
    assert frames_in_use(ctx) == start + len(group)
    ctx.close()


def _segment_map_frame(ctx, w, h):
    """an inter frame of a golden vector of this size that update_residues refuses (it updates the segment map)"""
    from alfalfa_b200 import Decoder, Encoder, capi
    from conftest import golden_vectors
    for name in golden_vectors():
        vw, vh, chunks = _golden(name)
        if (vw, vh) != (w, h):
            continue
        d = Decoder(ctx)
        pfs = []
        for c in chunks[:12]:
            pf = d.parse_frame(c, keep_labels=True)
            d.decode_frame(pf)
            pfs.append(pf)
        enc = Encoder.from_decoder(ctx, Decoder(ctx))
        for pf in pfs[1:]:
            if pf.desc.key_frame:
                continue
            try:
                enc.copy().update_residues(*synth(w, h, 0), pf)
            except capi.Unsupported:
                return pf
    return None


def test_refusals_are_per_job():
    """a segment-map update (UNSUPPORTED), a key-frame prediction (LOGIC) and a too small output buffer (NOMEM, size
    set) fail their own job and leave its Encoder as it was; the other jobs are the single calls' and advance.  The same
    Encoder twice or one of another context fail the whole call (LOGIC) and no Encoder moves.  No raster is leaked."""
    from alfalfa_b200 import Encoder, capi
    w, h = 176, 144
    ctx = _ctx(w, h, 5)
    state, pred, targets = synth_case(ctx, 31, 3, 40, 50)
    preds = _parsed(ctx, pred)
    seg = _segment_map_frame(ctx, w, h)
    assert seg is not None, "no golden vector of %dx%d has an inter frame that updates the segment map" % (w, h)
    encs = [_encoder(ctx, state) for _ in range(5)]
    solo = [_encoder(ctx, state) for _ in range(2)]
    start = frames_in_use(ctx)
    hashes = [e.minihash() for e in encs]

    def jobs_of(specs):
        arr = (capi.ReencodeJob * len(specs))()
        keep = []
        for j, (enc, pf, cap) in zip(arr, specs):
            y, u, v = enc._planes(*targets[1])
            keep.append((y, u, v))
            j.encoder, j.y, j.u, j.v, j.y_stride, j.uv_stride = enc.h.value, y.ctypes.data, u.ctypes.data, v.ctypes.data, y.shape[1], u.shape[1]
            j.prediction_frame, j.y_ac_qi, j.last_frame, j.out, j.cap = pf.h.value, -1, 0, enc._out.ctypes.data, cap
        return arr, keep

    specs = [(encs[0], preds[1], encs[0]._out.size), (encs[1], preds[0], encs[1]._out.size), (encs[2], preds[1], 10),
             (encs[3], preds[1], encs[3]._out.size)]
    specs.append((encs[4], seg, encs[4]._out.size))
    arr, keep = jobs_of(specs)
    rc = ctx.L.vp8gpu_encoder_update_residues_batch(arr, len(specs))
    want = [e.update_residues(*targets[1], preds[1]) for e in solo]
    assert rc == capi.ERR_LOGIC  # the first failed job's, and the context's last error names it
    assert ctx.L.vp8gpu_last_error(ctx.h).decode().startswith("update_residues_batch: job 1 of 5 failed: update_residues: the prediction "
                                                              "frame is a key frame")
    assert [j.status for j in arr] == [capi.OK, capi.ERR_LOGIC, capi.ERR_NOMEM, capi.OK, capi.ERR_UNSUPPORTED]
    assert arr[2].size == len(want[0])
    assert encs[0]._out[:arr[0].size].tobytes() == want[0] and encs[3]._out[:arr[3].size].tobytes() == want[0]
    for k in (1, 2, 4):
        assert encs[k].minihash() == hashes[k], k
    assert encs[0].export_decoder() == solo[0].export_decoder() and encs[3].export_decoder() == solo[0].export_decoder()
    assert frames_in_use(ctx) == start + 4  # four Encoders advanced: a new LAST each, the old one kept as GOLDEN and ALTREF

    hashes = [e.minihash() for e in encs]
    other = _ctx(w, h, 1)
    foreign = _encoder(other, state)
    for bad in ([(encs[1], preds[1], encs[1]._out.size), (encs[1], preds[1], encs[1]._out.size)],
                [(encs[1], preds[1], encs[1]._out.size), (foreign, preds[1], foreign._out.size)]):
        arr, keep = jobs_of(bad)
        assert ctx.L.vp8gpu_encoder_update_residues_batch(arr, len(bad)) == capi.ERR_LOGIC
        assert all(j.status == capi.ERR_LOGIC for j in arr)
        assert [e.minihash() for e in encs] == hashes
    assert ctx.L.vp8gpu_encoder_update_residues_batch(None, -1) == capi.ERR_LOGIC
    with pytest.raises(capi.LogicError):
        Encoder.update_residues_batch([(encs[1], *targets[1], preds[1]), (encs[1], *targets[1], preds[1])])
    assert frames_in_use(ctx) == start + 4
    del foreign
    other.close()
    ctx.close()


def _speculate_child():
    """(child process) one small batch; prints the digests of what it emitted"""
    ctx = _ctx(176, 144, 3)
    cases = [synth_case(ctx, 61 + c, 4, 38, 52) for c in range(3)]
    got, _ = batched(ctx, cases, 0.75, False)
    print(repr([R.digests(g) for g in got]))


def test_batch_the_same_with_the_shortcuts_off():
    """VP8GPU_ENC_SPECULATE=0: the emitted frames are decoded through the full parse instead of the token lists they were
    written from -- the same bytes"""
    code = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_gpu_reencode_batch as T; T._speculate_child()" % (
        ROOT, os.path.join(ROOT, "tests"))
    outs = []
    for spec in ("1", "0"):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, VP8GPU_ENC_SPECULATE=spec), cwd=os.path.join(ROOT, "tests"))
        assert r.returncode == 0, (r.stdout + r.stderr)[-1500:]
        outs.append(r.stdout.strip().splitlines()[-1])
    assert outs[0] == outs[1]


EDGE_NAMES = [n for n in E.reencode_names() if not (EMULATED and ("16383" in n or "1024x" in n))]


@pytest.mark.parametrize("name", EDGE_NAMES)
def test_edge_shapes(name):
    """tools/make_edge_stream.py's re-encodable streams (degenerate shapes, the saturate family): 3 chunks of the shape
    from different receiver states towards different targets (own pictures, checkerboard, noise), extra-frame and whole"""
    w, h, chunks = O.read_ivf(E.make_reencodable(name))
    _, _, prev = O.read_ivf(E.make_reencodable(name, previous=True))
    ctx = _ctx(w, h, 3)
    targets = [_decoded_targets(w, h, chunks), [checker(w, h, i) for i in range(len(chunks))], [noise(w, h, i) for i in range(len(chunks))]]
    cases = [(_state(ctx, prev, len(prev) - k), chunks, t) for k, t in enumerate(targets)]
    for kfw, extra in ((0.75, True), (0.5, False)):
        assert_same(ctx, cases, kfw, extra, name)
    ctx.close()


@pytest.mark.parametrize("extra_frame_chunk", [0, 1])
def test_cxx_batch_equals_python_single_calls(tmp_path, extra_frame_chunk):
    """tests/cxx/reencode_batch.cc: three chunks of different lengths through alfalfa_gpu::update_residues_batch on the
    C++ mirror (xc-enc --reencode, position by position); each chunk's IVF equals Encoder.reencode of that chunk alone,
    and the same Encoder twice in one batch throws"""
    lib = os.environ.get("VP8GPU_LIB", os.path.join(ROOT, "alfalfa_b200", "libvp8gpu.so"))
    exe = str(tmp_path / "reencode_batch")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-pthread", os.path.join(ROOT, "tests", "cxx", "reencode_batch.cc"),
                           "-o", exe, "-L" + os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Wl,-rpath," + os.path.dirname(lib)])
    w, h = 176, 144
    ctx = _ctx(w, h, 3)
    cases = [synth_case(ctx, 71 + c, 3 + c, 34 + 6 * c, 48 + 4 * c) for c in range(3)]
    want, _ = alone(ctx, cases, 0.75, bool(extra_frame_chunk))
    ctx.close()
    args = []
    for c, (state, pred, targets) in enumerate(cases):
        raw, pivf, sbin = (str(tmp_path / ("%d.%s" % (c, x))) for x in ("yuv", "ivf", "bin"))
        with open(raw, "wb") as f:
            for planes in targets:
                for p in planes:
                    f.write(np.ascontiguousarray(p).tobytes())
        from alfalfa_b200 import write_ivf
        open(pivf, "wb").write(write_ivf(w, h, pred))
        open(sbin, "wb").write(state)
        args += [raw, pivf, sbin]
    prefix = str(tmp_path / "out")
    r = subprocess.run([exe, prefix, str(w), str(h), "0.75", str(extra_frame_chunk)] + args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.startswith("ok 3"), (r.stdout + r.stderr)[-800:]
    for c in range(3):
        _, _, got = O.read_ivf(open("%s.%d.ivf" % (prefix, c), "rb").read())
        assert got == want[c], c
