"""The loop-filter kernels against the oracle on designed records (tests/lf_maps.py): the reference raster is
uploaded, vp8gpu_decode_batch reconstructs and filters every job of a batch in one set of launches, and each output's
macroblock-aligned planes must equal vp8o_reconstruct + vp8o_loopfilter on the same records byte for byte.

The per-macroblock level maps decide which macroblocks each row filters, and with that which words k_loopfilter_band
takes from the ring of the row above, from the previous macroblock or from the frame; tests/test_lf_maps.py asserts
that the maps drive every one of those paths.  Each case runs under every loop-filter kernel (VP8GPU_WAVEFRONT, read
at context creation): the default k_loopfilter_band, k_loopfilter (legacy, intra-ll) and k_loopfilter_ll (ll, lf-ll).

Shapes: 1..9, 13 and 17 macroblock rows (every residue mod LF_BAND = 4, one to five bands) by 1..1024 columns (1024 =
32 bitmask words: every lane's above_word is used), plus the bench's shape, 64 jobs at 1920x1080 in one launch, where
the bands of different jobs interleave over all SMs and hand over through lf_progress.  What no test can force is
back-pressure on a row's `free` flag: whether a row catches up with the row below it depends on timing, not on data."""
import ctypes as C

import numpy as np
import pytest

import lf_maps as M

pytestmark = pytest.mark.gpu

# None = the default (k_intra_ll + k_loopfilter_band); legacy = k_intra + k_loopfilter; intra-ll = k_intra_ll +
# k_loopfilter; ll = k_intra_ll + k_loopfilter_ll; lf-ll = k_intra + k_loopfilter_ll
KERNELS = [None, "legacy", "intra-ll", "ll", "lf-ll"]
KERNEL_IDS = ["band", "legacy", "intra-ll", "ll", "lf-ll"]
_oracle = {}  # the oracle's answers of the last case (the kernel parameter varies fastest)


def _case(key, make):
    if key not in _oracle:
        _oracle.clear()
        cols, rows, jobs = make()
        ref = M.reference_picture(cols, rows, M.shape_seed(cols, rows))
        _oracle[key] = (cols, rows, jobs, ref, [M.oracle_decode(j, ref) for j in jobs])
    return _oracle[key]


def _first_difference(got, want, job):
    for p, (g, w) in enumerate(zip(got, want)):
        d = np.argwhere(g != w)
        if d.size:
            y, x = (int(v) for v in d[0])
            s = 16 if p == 0 else 8
            mr, mc = y // s, x // s
            return ("job %s: plane %s row %d col %d (macroblock row %d col %d, level %d): got %d want %d; %d bytes differ"
                    % (job.name, "YUV"[p], y, x, mr, mc, int(job.lf_map[mr, mc]), int(g[y, x]), int(w[y, x]),
                       int(sum((a != b).sum() for a, b in zip(got, want)))))
    return None


def _decode_and_compare(kernel, monkeypatch, width, height, case):
    if kernel is None:
        monkeypatch.delenv("VP8GPU_WAVEFRONT", raising=False)
    else:
        monkeypatch.setenv("VP8GPU_WAVEFRONT", kernel)
    from alfalfa_b200 import Context, capi
    cols, rows, jobs, ref, wants = case
    ctx = Context(width, height, max_frames=len(jobs) + 4)
    assert (ctx.mb_cols, ctx.mb_rows) == (cols, rows)
    ref_h = ctx.alloc_frame()
    ref_h.upload(*ref)
    keep, outs = [], []
    cj = (capi.Job * len(jobs))()
    for i, j in enumerate(jobs):
        desc = capi.FrameDesc.from_buffer_copy(bytes(j.desc))
        keep.append(desc)
        out = ctx.alloc_frame()
        outs.append(out)
        cj[i].desc = C.pointer(desc)
        cj[i].mbs = j.mbs.ctypes.data
        cj[i].tokens = j.tokens.ctypes.data if j.tokens.size else None
        cj[i].split = j.split.ctypes.data if j.split.size else None
        cj[i].refs[:] = [ref_h.id] * 3
        cj[i].out = out.id
    capi.check(ctx.L.vp8gpu_decode_batch(ctx.h, 0, cj, len(jobs)), ctx.h, "decode_batch")
    bad = []
    for j, out, want in zip(jobs, outs, wants):
        msg = _first_difference(out.planes(), want, j)
        if msg:
            bad.append(msg)
        out.release()
    ref_h.release()
    ctx.close()
    assert not bad, "%d of %d jobs differ from the oracle; %s" % (len(bad), len(jobs), "; ".join(bad[:4]))


@pytest.mark.parametrize("kernel", KERNELS, ids=KERNEL_IDS)
@pytest.mark.parametrize("shape", M.SHAPES, ids=["%dx%d" % s for s in M.SHAPES])
def test_designed_maps_match_the_oracle(shape, kernel, monkeypatch):
    """one launch: every map of lf_maps.maps() at this shape (each with its own levels, sharpness and key / inter
    flag) and a job whose frame level is 0 while its macroblock levels are not"""
    cols, rows = shape
    case = _case(shape, lambda: (cols, rows, M.batch(cols, rows, M.shape_seed(cols, rows))))
    _decode_and_compare(kernel, monkeypatch, min(16 * cols, 16383), 16 * rows, case)


@pytest.mark.parametrize("kernel", KERNELS, ids=KERNEL_IDS)
def test_bench_shape_64_jobs_at_1080p(kernel, monkeypatch):
    """64 jobs at 1920x1080 (120 x 68 macroblocks, 17 bands each) with Bernoulli maps from p = 0.1 to 0.9 in one
    launch"""
    case = _case("bench", lambda: (120, 68, M.bench_batch()))
    _decode_and_compare(kernel, monkeypatch, 1920, 1080, case)
