"""tests/test_gpu_reencode_batch.py (many chunks re-encoded in one set of launches: per-job target, records, token pool and
counters, the ticket mapping of k_reenc_intra over several jobs, the rasters the jobs share) under the SIMT emulator, in
the default thread order and with SIMT_ORDER=reverse, and once under the alignment sanitizer.  The 1080p, 16-chunk
640x360 and 1024-column cases stay on the GPU (the test file skips them when emulated)."""
import os
import subprocess

import pytest

from test_simt_emulation import ROOT, SIMT_DIR, pytestmark, run_gpu_tests_emulated, simt_lib  # noqa: F401

ARGS = ["tests/test_gpu_reencode_batch.py"]


@pytest.mark.parametrize("order", ["default", "reverse"])
def test_batched_reencode_emulated(simt_lib, order):  # noqa: F811
    run_gpu_tests_emulated(simt_lib, ARGS, timeout=3600, env_extra={"SIMT_ORDER": order} if order == "reverse" else None)


def test_batched_reencode_alignment_sanitized():
    ubsan = subprocess.run(["g++", "-print-file-name=libubsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(ubsan) or not os.path.exists(ubsan):
        pytest.skip("libubsan not available")
    r = subprocess.run(["sh", os.path.join(SIMT_DIR, "build.sh")], env=dict(os.environ, SIMT_SANITIZE="alignment"), capture_output=True,
                       text=True, timeout=900)
    san = os.path.join(SIMT_DIR, "_build", "san", "libvp8gpu_simt.so")
    assert r.returncode == 0 and os.path.exists(san), r.stderr[-2000:]
    run_gpu_tests_emulated(san, ARGS, timeout=3600, env_extra={"LD_PRELOAD": ubsan})
