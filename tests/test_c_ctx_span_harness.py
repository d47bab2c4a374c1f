"""tests/c_ctx_span_harness.c: a plain-C caller that performs the per-tick loop over two ctxs (Fire -> TickTouched per ctx ->
ScheduleResidentCtxs -> Commit -> TransferToCtx -> TickTouched, go/frontier/frontier.go) through the entry points and flat
wrappers of go/frontier/shim.h.  Compiling it is a CPU test (the header and the shim are valid, warning-free C); running it needs
an H100."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bobrapet_b200", "lib")


def _build(tmp_path):
    exe = str(tmp_path / "c_ctx_span_harness")
    cmd = ["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "go", "frontier"),
           os.path.join(ROOT, "tests", "c_ctx_span_harness.c"), "-L" + LIB, "-lbobrafrontier", "-Wl,-rpath," + LIB, "-o", exe]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return exe


def test_ctx_span_harness_compiles_as_c(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True)       # without a GPU bf_create fails cleanly with a status
    assert out.returncode in (0, 1) and "Segmentation" not in out.stderr


@pytest.mark.gpu
def test_ctx_span_harness_runs_the_go_call_sequence(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "c_ctx_span_harness: ok" in out.stdout, (out.stdout, out.stderr)
