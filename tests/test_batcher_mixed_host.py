"""Host logic of the batcher's mixed key (OC_BATCHER_MIXED, oramacore_b200/csrc/batcher.h) with its own fake executor,
which honours q_params: tests/batcher_mixed_test.cpp is compiled with g++ (no CUDA), -O2 and under ThreadSanitizer, and
16 threads submit requests with random modes, limits, offsets, similarities, thresholds, vector limits and OMC arrays.
mixed: every caller gets its own answer at its own limit, requests with different scalars and with OMC shared merged
calls, a merged call's row stride is its largest limit, its requests share the two route flags (threshold, vector depth
above the tensor-core limit) and the OMC arrays, and requests the library would refuse for their scalars ran alone.
default: the same traffic never merges requests with different scalars or with OMC."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=[["-O2"], ["-O1", "-g", "-fsanitize=thread"]], ids=["O2", "tsan"])
def mixed_exe(request, tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    flags = request.param
    exe = str(tmp_path_factory.mktemp("batcher_mixed") / "batcher_mixed_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_mixed_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize("scenario", ["mixed", "default"])
def test_batcher_mixed_key_under_concurrency(mixed_exe, scenario):
    r = subprocess.run([mixed_exe, scenario], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
