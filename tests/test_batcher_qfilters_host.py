"""Host logic of per-query device filters in the micro-batching queue (oramacore_b200/csrc/batcher.h) with a fake
executor: tests/batcher_qfilter_test.cpp is compiled with g++ (no CUDA) and run with 12 submitting threads.  It fails
unless every merged batch carries each request's device filter at its position in q_filters (NULL for an unfiltered
request, a NULL array when no request is filtered) and host-bitmap (filter_bits) requests run directly."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-O2"], ["-O1", "-g", "-fsanitize=thread"]])
def test_batcher_carries_per_query_filters(tmp_path, flags):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "batcher_qfilter_test")
    r = subprocess.run(["g++", "-std=c++17", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_qfilter_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
