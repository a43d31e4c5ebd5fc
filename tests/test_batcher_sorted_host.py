"""Host logic of sorted and pinned requests in the micro-batching queue (oramacore_b200/csrc/batcher.h) with fake
executors: tests/batcher_sorted_test.cpp is compiled with g++ (no CUDA) and run with 12 submitting threads.  It fails
unless every merged batch with a sort or an item reaches the sorted executor with each request's sort, promote items
and device filter at its own position, batches with neither reach the plain executor, sort values and per-item pin
outputs go back to the right caller, and malformed requests are refused without joining a batch."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-O2"], ["-O1", "-g", "-fsanitize=thread"]])
def test_batcher_carries_sorts_and_pins(tmp_path, flags):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "batcher_sorted_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_sorted_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
