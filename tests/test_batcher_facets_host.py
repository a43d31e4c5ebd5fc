"""Host logic of faceted requests in the micro-batching queue (oramacore_b200/csrc/batcher.h) with fake executors:
tests/batcher_facets_test.cpp is compiled with g++ (no CUDA) and run with 12 submitting threads.  It fails unless
faceted requests batch only with faceted requests on the same facet store, each caller gets its own counts and group
rows back, a batch that runs out of device memory is split in halves until every request succeeds, and a request the
facet check refuses fails alone while its neighbours succeed."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-O2"], ["-O1", "-g", "-fsanitize=thread"]])
def test_batcher_carries_facets(tmp_path, flags):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "batcher_facets_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_facets_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
