"""Host logic of the micro-batching queue (oramacore_b200/csrc/batcher.h) with one fake executor: tests/batcher_test.cpp
is compiled with g++ (no CUDA), -O2 and under ThreadSanitizer, and each scenario runs with 12 or 16 submitting threads.
A scenario fails unless every caller receives exactly its own query's answer (hits, sort values, items, group rows,
facet counts), requests were coalesced, only requests of the same key shared a merged call and that call ran as the
right entry point, a merged grouped or faceted call that runs out of device memory was split, and refused requests
never reached the executor.  Scenarios: plain requests of every mode; per-query device filters; sorted and pinned
requests; grouped requests; faceted requests."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=[["-O2"], ["-O1", "-g", "-fsanitize=thread"]], ids=["O2", "tsan"])
def batcher_exe(request, tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    flags = request.param
    exe = str(tmp_path_factory.mktemp("batcher") / "batcher_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize("scenario", ["plain", "qfilters", "sorted", "groups", "facets"])
def test_batcher_merge_scatter_under_concurrency(batcher_exe, scenario):
    r = subprocess.run([batcher_exe, scenario], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
