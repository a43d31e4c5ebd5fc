"""Host logic of where programs in the batcher (oramacore_b200/csrc/batcher.h) with its own fake executor:
tests/batcher_where_test.cpp is compiled with g++ (no CUDA), -O2 and under ThreadSanitizer, and 16 threads submit
requests with a where program, a device filter handle or neither.  programs: merged calls carry q_where with each
request's nodes concatenated, polygon vertices rebased, handles as FILTER nodes and empty ranges for unfiltered
requests, and a program the where check refuses runs alone.  handles: with no program in the traffic, merged calls
carry q_filters as before."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=[["-O2"], ["-O1", "-g", "-fsanitize=thread"]], ids=["O2", "tsan"])
def where_exe(request, tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    flags = request.param
    exe = str(tmp_path_factory.mktemp("batcher_where") / "batcher_where_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", *flags, "-pthread", "-I", ROOT,
                        os.path.join(ROOT, "tests", "batcher_where_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize("scenario", ["programs", "handles"])
def test_batcher_carries_where_programs(where_exe, scenario):
    r = subprocess.run([where_exe, scenario], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0 bad=0" in r.stdout
