"""Host logic of the in-process collective group (oramacore_b200/csrc/comm_local.h), the transport that lets several
contexts of one process, e.g. on one GPU, run a sharded search together: tests/comm_local_test.cpp is compiled with g++
(no CUDA), -O2 and under ThreadSanitizer.  W = 1, 2, 3 and 16 threads run thousands of rounds of all-gathers (0-byte
ones included) and u32 sums (in place and not), checked against a plain loop over what every rank sent; ranks that
call different collectives or sizes all fail and the next round succeeds; a rank that leaves fails the waiting ranks at
once; a rank that never arrives fails the others after the timeout, named in the error."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=[["-O2"], ["-O1", "-g", "-fsanitize=thread"]], ids=["O2", "tsan"])
def comm_exe(request, tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    flags = request.param
    exe = str(tmp_path_factory.mktemp("comm_local") / "comm_local_test")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", *flags, "-pthread",
                        os.path.join(ROOT, "tests", "comm_local_test.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "-fsanitize=thread" in flags:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize("scenario", [["rounds", "1"], ["rounds", "2"], ["rounds", "3"], ["rounds", "16"],
                                      ["mismatch"], ["leave"], ["timeout"]], ids=lambda s: "-".join(s))
def test_comm_local_group(comm_exe, scenario):
    r = subprocess.run([comm_exe, *scenario], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-2000:])
    assert "wrong=0" in r.stdout and "checked=0 " not in r.stdout, r.stdout
