"""CPU-only: the host rendezvous of a local group (badslam_b200/csrc/rendezvous.hpp), driven by tests/harness/rendezvous_main.cpp
with 2..9 std::threads and no GPU:

* thousands of rounds per group size, every rank receiving every rank's slot of the same round (generations in order);
* a poison from any rank releases every rank waiting in that round, and every later round returns at once;
* reset restores service;
* the same program under AddressSanitizer + UBSan and under ThreadSanitizer (skipped when g++ has no such runtime).
Every run has a time limit, so a rank that waits forever fails the test instead of hanging it."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "harness", "rendezvous_main.cpp")


def _build(tmp_path, sanitize):
    exe = str(tmp_path / "rendezvous")
    cmd = ["g++", "-O2" if not sanitize else "-O1", "-g", "-std=c++17", "-pthread", SRC, "-o", exe]
    if sanitize:
        cmd[1:1] = [f"-fsanitize={sanitize}", "-fno-omit-frame-pointer"]
    built = subprocess.run(cmd, capture_output=True, text=True)
    if built.returncode != 0:
        if sanitize:
            pytest.skip(f"no {sanitize} runtime for this g++: " + built.stderr[-200:])
        raise AssertionError(built.stderr)
    return exe


@pytest.mark.parametrize("sanitize,rounds", [(None, 20000), ("address,undefined", 5000), ("thread", 2000)],
                         ids=["plain", "asan", "tsan"])
def test_rendezvous(tmp_path, sanitize, rounds):
    exe = _build(tmp_path, sanitize)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", TSAN_OPTIONS="halt_on_error=1")
    run = subprocess.run([exe, str(rounds)], capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0, (run.stdout[-2000:], run.stderr[-2000:])
    for bad in ("runtime error", "AddressSanitizer", "ThreadSanitizer"):
        assert bad not in run.stderr, run.stderr[-2000:]
    for n in range(2, 10):
        assert f"n {n}: {rounds} rounds in order" in run.stdout
        assert f"n {n}: poison from every rank releases every waiter; reset restores service" in run.stdout
    assert "outside poison releases the waiting ranks" in run.stdout and "all ok" in run.stdout
