"""CPU-only: the request combiner behind the herumi-API entry points (harmony_b200/csrc/coalesce.hpp) with a fake executor under
ThreadSanitizer -- 1, 2, 8 and 64 caller threads, thousands of requests: every request gets its own result exactly once, turn sizes
add up, a lone request runs as a turn of one on its own thread, requests over a cap wait for the next turn, a failing turn fails
its requests and only those, and nothing deadlocks (timeout)."""
import os, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def test_combiner_under_thread_sanitizer(tmp_path):
    src = os.path.join(ROOT, "tests", "coalesce", "coalesce_driver.cpp")
    exe = str(tmp_path / "coalesce_driver")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=thread", "-pthread", "-o", exe, src])
    env = {**os.environ, "TSAN_OPTIONS": "halt_on_error=1 exitcode=66"}
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stdout and "ThreadSanitizer" not in r.stderr, r.stdout + r.stderr
