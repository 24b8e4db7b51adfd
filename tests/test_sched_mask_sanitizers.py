"""Constrained requests in the session scheduler (jlama_b200/csrc/jl_sched.cu) under AddressSanitizer + UBSan and ThreadSanitizer: the
mask provider runs on the stepping thread without the scheduler's lock and calls jl_sched_result / jl_sched_cancel while producer
threads submit constrained requests (tests/native/sched_mask_sanitize.cpp).  A data race, a use-after-free or an overflow ends the run
with a non-zero exit code; the harness itself checks that every constrained token was allowed and that the provider saw each selection
once."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "native", "sched_mask_sanitize.cpp")


@pytest.mark.parametrize("name,flags", [("asan_ubsan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"]), ("tsan", ["-fsanitize=thread"])])
def test_constrained_scheduler_under_sanitizers(tmp_path, name, flags):
    exe = str(tmp_path / ("sched_mask_" + name))
    cmd = ["g++", "-std=c++17", "-x", "c++", "-g", "-O1", "-Wno-subobject-linkage", "-I", os.path.join(ROOT, "include")] + flags + [SRC, "-o", exe, "-pthread"]
    b = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=os.path.dirname(SRC))
    if b.returncode != 0 and ("cannot find" in b.stdout or "unrecognized" in b.stdout):
        pytest.skip("this g++ has no %s runtime: %s" % (name, b.stdout[-200:]))
    assert b.returncode == 0, b.stdout[-2000:]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66", ASAN_OPTIONS="detect_leaks=1", UBSAN_OPTIONS="halt_on_error=1")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().splitlines()[-1].startswith("ok:"), r.stdout[-4000:]
    assert "WARNING: ThreadSanitizer" not in r.stdout and "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout
