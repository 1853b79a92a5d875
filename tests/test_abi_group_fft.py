"""CPU (and GPU when present): the N-API shim's group-FFT workers (groupFft, groupApplyKey) compile against the N-API
stand-in, type-check against include/snarkb200.h, link against libsnarkb200.so and are exported; with a GPU the driver
also pushes a group ifft and a batchApplyKey through them (tests/host/napi_group_fft_check.cpp)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_napi_group_fft_workers(tmp_path):
    from snarkjs_b200 import _native
    exe = str(tmp_path / "napi_group_fft_check")
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + os.path.join(ROOT, "tests", "host", "napi_stub"), "-I" + os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(ROOT, "tests", "host", "napi_group_fft_check.cpp"), "-L" + libdir, "-lsnarkb200",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "GROUP FFT SHIM CHECK PASSED" in out.stdout, out.stdout + out.stderr
