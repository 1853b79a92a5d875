"""CPU: XYZZ::add_i, the full point addition the MSM fold and bucket-reduction kernels run, gives the bytes of XYZZ::add on
all four groups (ec.cuh compiled with g++, with the PTX carry chains emulated and with the fast host multiply)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-DSB_HOST_EMULATE_PTX"], []])
def test_host_add_i_matches_add(tmp_path, flags):
    exe = str(tmp_path / "host_add_i_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", *flags, "-o", exe, os.path.join(ROOT, "tests", "host", "host_add_i_check.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "ADD_I CHECK PASSED" in out.stdout, out.stdout + out.stderr
