"""CPU: the exact fp.cuh / ec.cuh template code the kernels use, compiled with g++ (PTX carry chains emulated and the
fast host multiply), checked against the oracle: field ops on all four fields, XYZZ mixed/full adds incl. doubling,
cancellation and infinity cases."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-DSB_HOST_EMULATE_PTX"], []])
def test_host_fp_check(tmp_path, flags):
    from oracle import oracle as O
    so = O.build()
    exe = str(tmp_path / "host_fp_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", *flags, "-o", exe, os.path.join(ROOT, "tests", "host", "host_fp_check.cpp"), "-ldl"])
    out = subprocess.run([exe, so], capture_output=True, text=True)
    assert out.returncode == 0 and "HOST CHECK PASSED" in out.stdout, out.stdout + out.stderr


def test_zkey_parsers_survive_mutation_fuzzing(tmp_path, golden):
    """plonk_parse_zkey / fflonk_parse_zkey (the code sb_plonk_load / sb_fflonk_load run on caller bytes) and the host-side
    load logic behind them, under AddressSanitizer + UBSan on mutated containers: truncations, bit flips in the section
    table and headers, wild 32/64-bit fields, smashed section headers, garbage in the signal / map sections.  Every input is
    either rejected with a message or read strictly inside its exact-size buffer."""
    from oracle import plonk
    exe = str(tmp_path / "host_parse_fuzz")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "host_parse_fuzz.cpp")])
    gates, adds, n_vars, n_pub, _ = plonk.chain_gates(13)
    cases = [("plonk", bytes(golden("plonk_case.npz")["zkey"]), 60000),
             ("plonk", plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99), 40000),     # with additions
             ("fflonk", bytes(golden("fflonk_case.npz")["zkey"]), 15000)]
    for i, (proto, zkey, iters) in enumerate(cases):
        path = str(tmp_path / f"k{i}.zkey")
        open(path, "wb").write(zkey)
        out = subprocess.run([exe, proto, path, str(iters)], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0 and "FUZZ OK" in out.stdout, out.stdout + out.stderr[-2000:]
