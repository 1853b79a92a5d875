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


@pytest.fixture(scope="module")
def parse_fuzz(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fuzz") / "host_parse_fuzz")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "host_parse_fuzz.cpp")])
    return exe


def test_zkey_parsers_survive_mutation_fuzzing(tmp_path, golden, parse_fuzz):
    """The zkey.h parsers (the code sb_groth16_load, sb_groth16_prove_wtns, sb_plonk_load and sb_fflonk_load run on caller
    bytes) and the host-side load logic behind them, under AddressSanitizer + UBSan on mutated containers: truncations,
    bit flips in the section table and headers, wild 32/64-bit fields, smashed section headers, garbage in the signal /
    map / coefficient sections.  Every input is either rejected with a message or read strictly inside its exact-size
    buffer, every span and CSR entry the parser returned included."""
    from oracle import plonk
    gates, adds, n_vars, n_pub, _ = plonk.chain_gates(13)
    g16 = golden("groth16_case.npz")
    cases = [("plonk", bytes(golden("plonk_case.npz")["zkey"]), 60000),
             ("plonk", plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99), 40000),     # with additions
             ("fflonk", bytes(golden("fflonk_case.npz")["zkey"]), 15000),
             ("groth16", g16["zkey"].tobytes(), 30000),
             ("wtns", g16["wtns"].tobytes(), 60000)]
    for i, (proto, data, iters) in enumerate(cases):
        path = str(tmp_path / f"k{i}.bin")
        open(path, "wb").write(data)
        out = subprocess.run([parse_fuzz, proto, path, str(iters)], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0 and "FUZZ OK" in out.stdout, out.stdout + out.stderr[-2000:]


def test_groth16_and_wtns_parsers_reject_malformed_containers(tmp_path, golden, parse_fuzz):
    """The malformed containers the GPU tests hand to sb_groth16_load, sb_groth16_load_file and sb_groth16_prove_wtns,
    parsed on the host (zero fuzzing iterations: the input as given): same rejection messages."""
    import struct
    g = golden("groth16_case.npz")
    zkey, wtns = g["zkey"].tobytes(), g["wtns"].tobytes()

    def parse(proto, data):
        path = str(tmp_path / "in.bin")
        open(path, "wb").write(data)
        out = subprocess.run([parse_fuzz, proto, path, "0"], capture_output=True, text=True, timeout=60)
        if out.returncode == 0:
            return None
        assert "the unmodified key was rejected: " in out.stderr, out.stderr[-2000:]
        return out.stderr.split("the unmodified key was rejected: ", 1)[1].splitlines()[0]

    assert parse("groth16", zkey) is None and parse("wtns", wtns) is None
    wrapped = bytearray(zkey)
    struct.pack_into("<Q", wrapped, 16, (1 << 64) - 12 - 12)        # a section length near 2^64 must not wrap the bounds check
    assert parse("groth16", bytes(wrapped)) == "Invalid file size"
    assert parse("groth16", zkey[:len(zkey) - 100]) == "Invalid file size"
    assert parse("groth16", b"nope" + zkey[4:]) == "zkey: Invalid File format"
    wrapped = bytearray(wtns)
    struct.pack_into("<Q", wrapped, 16, (1 << 64) - 24)
    assert parse("wtns", bytes(wrapped)) == "Invalid file size"
