"""CPU: the C-ABI library loads and exports every symbol include/snarkb200.h declares; host-only entry points work;
device entry points fail loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

from snarkjs_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    h = open(os.path.join(ROOT, "include", "snarkb200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    return sorted(set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", h)))


def test_library_exports_every_declared_symbol():
    assert os.path.exists(N.LIB_PATH), "libsnarkb200.so not built (python __graft_entry__.py)"
    L = ctypes.CDLL(N.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(L, s), f"{s} declared in snarkb200.h but not exported"
    # the ctypes binding covers the same set
    assert set(N.EXPORTED_SYMBOLS) == set(syms), set(N.EXPORTED_SYMBOLS) ^ set(syms)
    assert N.lib().sb_version().startswith(b"snarkb200")


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import snarkjs_b200
    with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
        snarkjs_b200.getCurveFromName("bn128")
    with pytest.raises(snarkjs_b200.SbError, match="Curve not supported"):
        snarkjs_b200.getCurveFromName("secp256k1")


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "snarkjs_b200")
    for dirpath, _d, files in os.walk(pkg):
        if "build" in dirpath:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".inl")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "liboracle" not in txt and "from oracle" not in txt and "import oracle" not in txt and "snark_oracle" not in txt, f


def test_shard_range_partitions():
    L = N.lib()
    for total in (0, 1, 7, 1000, 1 << 20, (1 << 20) + 3):
        for ws in (1, 2, 3, 8):
            nxt, tot = 0, 0
            for r in range(ws):
                a, b = ctypes.c_uint64(), ctypes.c_uint64()
                L.sb_shard_range(total, r, ws, ctypes.byref(a), ctypes.byref(b))
                assert a.value == min(nxt, total) or b.value == 0
                nxt = a.value + b.value
                tot += b.value
            assert tot == total and nxt == total


def test_msm_chunk_tuning_is_bounded():
    """sb_set_tuning(6, v) sets chunks of 2^v points: 0 (the 2^23 default) and 1..23 are taken; a negative log, one past the
    default and shift counts of 64 and more (undefined for the 64-bit chunk size) are SB_ERR_ARG.  No device is needed."""
    L = N.lib()
    try:
        for v in (0, 1, 23):
            assert L.sb_set_tuning(6, v) == 0, v
        for v in (-1, 24, 64, 1 << 30):
            assert L.sb_set_tuning(6, v) == -1, v
    finally:
        assert L.sb_set_tuning(6, 0) == 0


def test_prover_entry_points_reject_null_context():
    """The PLONK / fflonk entry points return SB_ERR_ARG (-1) instead of touching a null context."""
    L = N.lib()
    h = ctypes.c_uint64()
    buf = ctypes.create_string_buffer(64)
    for load in (L.sb_plonk_load, L.sb_fflonk_load):
        assert load(None, buf, 64, ctypes.byref(h)) == -1
    for load_file in (L.sb_plonk_load_file, L.sb_fflonk_load_file):
        assert load_file(None, b"/nonexistent.zkey", ctypes.byref(h)) == -1
    for prove in (L.sb_plonk_prove, L.sb_fflonk_prove):
        assert prove(None, 1, buf, 1, buf.raw, buf) == -1
    for release in (L.sb_plonk_release, L.sb_fflonk_release):
        assert release(None, 1) == -1
    assert L.sb_plonk_proof_bytes(None) == 0 and L.sb_fflonk_proof_bytes(None) == 0
    assert L.sb_plonk_info(None, 1, None, None, None, None) == -1 and L.sb_fflonk_info(None, 1, None, None, None, None) == -1


def test_dist_entry_points_without_gpu():
    """Chain placement is a pure function; the communicator entry points refuse null contexts; asking for a unique id
    loads libnccl.so.2 lazily (present in this image) without touching a device."""
    L = N.lib()
    assert [L.sb_dist_chain_owner(j, 1) for j in range(3)] == [0, 0, 0]
    assert [L.sb_dist_chain_owner(j, 2) for j in range(3)] == [0, 1, 0]
    assert [L.sb_dist_chain_owner(j, 8) for j in range(3)] == [0, 1, 2]
    idb = np.zeros(128, np.uint8)
    assert L.sb_comm_init_rank(None, 2, 0, idb.ctypes.data_as(ctypes.c_void_p)) == -1
    assert L.sb_groth16_prove_dist(None, 1, None, 0, None, None, None) == -1
    assert L.sb_comm_info(None, None, None) == -1


def test_napi_shim_compiles_links_and_reports_no_device(tmp_path):
    """integration/napi/snarkb200_napi.cc cannot be built for Node here (no node, no node-addon-api).  It is compiled against
    an in-process stand-in for the N-API classes it uses (tests/host/napi_stub/napi.h), linked against the real
    libsnarkb200.so and driven by tests/host/napi_shim_check.cpp: every C-ABI call of the shim type-checks against
    include/snarkb200.h, all sixteen functions snarkb200.mjs calls are exported, and createContext surfaces the library's
    no-device error without a GPU (with a GPU the same driver pushes an NTT and an MSM through the AsyncWorkers)."""
    import subprocess
    from snarkjs_b200 import _native
    exe = str(tmp_path / "napi_shim_check")
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + os.path.join(ROOT, "tests", "host", "napi_stub"), "-I" + os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(ROOT, "tests", "host", "napi_shim_check.cpp"), "-L" + libdir, "-lsnarkb200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "SHIM CHECK PASSED" in out.stdout, out.stdout + out.stderr
