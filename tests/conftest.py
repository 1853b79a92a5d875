import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _gpu_available() -> bool:
    """True when libsnarkb200.so can open a context (sb_create != SB_ERR_NODEVICE)."""
    try:
        from snarkjs_b200 import _native
        import ctypes
        h = ctypes.c_void_p()
        rc = _native.lib().sb_create(0, 0, ctypes.byref(h))
        if rc == 0:
            _native.lib().sb_destroy(h)
        return rc == 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without CUDA skips the gpu-marked parity tests instead of erroring in their fixtures.
    (`-m gpu` on an H100 runs them; there a missing library or device is a hard failure, not a skip.)"""
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if not gpu_items or "gpu" in (config.getoption("-m") or "").replace("not gpu", ""):
        return
    if not _gpu_available():
        skip = pytest.mark.skip(reason="no CUDA device: gpu parity tests run on an H100")
        for it in gpu_items:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return dict(np.load(os.path.join(GOLDEN, name)))
    return load


@pytest.fixture(scope="session")
def reference_plonk_key():
    return _reference_plonk_key


def _reference_plonk_key(g, tag):
    """Rebuilds a PLONK zkey the reference ships (tests/golden/plonk_setup_cases.npz: its r1cs + the ptau slices `plonk setup`
    reads) with oracle.plonk.plonk_setup, and checks it is the reference's file byte for byte (sha256)."""
    import hashlib
    from oracle import oracle as orc
    from oracle import plonk
    n = int(g[f"{tag}_n"][0])
    ptau = orc.write_binfile("ptau", 1, [(1, bytes(g["ptau_header"])), (2, bytes(g[f"{tag}_ptau2"])), (3, bytes(g["ptau3"])),
                                         (12, bytes((n - 1) * 64) + bytes(g[f"{tag}_ptau12"]))])
    zkey = plonk.plonk_setup(bytes(g[f"{tag}_r1cs"]), ptau)
    assert hashlib.sha256(zkey).digest() == bytes(g[f"{tag}_zkey_sha256"]), "plonk_setup does not reproduce the reference zkey"
    return zkey, bytes(g[f"{tag}_wtns"])
