"""CPU: sb_fflonk_prove_batch refuses a null context, its Python wrappers fail with the no-device error without a GPU, and
the ctypes signature in _native.py matches the prototype in include/snarkb200.h."""
import ctypes
import os
import re

import numpy as np
import pytest

from snarkjs_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fflonk_batch_rejects_null_context():
    L = N.lib()
    buf = ctypes.create_string_buffer(512)
    st = (ctypes.c_int32 * 2)()
    assert L.sb_fflonk_prove_batch(None, 1, buf, 1, 1, buf, buf, st) == -1
    assert L.sb_fflonk_prove_batch(None, 1, None, 0, 0, None, None, None) == -1


def test_fflonk_batch_wrappers_raise_no_device_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import snarkjs_b200
    from oracle import fflonk as ofl
    from oracle import plonk as oplonk
    gates, adds, n_vars, n_pub, wit = oplonk.chain_gates(13)
    zkey = ofl.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    wt = oplonk.wtns_bytes(wit)
    with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
        snarkjs_b200.fflonk.prove_batch(zkey, [wt, wt])
    with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
        snarkjs_b200.fflonk.ProvingKey(zkey).prove_batch_raw([np.zeros(len(wit) * 32, np.uint8)], [bytes(9 * 32)])


def test_fflonk_batch_signature_matches_header():
    hdr = open(os.path.join(ROOT, "include", "snarkb200.h")).read()
    m = re.search(r"int\s+sb_fflonk_prove_batch\s*\(([^)]*)\)\s*;", hdr)
    assert m, "prototype not found"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    want = {"uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}
    restype, argtypes = N._SIGNATURES["sb_fflonk_prove_batch"]
    assert restype is ctypes.c_int
    assert len(argtypes) == len(params) == 8
    for p, t in zip(params, argtypes):
        if "*" in p:
            assert t in (ctypes.c_void_p, ctypes.c_char_p), p
        else:
            assert t is want[p.split()[0]], p
