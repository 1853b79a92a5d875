"""GPU: the in-library multi-GPU Groth16 path (sb_comm_*, sb_groth16_prove_dist, sb_*_multi).
The world-1 case runs on one GPU (NCCL loaded, communicator of one rank, every exchange step executed); the
world-2 / world-N cases need that many devices and are skipped otherwise.  In every case the
distributed proof must equal the single-GPU proof byte for byte, which itself equals the CPU oracle's
(tests/test_gpu_parity.py)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402  (checker only)


def _ndev():
    import torch
    return torch.cuda.device_count()


def test_world_1_communicator_matches_plain_prove():
    import snarkjs_b200
    from snarkjs_b200 import groth16, synth
    c = snarkjs_b200.getCurveFromName("bn128")
    L = 14
    zkey = synth.synth_groth16_zkey(c, L, seed=21)
    w = synth.chain_witness(c.r, L)
    ci = O.CURVES[O.BN254]
    r, s = ci.fr_to_mont(1234), ci.fr_to_mont(4321)
    pk = groth16.ProvingKey(zkey, curve=c)
    want = pk.prove_raw(w, r, s)
    oproof, _ = O.groth16_prove(zkey, synth.wtns_container(c.r, w), r, s)
    assert groth16.proof_to_object(c, want) == oproof
    c.comm_init(1, 0, c.comm_unique_id())
    assert pk.prove_dist(w, r, s) == want
    assert pk.prove_dist(None, r, s) == want          # resident witness
    pk.release()
    c.terminate()


@pytest.mark.parametrize("L", [10, 15])
def test_single_process_multi_gpu_proof_equals_single_gpu(L):
    n = min(_ndev(), 8)
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    import snarkjs_b200
    from snarkjs_b200 import groth16, synth, _native
    from snarkjs_b200.curve import _ptr
    lib = _native.lib()
    c0 = snarkjs_b200.getCurveFromName("bn128")
    zkey = synth.synth_groth16_zkey(c0, L, seed=33)
    w = synth.chain_witness(c0.r, L)
    ci = O.CURVES[O.BN254]
    r, s = ci.fr_to_mont(777), ci.fr_to_mont(888)
    pk = groth16.ProvingKey(zkey, curve=c0)
    want = pk.prove_raw(w, r, s)
    pk.release()
    c0.terminate()
    for world in sorted({2, n}):
        devs = (ctypes.c_int * world)(*range(world))
        ctxs = (ctypes.c_void_p * world)()
        assert lib.sb_create_multi(0, devs, world, ctxs) == 0
        handles = (ctypes.c_uint64 * world)()
        zb = np.frombuffer(zkey, np.uint8)
        assert lib.sb_groth16_load_multi(ctxs, world, _ptr(zb), zb.size, handles) == 0, lib.sb_last_error(ctxs[0])
        out = np.zeros(256, np.uint8)
        for _ in range(2):
            rc = lib.sb_groth16_prove_multi(ctxs, handles, world, _ptr(w), w.size // 32, r, s, _ptr(out))
            assert rc == 0, [lib.sb_last_error(ctxs[i]) for i in range(world)]
            assert out.tobytes() == want, f"world {world}"
        for i in range(world):
            lib.sb_destroy(ctxs[i])
