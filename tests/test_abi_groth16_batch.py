"""CPU: the batch entry points (sb_groth16_prove_batch, sb_msm_registered_batch) refuse a null context, their Python
wrappers fail with the no-device error without a GPU, and the sub-batch bound of msm_geom.h keeps every bucket key of a
batched sort below the INVALID key 2^32 - 1."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from snarkjs_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "snarkjs_b200", "csrc")


def test_batch_entries_reject_null_context():
    L = N.lib()
    buf = ctypes.create_string_buffer(256)
    assert L.sb_groth16_prove_batch(None, 1, buf, 1, 1, buf, buf, buf) == -1
    assert L.sb_groth16_prove_batch(None, 1, None, 0, 0, None, None, None) == -1
    assert L.sb_msm_registered_batch(None, 1, 0, buf, 32, 1, 1, buf) == -1
    assert L.sb_msm_registered_batch(None, 1, 0, None, 32, 0, 0, None) == -1


def test_batch_wrappers_raise_no_device_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import snarkjs_b200
    from snarkjs_b200 import groth16, synth
    from snarkjs_b200.curve import _Q, _R
    # a container with the chain circuit's shape and dummy bases: the key is parsed on the host, then the context fails
    zkey = synth.groth16_zkey_image(_Q[(32,)], _R["bn128"], 32, 3, lambda grp, sd, k: bytes(64 * grp * k))
    wt = synth.wtns_container(_R["bn128"], synth.chain_witness(_R["bn128"], 3))
    with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
        groth16.prove_batch(zkey, [wt, wt])
    with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
        groth16.ProvingKey(zkey).prove_batch_raw([np.zeros(8 * 32, np.uint8)], [(bytes(32), bytes(32))])


LIMIT_CHECK = r"""
#include <cstdio>
#include "msm_geom.h"
using namespace sb;
int main() {
    const uint64_t ns[] = {1, 2, 49, 1000, 4096, 65536, 1ull << 20, 1ull << 23, 1ull << 26};
    long checked = 0, bad = 0;
    for (uint64_t n : ns)
        for (int c = 3; c <= 22; c++)
            for (int sbytes = 1; sbytes <= 64; sbytes++)
                for (int pre = 0; pre <= 1; pre++) {
                    const int W = (8 * sbytes + 1 + c - 1) / c;
                    MsmGeom g; g.c = c; g.W = W; g.B = 1u << (c - 1); g.precomp = pre;
                    const uint64_t K = msm_batch_limit(n, c, W, pre);
                    // the largest key of the batch, and the number of sorted entries
                    const unsigned __int128 keys = (unsigned __int128)K * g.windows_per_proof() * g.B;
                    const unsigned __int128 entries = (unsigned __int128)K * n * (uint64_t)W;
                    const unsigned __int128 keys1 = (unsigned __int128)(K + 1) * g.windows_per_proof() * g.B;
                    const unsigned __int128 entries1 = (unsigned __int128)(K + 1) * n * (uint64_t)W;
                    // K = 0: not even one vector fits the bound (sets above 2^23 points, which the library cuts into chunks)
                    if (keys >= 0xffffffffull || entries > 0xffffffffull) { bad++; printf("over: n=%llu c=%d W=%d pre=%d K=%llu\n", (unsigned long long)n, c, W, pre, (unsigned long long)K); }
                    if (keys1 < 0xffffffffull && entries1 <= 0xffffffffull) { bad++; printf("not the largest: n=%llu c=%d W=%d pre=%d K=%llu\n", (unsigned long long)n, c, W, pre, (unsigned long long)K); }
                    g.K = (uint32_t)(K < 0xffffffffull ? K : 0xffffffffull);
                    if (K <= 0xffffffffull && (uint64_t)g.windows() * g.B != (uint64_t)keys) { bad++; printf("windows() disagrees\n"); }
                    checked++;
                }
    printf("checked %ld bad %ld\n", checked, bad);
    return bad ? 1 : 0;
}
"""


def test_batch_limit_keeps_keys_below_invalid(tmp_path):
    """Every (n, c, W, table mode) the library can meet: K * windows_per_proof * B < 2^32 - 1 and K * n * W < 2^32 hold for
    the K msm_batch_limit returns, and K + 1 breaks one of them (the limit is the largest such batch; 0 when one vector
    already breaks them)."""
    src = tmp_path / "limit.cpp"
    src.write_text(LIMIT_CHECK)
    exe = str(tmp_path / "limit")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + CSRC, "-o", exe, str(src)])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr
    assert "bad 0" in out.stdout
