"""GPU: the bench workloads of BASELINE.json config #5 at a size the CPU port finishes in seconds — PLONK on BLS12-381 and
fflonk on BN254 at domain 2^16 (the verdict's ">= 2^18" cases run in bench.py --workload plonk|fflonk at 2^20 with the same
live comparison).  The key is built by snarkjs_b200/synth.py with the library's NTT; the CPU port (tests/host/ flow compiled
with OpenMP, oracle NTT / MSM) proves the key built with the oracle's NTT.  Both keys must be the same bytes and both proofs
the same bytes; the resident-witness entry must reproduce the proof."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("proto,cname,L", [("plonk", "bls12381", 16), ("fflonk", "bn128", 16), ("plonk", "bn128", 13)])
def test_bench_workload_matches_cpu_port(proto, cname, L):
    import snarkjs_b200
    from snarkjs_b200 import fflonk, plonk, synth
    import bench_plonk as B
    curve = snarkjs_b200.getCurveFromName(cname)
    try:
        zkey, wit = (synth.synth_plonk_zkey if proto == "plonk" else synth.synth_fflonk_zkey)(curve, L)
        ozkey, owit, ci = B.oracle_key(proto, cname, L)
        assert hashlib.sha256(zkey).digest() == hashlib.sha256(ozkey).digest(), "GPU-built and oracle-built keys differ"
        assert wit.tobytes() == owit.tobytes()
        mod = plonk if proto == "plonk" else fflonk
        pk = mod.ProvingKey(zkey, curve)
        bl = B._blinders(curve.r, proto)
        raw = pk.prove_raw(wit, bl)
        _, want = B.cpu_prove(proto, ozkey, owit, ci.r, ci.n8q, 8)
        assert raw == want
        assert pk.prove_raw(None, bl) == raw                       # witness resident in HBM
        bl2 = bl[32:] + bl[:32]
        assert pk.prove_raw(None, bl2) == pk.prove_raw(wit, bl2) != raw
        pk.release()
    finally:
        curve.terminate()


def test_resident_needs_a_witness():
    import snarkjs_b200
    from snarkjs_b200 import plonk, synth
    from snarkjs_b200.curve import SbError
    import bench_plonk as B
    curve = snarkjs_b200.getCurveFromName("bn128")
    try:
        zkey, wit = synth.synth_plonk_zkey(curve, 8)
        pk = plonk.ProvingKey(zkey, curve)
        with pytest.raises(SbError, match="no witness resident"):
            pk.prove_raw(None, B._blinders(curve.r, "plonk"))
        pk.release()
    finally:
        curve.terminate()


@pytest.mark.parametrize("proto,cname,L", [("plonk", "bls12381", 18), ("fflonk", "bn128", 18), ("plonk", "bls12381", 20), ("fflonk", "bn128", 20)])
def test_bench_workload_at_config_size_matches_committed_cpu_hash(proto, cname, L):
    """BASELINE config #5 at 2^18 and at its stated size 2^20: the proof of the bench key equals the CPU port's, through
    the hash the CPU port committed (tests/golden/bench_proof_hashes.json, made by make_bench_hashes.py; the port needs
    40 s per 2^20 proof, so it is not re-run here), from a host witness and from the resident one.

    The same key then proves a batch of three copies of the witness in sub-batches of 2 and 1 (sb_set_tuning(14, 2)),
    with the bench blinders, other blinders and the bench blinders again: slots 0 and 2 have the committed hash, slot 1
    is prove_raw's proof, and the resident witness still gives the committed proof.  This runs the batch flow at the
    configuration sizes: the commitment sort of 3K' rows, the keyed scans and segmented reductions over tens of millions
    of elements, the sub-batch sized from free memory and the three-pass strided NTTs.  fflonk at 2^20 has rows of
    9n = 9 * 2^20 > 2^23 points, more than one MSM chunk, so its batch is the unforced run of the row-by-row commitments."""
    import snarkjs_b200
    from snarkjs_b200 import fflonk, plonk, synth
    import bench_plonk as B
    from bench import proof_hash
    want = B.golden_hash(proto, cname, L)
    assert want, "no committed hash for this workload"
    curve = snarkjs_b200.getCurveFromName(cname)
    try:
        zkey, wit = (synth.synth_plonk_zkey if proto == "plonk" else synth.synth_fflonk_zkey)(curve, L)
        mod = plonk if proto == "plonk" else fflonk
        pk = mod.ProvingKey(zkey, curve)
        del zkey
        bl = B._blinders(curve.r, proto)
        raw = pk.prove_raw(wit, bl)
        assert proof_hash(mod.proof_to_object(curve, raw)) == want
        assert pk.prove_raw(None, bl) == raw
        row = (1 << L) + 6 if proto == "plonk" else 9 << L          # points per commitment row of a batch
        assert (row > 1 << 23) == (proto == "fflonk" and L == 20)   # only fflonk at 2^20 commits row by row unforced
        bl2 = bl[32:] + bl[:32]
        try:
            assert curve.lib.sb_set_tuning(14, 2) == 0
            got = pk.prove_batch_raw([wit] * 3, [bl, bl2, bl])
        finally:
            curve.lib.sb_set_tuning(14, 0)
        assert got[0] == got[2] == raw
        assert pk.prove_raw(None, bl) == raw                       # the batch left the resident witness as it was
        assert got[1] == pk.prove_raw(wit, bl2) != raw
        pk.release()
    finally:
        curve.terminate()


def test_groth16_2_20_eight_point_range_shards_match_oracle_hash():
    """BASELINE config #4's layout at the benchmark size on one device: the 2^20 bench key loaded as eight point-range
    shards (each with its own window tables, 1/8 of the key per load), every shard's five partial MSMs, the gathered
    partials finished to the proof -- which must be the CPU oracle's proof of this key (committed hash) and the unsharded
    key's proof."""
    import snarkjs_b200
    from snarkjs_b200 import groth16, synth
    from bench import golden_hash, proof_hash
    L, NS = 20, 8
    want = golden_hash("groth16", "bn128", L, False)
    assert want
    curve = snarkjs_b200.getCurveFromName("bn128")
    try:
        zkey = synth.synth_groth16_zkey(curve, L, seed=1)
        w = synth.chain_witness(curve.r, L)
        r = (5 * (1 << 256) % curve.r).to_bytes(32, "little")
        s = (7 * (1 << 256) % curve.r).to_bytes(32, "little")
        parts = []
        for i in range(NS):                       # one shard resident at a time: what one GPU of eight holds
            k = groth16.ProvingKey(zkey, curve=curve, shard=i, n_shards=NS)
            parts.append(np.array(k.prove_shard(w, i, NS), copy=True))
            if i < NS - 1:
                k.release()
        proof = k.finish(np.concatenate(parts), NS, r, s)
        k.release()
        assert proof_hash(groth16.proof_to_object(curve, proof)) == want
        full = groth16.ProvingKey(zkey, curve=curve)
        assert full.prove_raw(w, r, s) == proof
        full.release()
    finally:
        curve.terminate()
