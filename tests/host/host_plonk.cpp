// Host backend for snarkjs_b200/csrc/plonk_flow.h: the PLONK control flow and the plonk.cuh element functions
// compiled with g++, bulk NTT / MSM borrowed from the CPU oracle (dlopen).  Built as a shared library and driven by
// tests/test_host_plonk.py, which compares the proof bytes with oracle/plonk.py.  Test infrastructure only.
#include "host_backend.h"

template <class PQ, class PR>
static int prove_impl(void* so, int curve, const PlonkZkey& z, const uint8_t* witness, uint64_t n_wit, const uint8_t* blinders, uint8_t* proof, std::string& err) {
    typedef Fp<PR> F;
    HostBackend<F> be;
    be.fft = (or_fft_t)dlsym(so, "or_fr_fft"); be.msm = (or_msm_t)dlsym(so, "or_multiexp_affine"); be.gop = (or_gop_t)dlsym(so, "or_group_op");
    or_root_t root = (or_root_t)dlsym(so, "or_fr_root");
    if (!be.fft || !be.msm || !be.gop || !root) { err = "oracle symbols missing"; return -1; }
    be.curve = curve; be.n8q = z.n8q; be.ptau = z.lay.ptau.p;
    be.pow_store.reserve(64);
    PlonkKeyView<F> k;
    k.nVars = z.nVars; k.nPublic = z.nPublic; k.n = z.n; k.nAdditions = z.nAdditions; k.nConstraints = z.nConstraints; k.power = z.power;
    memcpy(&k.k1, z.k1, 32); memcpy(&k.k2, z.k2, 32);
    F w2; root(curve, z.power, (uint8_t*)&k.wn); root(curve, z.power + 2, (uint8_t*)&k.w4n); root(curve, 2, (uint8_t*)&w2);
    plonk_mulz_tables<F>(w2, k.z1, k.z2, k.z3);
    k.hdr_pts = z.hdr_pts; k.aff_bytes = 2 * z.n8q;
    const uint64_t n = z.n;
    HostKeyArrays<F> arrays; arrays.fill(z, z.lay, k);
    be.make_pow(k.wn, n, k.wpow, 0);
    be.make_pow(k.w4n, 4 * n, k.w4pow, 0);
    PlonkWork<F> w;
    std::vector<std::vector<F>> store;
    auto alloc = [&](size_t cnt) { store.emplace_back(cnt, F::zero()); return store.back().data(); };
    store.reserve(64);
    w.W = alloc(z.nVars + 2);
    w.bufA = alloc(n); w.bufB = alloc(n); w.bufC = alloc(n); w.bufZ = alloc(n); w.num = alloc(n); w.den = alloc(n); w.ratio = alloc(n); w.sn = alloc(n);
    w.cA = alloc(n + 8); w.cB = alloc(n + 8); w.cC = alloc(n + 8); w.cZ = alloc(n + 8); w.T1 = alloc(n + 8); w.T2 = alloc(n + 8); w.T3 = alloc(n + 8);
    w.g = alloc(n + 8); w.P = alloc(n + 8); w.scal = alloc(n + 8);
    w.evA = alloc(4 * n); w.evB = alloc(4 * n); w.evC = alloc(4 * n); w.evZ = alloc(4 * n); w.T = alloc(4 * n); w.Tz = alloc(4 * n); w.s4a = alloc(4 * n); w.s4b = alloc(4 * n);
    return plonk_prove_flow<PQ, PR>(be, k, w, witness, n_wit, blinders, proof, err);
}

extern "C" {
int hp_keccak256(const uint8_t* data, uint64_t len, uint8_t* out) { keccak256(data, len, out); return 0; }

// proof = 9 affine points (Montgomery) | 6 evaluations (Montgomery); returns 0 or a negative code with err filled
int hp_plonk_prove(const char* oracle_so, const uint8_t* zkey, uint64_t zlen, const uint8_t* witness, uint64_t n_wit, const uint8_t* blinders,
                   uint8_t* proof, char* errbuf, int errlen) {
    std::string err;
    void* so = dlopen(oracle_so, RTLD_NOW);
    if (!so) { snprintf(errbuf, errlen, "dlopen failed: %s", dlerror()); return -1; }
    PlonkZkey z;
    int rc = plonk_parse_zkey(zkey, zlen, z, err);
    if (!rc) {
        if (z.n8q == 32) rc = prove_impl<BnFq, BnFr>(so, 0, z, witness, n_wit, blinders, proof, err);
        else rc = prove_impl<BlsFq, BlsFr>(so, 1, z, witness, n_wit, blinders, proof, err);
    }
    snprintf(errbuf, errlen, "%s", err.c_str());
    return rc;
}
}
