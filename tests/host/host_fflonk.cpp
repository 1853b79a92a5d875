// Host backend for snarkjs_b200/csrc/fflonk_flow.h: the fflonk control flow and the fflonk.cuh / plonk.cuh element
// functions compiled with g++; bulk NTT / MSM borrowed from the CPU oracle.  Driven by tests/test_host_fflonk.py, which
// compares the proof with oracle/fflonk.py.  Test infrastructure only.
#include "host_backend.h"
#include "../../snarkjs_b200/csrc/fflonk_flow.h"

template <class F> struct HostFflonkBackend : HostBackend<F> {
    void wire_blind(F* A, F* B, F* C, uint64_t n, const F raw[6]) { F* bufs[3] = {A, B, C}; for (int j = 0; j < 3; j++) ff_wire_blind<F>(bufs[j], n, raw[2 * j], raw[2 * j + 1]); }
    void t0(const PlonkTIn& in, uint64_t n4, F* T0) { _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < n4; i++) ff_t0<F>(i, n4, in, T0); }
    void t1(uint64_t n2, const F* evZ, const F* lag1, const PlonkPow<F>& w2pow, const PlonkRound<F>& r, F* T1, F* T1z) { _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < n2; i++) ff_t1<F>(i, evZ, lag1, w2pow, r, T1, T1z); }
    void t2(const PlonkTIn& in, uint64_t n4, const PlonkPow<F>& w4pow, const PlonkRound<F>& r, F* T2, F* T2z) { _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < n4; i++) ff_t2<F>(i, n4, in, w4pow, r, T2, T2z); }
    int divzh_n(uint64_t n, int blocks, const F* t, const F* tz, F* out, uint64_t bound) { int f = 0; _Pragma("omp parallel for schedule(static) reduction(|:f)") for (uint64_t i = 0; i < n; i++) f |= ff_divzh<F>(i, n, blocks, t, tz, out, bound); return f; }
    void interleave(const FfParts& parts, uint64_t total, F* out) { _Pragma("omp parallel for schedule(static)") for (uint64_t k = 0; k < total; k++) ff_interleave<F>(k, parts, out); }
    int quot_m(const F* f, uint64_t len, const FfSmall<F>& R, const F& scale, int m, uint64_t rows, const PlonkPow<F>& bpow, const PlonkPow<F>& ibpow, F* G, F* P, F* q) {
        const uint64_t total = rows * m;
        std::vector<F> src(f, f + (len < total ? len : total));           // f may alias q (second division of f3)
        _Pragma("omp parallel for schedule(static)") for (uint64_t k = 0; k < total; k++) ff_qm_g<F>(k, src.data(), src.size(), R, scale, m, rows, bpow, G);
        for (int j = 0; j < m; j++) { F acc = F::zero(); for (uint64_t t = 0; t < rows; t++) { acc = F::add(acc, G[j * rows + t]); P[j * rows + t] = acc; } }   // segmented scan
        int bad = 0;
        _Pragma("omp parallel for schedule(static) reduction(|:bad)") for (uint64_t k = 0; k < total; k++) bad |= ff_qm_q<F>(k, m, rows, P, ibpow, q);
        return bad;
    }
    void add3(uint64_t total, const F* a, const F* b, const F* c, F* out) { _Pragma("omp parallel for schedule(static)") for (uint64_t k = 0; k < total; k++) out[k] = F::add(F::add(a[k], b[k]), c[k]); }
    int quot_l(uint64_t total, const F* C0, uint64_t l0, const F* C1, uint64_t l1, const F* C2, uint64_t l2, const F* Fp, uint64_t lf,
               const FfLin<F>& L, const PlonkPow<F>& ypow, const PlonkPow<F>& iypow, F* g, F* P, F* q_plain) {
        _Pragma("omp parallel for schedule(static)") for (uint64_t k = 0; k < total; k++) g[k] = F::mul(ff_l_coef<F>(k, C0, l0, C1, l1, C2, l2, Fp, lf, L), pl_pow(ypow, k));
        F acc = F::zero();
        for (uint64_t k = 0; k < total; k++) { acc = F::add(acc, g[k]); P[k] = acc; }
        _Pragma("omp parallel for schedule(static)") for (uint64_t j = 0; j < total; j++) q_plain[j] = F::from_mont(pl_quot_coef<F>(j, total, P, iypow));
        return P[total - 1].is_zero() ? 0 : 1;
    }
};

template <class PQ, class PR>
static int prove_impl(void* so, int curve, const FflonkZkey& z, const uint8_t* witness, uint64_t n_wit, const uint8_t* blinders, uint8_t* proof, std::string& err) {
    typedef Fp<PR> F;
    HostFflonkBackend<F> be;
    be.fft = (or_fft_t)dlsym(so, "or_fr_fft"); be.msm = (or_msm_t)dlsym(so, "or_multiexp_affine"); be.gop = (or_gop_t)dlsym(so, "or_group_op");
    or_root_t root = (or_root_t)dlsym(so, "or_fr_root");
    if (!be.fft || !be.msm || !be.gop || !root) { err = "oracle symbols missing"; return -1; }
    const uint64_t n = z.n;
    // the reference reserves 16n points and leaves zeros past 9n + 18 (fflonk_prove.js:164-169); 9n + 18 are enough here
    be.curve = curve; be.n8q = z.n8q; be.ptau = z.lay.ptau.p;
    be.pow_store.reserve(256);
    FflonkKeyView<F> k;
    k.nVars = z.nVars; k.nPublic = z.nPublic; k.n = z.n; k.nAdditions = z.nAdditions; k.nConstraints = z.nConstraints; k.power = z.power;
    memcpy(&k.k1, z.k1, 32); memcpy(&k.k2, z.k2, 32); memcpy(&k.w3, z.w3, 32); memcpy(&k.w4, z.w4, 32); memcpy(&k.w8, z.w8, 32); memcpy(&k.wr, z.wr, 32);
    F w2n, w4n; root(curve, z.power, (uint8_t*)&k.wn); root(curve, z.power + 1, (uint8_t*)&w2n); root(curve, z.power + 2, (uint8_t*)&w4n);
    k.c0_point = z.C0; k.aff_bytes = 2 * z.n8q;
    HostKeyArrays<F> arrays; arrays.fill(z, z.lay, k);
    std::vector<F> c0;
    k.c0 = HostKeyArrays<F>::copy(c0, z.lay.c0);
    k.c0_is_interleave = fflonk_c0_is_interleave(z);
    be.make_pow(k.wn, n, k.wpow, 0);
    be.make_pow(w2n, 2 * n, k.w2pow, 0);
    be.make_pow(w4n, 4 * n, k.w4pow, 0);
    FflonkWork<F> w;
    std::vector<std::vector<F>> store;
    store.reserve(64);
    auto alloc = [&](size_t cnt) { store.emplace_back(cnt, F::zero()); return store.back().data(); };
    w.W = alloc(z.nVars + 2);
    w.bufA = alloc(n); w.bufB = alloc(n); w.bufC = alloc(n); w.bufZ = alloc(n); w.num = alloc(n); w.den = alloc(n); w.ratio = alloc(n);
    w.pA = alloc(n); w.pB = alloc(n); w.pC = alloc(n); w.cZ = alloc(n + 8);
    w.evA = alloc(4 * n); w.evB = alloc(4 * n); w.evC = alloc(4 * n); w.evZ = alloc(4 * n); w.T = alloc(4 * n); w.Tz = alloc(4 * n); w.s4a = alloc(4 * n); w.s4b = alloc(4 * n);
    w.pT0 = alloc(4 * n); w.pT2 = alloc(4 * n); w.pT1 = alloc(2 * n); w.C1 = alloc(8 * n);
    w.C2 = alloc(9 * n + 8); w.Fq = alloc(9 * n + 8); w.F1 = alloc(9 * n + 8); w.F2 = alloc(9 * n + 8); w.G = alloc(9 * n + 8); w.P = alloc(9 * n + 8); w.scal = alloc(9 * n + 8);
    return fflonk_prove_flow<PQ, PR>(be, k, w, witness, n_wit, blinders, proof, err);
}

extern "C" {
// proof = C1 C2 W1 W2 (affine Montgomery) | 16 evaluations (Montgomery): ql qr qm qo qc s1 s2 s3 a b c z zw t1w t2w inv
int hp_fflonk_prove(const char* oracle_so, const uint8_t* zkey, uint64_t zlen, const uint8_t* witness, uint64_t n_wit, const uint8_t* blinders,
                    uint8_t* proof, char* errbuf, int errlen) {
    std::string err;
    void* so = dlopen(oracle_so, RTLD_NOW);
    if (!so) { snprintf(errbuf, errlen, "dlopen failed: %s", dlerror()); return -1; }
    FflonkZkey z;
    int rc = fflonk_parse_zkey(zkey, zlen, z, err);
    if (!rc) {
        if (z.n8q == 32) rc = prove_impl<BnFq, BnFr>(so, 0, z, witness, n_wit, blinders, proof, err);
        else rc = prove_impl<BlsFq, BlsFr>(so, 1, z, witness, n_wit, blinders, proof, err);
    }
    snprintf(errbuf, errlen, "%s", err.c_str());
    return rc;
}
}
