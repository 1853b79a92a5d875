// Host batch backend for snarkjs_b200/csrc/plonk_flow.h's plonk_prove_flow_batch: the batch steps as plain loops over the
// proofs and the same plonk.cuh element functions the batched kernels call, NTT / MSM borrowed from the CPU oracle through
// host_backend.h.  Commits at the batch's padded length n + 6 and reports per-proof status codes.  Built as a shared
// library and driven by tests/test_host_plonk_batch.py.  Test infrastructure only.
#include "host_backend.h"

template <class F> struct HostBatchBackend {
    HostBackend<F> one;                           // oracle NTT / MSM and the single-proof helpers
    const PlonkRound<F>* r = nullptr;
    const PlonkLin<F>* L = nullptr; const F* ezw = nullptr;
    uint64_t n = 0, P = 0;
    std::vector<std::vector<F>> pow_store;

    void zero(F* p, size_t cnt) { memset(p, 0, cnt * sizeof(F)); }
    void copy(F* dst, const F* src, size_t cnt) { memmove(dst, src, cnt * sizeof(F)); }
    void copy2d(F* dst, uint64_t dp, const F* src, uint64_t sp, uint64_t width, uint64_t rows) { for (uint64_t i = 0; i < rows; i++) memmove(dst + i * dp, src + i * sp, width * sizeof(F)); }
    void upload2d(F* dst, uint64_t dp, const F* host, uint64_t width, uint64_t rows) { copy2d(dst, dp, host, width, width, rows); }
    void zero2d(F* dst, uint64_t dp, uint64_t width, uint64_t rows) { for (uint64_t i = 0; i < rows; i++) zero(dst + i * dp, width); }
    void download2d(F* host, const F* src, uint64_t sp, uint64_t width, uint64_t rows) { copy2d(host, width, src, sp, width, rows); }
    F* ntt(F* a, F* b, uint64_t count, uint64_t len, bool inverse) {
        for (uint64_t i = 0; i < count; i++) one.ntt(a + i * len, b + i * len, len, inverse);
        return b;
    }
    void set_rounds(const PlonkRound<F>* rr, uint32_t) { r = rr; }
    void set_lin(const PlonkLin<F>* LL, const F* e, uint32_t) { L = LL; ezw = e; }
    void additions(const PlonkKeyView<F>& k, F* W, uint64_t sW, uint32_t K) { for (uint32_t q = 0; q < K; q++) one.additions(k, W + q * sW); }
    void wires(const PlonkKeyView<F>& k, const F* W, uint64_t sW, F* out, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) one.wires(k, W + q * sW, out + q * k.n, out + (K + q) * k.n, out + (2 * K + q) * k.n);
    }
    void blind(F* p, uint64_t stride, uint64_t nn, uint32_t groups, uint32_t K, const PlonkBlindIdx& bi) {
        for (uint32_t row = 0; row < groups * K; row++) {
            const uint32_t j = row / K, q = row % K;
            F bf[3]; for (int t = 0; t < bi.cnt; t++) bf[t] = r[q].b[bi.idx[j][t]];
            pl_blind<F>(p + row * stride, nn, bf, bi.cnt);
        }
    }
    void z(const PlonkKeyView<F>& k, const PlonkBatchWork<F>& w, uint32_t K, int* flags) {
        for (uint32_t q = 0; q < K; q++) {
            PlonkWork<F> s;
            s.bufA = w.wires + q * n; s.bufB = w.wires + (K + q) * n; s.bufC = w.wires + (2 * K + q) * n;
            s.num = w.num + q * n; s.den = w.den + q * n; s.ratio = w.ratio + q * n; s.bufZ = w.Z + q * n;
            flags[q] |= one.z(k, r[q], s);
        }
    }
    void t(const PlonkKeyView<F>& k, const F* ev, const F* evZ, const F* wires, F* T, uint32_t K) {
        const uint64_t n4 = 4 * n;
        for (uint32_t q = 0; q < K; q++) {
            PlonkWork<F> s;
            s.evA = (F*)ev + q * n4; s.evB = (F*)ev + (K + q) * n4; s.evC = (F*)ev + (2 * K + q) * n4; s.evZ = (F*)evZ + q * n4;
            s.bufA = (F*)wires + q * n; s.T = T + q * n4; s.Tz = T + (K + q) * n4;
            one.t(k, r[q], s);
        }
    }
    void divzh(uint64_t nn, const F* t, F* out, uint32_t K, int* flags) {
        for (uint32_t q = 0; q < K; q++) flags[q] |= one.divzh(nn, t + q * 4 * nn, t + (K + q) * 4 * nn, out + q * 4 * nn);
    }
    void tsplit(uint64_t nn, const F* t, F* cT, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) one.tsplit(nn, t + q * 4 * nn, r[q].b[10], r[q].b[11], cT + q * P, cT + (K + q) * P, cT + (2 * K + q) * P);
    }
    void make_pows(const F* bases, int slots, int, uint32_t K, PlonkPowK<F>* out) {
        const int h = plonk_pow_h(n + PLONK_PAD); const uint64_t nhi = ((n + PLONK_PAD) >> h) + 1;
        for (int s = 0; s < slots; s++) {
            std::vector<F> lo_all, hi_all;
            for (uint32_t q = 0; q < K; q++) {
                std::vector<F> lo, hi; plonk_pow_tables<F>(bases[(size_t)s * K + q], h, nhi, lo, hi);
                lo_all.insert(lo_all.end(), lo.begin(), lo.end()); hi_all.insert(hi_all.end(), hi.begin(), hi.end());
            }
            pow_store.push_back(lo_all); pow_store.push_back(hi_all);
            out[s].lo = pow_store[pow_store.size() - 2].data(); out[s].hi = pow_store.back().data(); out[s].h = h;
            out[s].slo = (uint64_t)1 << h; out[s].shi = nhi;
        }
    }
    void evals(const PlonkKeyView<F>& k, const PlonkBatchWork<F>& w, const PlonkPowK<F>& pxi, const PlonkPowK<F>& pxiw, uint32_t K, F* out) {
        for (uint32_t q = 0; q < K; q++) {
            const F* fs[6] = {w.cABC + q * P, w.cABC + (K + q) * P, w.cABC + (2 * K + q) * P, k.s_coef[0], k.s_coef[1], w.cZ + q * P};
            const uint64_t len[6] = {n + 2, n + 2, n + 2, n, n, n + 3};
            for (int e = 0; e < 6; e++) out[6 * q + e] = one.eval(fs[e], len[e], e == 5 ? pxiw.at(q) : pxi.at(q), nullptr, nullptr);
        }
    }
    void quotients(const PlonkKeyView<F>& k, const PlonkBatchWork<F>& w, const PlonkPowK<F> pw[4], uint32_t K, int* flags) {
        for (uint32_t q = 0; q < K; q++) {
            PlonkLinIn in;
            in.QM = k.q_coef[0]; in.QL = k.q_coef[1]; in.QR = k.q_coef[2]; in.QO = k.q_coef[3]; in.QC = k.q_coef[4];
            in.S1 = k.s_coef[0]; in.S2 = k.s_coef[1]; in.S3 = k.s_coef[2];
            in.A = w.cABC + q * P; in.B = w.cABC + (K + q) * P; in.C = w.cABC + (2 * K + q) * P; in.Z = w.cZ + q * P;
            in.T1 = w.cT + q * P; in.T2 = w.cT + (K + q) * P; in.T3 = w.cT + (2 * K + q) * P;
            F* g = w.X; F* Ps = w.Y;
            F* q1 = w.scal + q * P; F* q2 = w.scal + (K + q) * P;
            flags[q] |= one.quotient(nullptr, &in, &L[q], n, 0, n + 6, F::zero(), pw[0].at(q), pw[2].at(q), g, Ps, q1);
            zero(q2, P);
            flags[q] |= one.quotient(w.cZ + q * P, nullptr, nullptr, n, n + 3, n + 3, ezw[q], pw[1].at(q), pw[3].at(q), g, Ps, q2);
        }
    }
    int commit(const F* coef, uint32_t rows, F*, uint8_t* affine) {
        for (uint32_t i = 0; i < rows; i++) { int rc = one.commit(coef + i * P, P, affine + (size_t)i * 2 * one.n8q); if (rc) return rc; }
        return 0;
    }
    int commit_plain(const F* scal, uint32_t rows, uint8_t* affine) {
        for (uint32_t i = 0; i < rows; i++) { int rc = one.commit_plain(scal + i * P, P, affine + (size_t)i * 2 * one.n8q); if (rc) return rc; }
        return 0;
    }
};

template <class PQ, class PR>
static int prove_batch_impl(void* so, int curve, const PlonkZkey& z, const uint8_t* witnesses, uint64_t n_wit, uint32_t count, const uint8_t* blinders,
                            uint8_t* proofs, int32_t* status, std::string& err) {
    typedef Fp<PR> F;
    HostBatchBackend<F> be;
    HostBackend<F>& o = be.one;
    o.fft = (or_fft_t)dlsym(so, "or_fr_fft"); o.msm = (or_msm_t)dlsym(so, "or_multiexp_affine"); o.gop = (or_gop_t)dlsym(so, "or_group_op");
    or_root_t root = (or_root_t)dlsym(so, "or_fr_root");
    if (!o.fft || !o.msm || !o.gop || !root) { err = "oracle symbols missing"; return -1; }
    o.curve = curve; o.n8q = z.n8q; o.ptau = z.lay.ptau.p;
    PlonkKeyView<F> k;
    k.nVars = z.nVars; k.nPublic = z.nPublic; k.n = z.n; k.nAdditions = z.nAdditions; k.nConstraints = z.nConstraints; k.power = z.power;
    memcpy(&k.k1, z.k1, 32); memcpy(&k.k2, z.k2, 32);
    F w2; root(curve, z.power, (uint8_t*)&k.wn); root(curve, z.power + 2, (uint8_t*)&k.w4n); root(curve, 2, (uint8_t*)&w2);
    plonk_mulz_tables<F>(w2, k.z1, k.z2, k.z3);
    k.hdr_pts = z.hdr_pts; k.aff_bytes = 2 * z.n8q;
    if (plonk_witness_length(k, n_wit, err)) return 2;
    const uint64_t n = z.n, P = plonk_batch_p(n);
    be.n = n; be.P = P;
    HostKeyArrays<F> arrays; arrays.fill(z, z.lay, k);
    o.make_pow(k.wn, n, k.wpow, 0);
    o.make_pow(k.w4n, 4 * n, k.w4pow, 0);
    const uint64_t K = count;
    std::vector<std::vector<F>> store;
    auto alloc = [&](size_t cnt) { store.emplace_back(cnt, F::zero()); return store.back().data(); };
    PlonkBatchWork<F> w;
    w.sW = z.nVars + 2;
    w.W = alloc(K * w.sW); w.wires = alloc(3 * K * n);
    w.num = alloc(K * n); w.den = alloc(K * n); w.ratio = alloc(K * n); w.Z = alloc(K * n);
    w.cABC = alloc(3 * K * P); w.cZ = alloc(K * P); w.cT = alloc(3 * K * P); w.scal = alloc(3 * K * P);
    w.evZ = alloc(K * 4 * n); w.X = alloc(K * plonk_batch_xy(n)); w.Y = alloc(K * plonk_batch_xy(n));
    return plonk_prove_flow_batch<PQ, PR>(be, k, w, count, witnesses, n_wit, blinders, proofs, status);
}

extern "C" {
// proofs = count x (9 affine points | 6 evaluations); status = count codes (0, or 3..5 as plonk_error_text); returns 0, 2 with
// the witness-length text, or a negative code
int hp_plonk_prove_batch(const char* oracle_so, const uint8_t* zkey, uint64_t zlen, const uint8_t* witnesses, uint64_t n_wit, uint32_t count,
                         const uint8_t* blinders, uint8_t* proofs, int32_t* status, char* errbuf, int errlen) {
    std::string err;
    void* so = dlopen(oracle_so, RTLD_NOW);
    if (!so) { snprintf(errbuf, errlen, "dlopen failed: %s", dlerror()); return -1; }
    PlonkZkey z;
    int rc = plonk_parse_zkey(zkey, zlen, z, err);
    if (!rc) {
        if (z.n8q == 32) rc = prove_batch_impl<BnFq, BnFr>(so, 0, z, witnesses, n_wit, count, blinders, proofs, status, err);
        else rc = prove_batch_impl<BlsFq, BlsFr>(so, 1, z, witnesses, n_wit, count, blinders, proofs, status, err);
    }
    snprintf(errbuf, errlen, "%s", err.c_str());
    return rc;
}
}
