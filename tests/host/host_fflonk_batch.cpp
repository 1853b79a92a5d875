// Host batch backend for snarkjs_b200/csrc/fflonk_flow.h's fflonk_prove_flow_batch: the PLONK host batch backend's shared
// steps (host_plonk_batch.cpp) plus the fflonk steps as plain loops over the proofs and the same fflonk.cuh element
// functions the batched kernels call; NTT / MSM from the CPU oracle.  Commits at the batch's row length 9n and reports
// per-proof status codes.  Built as a shared library and driven by tests/test_host_fflonk_batch.py.  Test infrastructure only.
#include "host_plonk_batch.cpp"
#include "../../snarkjs_b200/csrc/fflonk_flow.h"

template <class F> struct HostFflonkBatchBackend : HostBatchBackend<F> {
    typedef HostBatchBackend<F> Base;
    using Base::one; using Base::r; using Base::n;
    std::vector<int> pending;                     // flags not yet read
    const FfQuot<F>* quot = nullptr; const FfLin<F>* lin = nullptr;

    void z_start(const PlonkKeyView<F>& k, const PlonkBatchWork<F>& w, uint32_t K) { Base::z(k, w, K, pending.data()); }
    void read_flags(int* flags) { for (size_t q = 0; q < pending.size(); q++) { flags[q] |= pending[q]; pending[q] = 0; } }
    void wire_blind(F* wires, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) for (int j = 0; j < 3; j++) ff_wire_blind<F>(wires + (j * K + q) * n, n, r[q].b[2 * j + 1], r[q].b[2 * j + 2]);
    }
    PlonkTIn tin(const FflonkKeyView<F>& k, const F* evABC, const F* evZ, uint32_t q, uint32_t K) {
        const uint64_t n4 = 4 * n;
        PlonkTIn in;
        in.A = evABC + q * n4; in.B = evABC + (K + q) * n4; in.C = evABC + (2 * K + q) * n4; in.Z = evZ ? evZ + q * n4 : nullptr;
        in.QL = k.q_ev[0]; in.QR = k.q_ev[1]; in.QM = k.q_ev[2]; in.QO = k.q_ev[3]; in.QC = k.q_ev[4];
        in.S1 = k.s_ev[0]; in.S2 = k.s_ev[1]; in.S3 = k.s_ev[2]; in.LAG = k.lag; in.pubA = nullptr; in.n_public = k.nPublic;
        return in;
    }
    void t0(const FflonkKeyView<F>& k, const F* evABC, const F* wires, F* T, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) {
            PlonkTIn in = tin(k, evABC, nullptr, q, K); in.pubA = wires + q * n;
            for (uint64_t i = 0; i < 4 * n; i++) ff_t0<F>(i, 4 * n, in, T + q * 4 * n);
        }
    }
    void t1(const FflonkKeyView<F>& k, const F* evZ, F* T, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) for (uint64_t i = 0; i < 2 * n; i++) ff_t1<F>(i, evZ + q * 4 * n, k.lag, k.w2pow, r[q], T + q * 2 * n, T + (K + q) * 2 * n);
    }
    void t2(const FflonkKeyView<F>& k, const F* evABC, const F* evZ, F* T, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) {
            const PlonkTIn in = tin(k, evABC, evZ, q, K);
            for (uint64_t i = 0; i < 4 * n; i++) ff_t2<F>(i, 4 * n, in, k.w4pow, r[q], T + q * 4 * n, T + (K + q) * 4 * n);
        }
    }
    void divzh(uint64_t nn, int blocks, const F* t, bool tz, F* out, uint64_t ostride, uint64_t bound, int shift, uint32_t K) {
        const uint64_t len = blocks * nn;
        for (uint32_t q = 0; q < K; q++) {
            int f = 0;
            for (uint64_t i = 0; i < nn; i++) f |= ff_divzh<F>(i, nn, blocks, t + q * len, tz ? t + (K + q) * len : nullptr, out + q * ostride, bound);
            pending[q] |= f << shift;
        }
    }
    void interleave(const FfParts& parts, const uint64_t strides[4], F* out, uint32_t K) {
        for (uint32_t q = 0; q < K; q++) {
            FfParts p = parts;
            for (int j = 0; j < parts.m; j++) p.p[j] = (const F*)parts.p[j] + q * strides[j];
            for (uint64_t k = 0; k < 9 * n; k++) ff_interleave<F>(k, p, out + q * 9 * n);
        }
    }
    void evals(const FflonkKeyView<F>& k, const FflonkBatchWork<F>& w, const PlonkPowK<F>* pw, uint32_t K, F* out) {
        const int segs = fflonk_batch_segs(k.c0_is_interleave);
        const FfEvalIn in = eval_in(k, w, K);
        for (uint32_t q = 0; q < K; q++)
            for (int e = 0; e < segs; e++) {
                uint64_t len; int p;
                const F* f = ff_eval_seg<F>(in, q, e, len, p);
                out[(size_t)q * segs + e] = one.eval(f, len, pw[p].at(q), nullptr, nullptr);
            }
    }
    static FfEvalIn eval_in(const FflonkKeyView<F>& k, const FflonkBatchWork<F>& w, uint32_t K) {
        FfEvalIn in;
        for (int j = 0; j < 5; j++) in.key[j] = k.q_coef[j];
        for (int j = 0; j < 3; j++) in.key[5 + j] = k.s_coef[j];
        in.key[8] = k.c0;
        in.pABC = w.pABC; in.cZ = w.cZ; in.pT0 = w.pT0; in.pT1 = w.pT1; in.pT2 = w.pT2; in.n = k.n; in.K = K; in.nz = fflonk_batch_nz(k.n);
        return in;
    }
    void set_quot(const FfQuot<F>* qt, uint32_t) { quot = qt; }
    void set_lin(const FfLin<F>* L, uint32_t) { lin = L; }
    void quot_m(const FfDiv<F>* divs, int cnt, F* G, F* P, uint32_t K) {
        for (int d = 0; d < cnt; d++) {
            const FfDiv<F>& v = divs[d];
            const uint64_t total = v.rows * v.m;
            for (uint32_t q = 0; q < K; q++) {
                const FfQuot<F>& qt = quot[(size_t)v.d * K + q];
                for (uint64_t k = 0; k < total; k++) ff_qm_g<F>(k, v.f + q * v.fs, v.len, qt.R, qt.scale, v.m, v.rows, v.bpow.at(q), G);
                for (int j = 0; j < v.m; j++) { F acc = F::zero(); for (uint64_t t = 0; t < v.rows; t++) { acc = F::add(acc, G[j * v.rows + t]); P[j * v.rows + t] = acc; } }
                F* o = v.out + q * 9 * n;
                int bad = 0;
                for (uint64_t k = 0; k < total; k++) bad |= ff_qm_q<F>(k, v.m, v.rows, P, v.ibpow.at(q), o);
                for (uint64_t k = total; k < 9 * n; k++) o[k] = F::zero();
                pending[q] |= bad;
            }
        }
    }
    void add3(uint64_t total, const F* a, const F* b, const F* c, F* out) { for (uint64_t k = 0; k < total; k++) out[k] = F::add(F::add(a[k], b[k]), c[k]); }
    void quot_l(const FflonkKeyView<F>& k, const FflonkBatchWork<F>& w, const PlonkPowK<F>& py, const PlonkPowK<F>& ipy, uint32_t K) {
        const uint64_t n9 = 9 * n;
        for (uint32_t q = 0; q < K; q++) {
            F* g = w.G; F* P = w.P;
            for (uint64_t i = 0; i < n9; i++)
                g[i] = F::mul(ff_l_coef<F>(i, k.c0, 8 * n, w.C1 + q * n9, 8 * n, w.C2 + q * n9, n9, w.Fq + q * n9, n9, lin[q]), pl_pow(py.at(q), i));
            F acc = F::zero();
            for (uint64_t i = 0; i < n9; i++) { acc = F::add(acc, g[i]); P[i] = acc; }
            for (uint64_t j = 0; j < n9; j++) w.scal[q * n9 + j] = F::from_mont(pl_quot_coef<F>(j, n9, P, ipy.at(q)));
            if (!P[n9 - 1].is_zero()) pending[q] |= 1;
        }
    }
    // the key's power-table geometry: 9n + 8 powers
    void make_pows(const F* bases, int slots, int, uint32_t K, PlonkPowK<F>* out) {
        const uint64_t big = 9 * n + PLONK_PAD;
        const int h = plonk_pow_h(big); const uint64_t nhi = (big >> h) + 1;
        for (int s = 0; s < slots; s++) {
            std::vector<F> lo_all, hi_all;
            for (uint32_t q = 0; q < K; q++) {
                std::vector<F> lo, hi; plonk_pow_tables<F>(bases[(size_t)s * K + q], h, nhi, lo, hi);
                lo_all.insert(lo_all.end(), lo.begin(), lo.end()); hi_all.insert(hi_all.end(), hi.begin(), hi.end());
            }
            this->pow_store.push_back(lo_all); this->pow_store.push_back(hi_all);
            out[s].lo = this->pow_store[this->pow_store.size() - 2].data(); out[s].hi = this->pow_store.back().data(); out[s].h = h;
            out[s].slo = (uint64_t)1 << h; out[s].shi = nhi;
        }
    }
};

template <class PQ, class PR>
static int fflonk_batch_impl(void* so, const FflonkZkey& z, const uint8_t* witnesses, uint64_t n_wit, uint32_t count, const uint8_t* blinders,
                             uint8_t* proofs, int32_t* status, std::string& err) {
    typedef Fp<PR> F;
    const int curve = 0;
    HostFflonkBatchBackend<F> be;
    HostBackend<F>& o = be.one;
    o.fft = (or_fft_t)dlsym(so, "or_fr_fft"); o.msm = (or_msm_t)dlsym(so, "or_multiexp_affine"); o.gop = (or_gop_t)dlsym(so, "or_group_op");
    or_root_t root = (or_root_t)dlsym(so, "or_fr_root");
    if (!o.fft || !o.msm || !o.gop || !root) { err = "oracle symbols missing"; return -1; }
    o.curve = curve; o.n8q = z.n8q; o.ptau = z.lay.ptau.p;
    be.pow_store.reserve(64); o.pow_store.reserve(64);
    FflonkKeyView<F> k;
    k.nVars = z.nVars; k.nPublic = z.nPublic; k.n = z.n; k.nAdditions = z.nAdditions; k.nConstraints = z.nConstraints; k.power = z.power;
    memcpy(&k.k1, z.k1, 32); memcpy(&k.k2, z.k2, 32); memcpy(&k.w3, z.w3, 32); memcpy(&k.w4, z.w4, 32); memcpy(&k.w8, z.w8, 32); memcpy(&k.wr, z.wr, 32);
    F w2n, w4n; root(curve, z.power, (uint8_t*)&k.wn); root(curve, z.power + 1, (uint8_t*)&w2n); root(curve, z.power + 2, (uint8_t*)&w4n);
    k.c0_point = z.C0; k.aff_bytes = 2 * z.n8q;
    if (fflonk_witness_length(k, n_wit, err)) return 2;
    HostKeyArrays<F> arrays; arrays.fill(z, z.lay, k);
    std::vector<F> c0;
    k.c0 = HostKeyArrays<F>::copy(c0, z.lay.c0);
    k.c0_is_interleave = fflonk_c0_is_interleave(z);
    o.make_pow(k.wn, z.n, k.wpow, 0);
    o.make_pow(w2n, 2 * z.n, k.w2pow, 0);
    o.make_pow(w4n, 4 * z.n, k.w4pow, 0);
    const uint64_t n = z.n, sW = (uint64_t)z.nVars + 2;
    be.n = n; be.P = 9 * n;
    be.pending.assign(count, 0);
    std::vector<F> work((size_t)count * fflonk_batch_elems(n, sW, k.c0_is_interleave), F::zero());
    const FflonkBatchWork<F> w = fflonk_batch_layout(work.data(), n, sW, k.c0_is_interleave, count);
    return fflonk_prove_flow_batch<PQ, PR>(be, k, w, count, witnesses, n_wit, blinders, proofs, status);
}

extern "C" {
// proofs = count x (C1 C2 W1 W2 | 16 evaluations); status = count codes (0, or 3..8 as fflonk_error_text); returns 0, 2 with
// the witness-length text, or a negative code
int hp_fflonk_prove_batch(const char* oracle_so, const uint8_t* zkey, uint64_t zlen, const uint8_t* witnesses, uint64_t n_wit, uint32_t count,
                          const uint8_t* blinders, uint8_t* proofs, int32_t* status, char* errbuf, int errlen) {
    std::string err;
    void* so = dlopen(oracle_so, RTLD_NOW);
    if (!so) { snprintf(errbuf, errlen, "dlopen failed: %s", dlerror()); return -1; }
    FflonkZkey z;
    int rc = fflonk_parse_zkey(zkey, zlen, z, err);
    if (!rc) rc = fflonk_batch_impl<BnFq, BnFr>(so, z, witnesses, n_wit, count, blinders, proofs, status, err);
    snprintf(errbuf, errlen, "%s", err.c_str());
    return rc;
}
// the reference's text of a status code
const char* hp_fflonk_error_text(int code) { return fflonk_error_text(code); }
}
