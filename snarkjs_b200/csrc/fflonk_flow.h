// fflonk_flow.h — the fflonk prover's control flow (src/fflonk_prove.js:51-1286): five rounds, the Keccak transcript, the
// opening-set roots, the three small interpolations and the batched inverse.  Pure host C++ on a Backend, exactly like
// plonk_flow.h: the CUDA backend lives in api_fflonk.inl, the host backend in tests/host/host_fflonk.cpp.
#pragma once
#include "plonk_flow.h"
#include "fflonk.cuh"

namespace sb {

// C0 == CPolynomial(8)(QL, QR, QO, QM, QC, S1, S2, S3) (src/fflonk_setup.js:441-464)?  One pass over the 8n coefficients.
inline bool fflonk_c0_is_interleave(const FflonkZkey& z) {
    const PlonkLayout& lay = z.lay;
    const Span* src[8] = {&lay.q_coef[0], &lay.q_coef[1], &lay.q_coef[3], &lay.q_coef[2], &lay.q_coef[4], &lay.s_coef[0], &lay.s_coef[1], &lay.s_coef[2]};
    for (uint64_t i = 0; i < z.n; i++)
        for (int j = 0; j < 8; j++)
            if (memcmp(lay.c0.p + (8 * i + j) * 32, src[j]->p + 32 * i, 32) != 0) return false;
    return true;
}

template <class F> struct FflonkKeyView {
    uint32_t nVars = 0, nPublic = 0, n = 0, nAdditions = 0, nConstraints = 0; int power = 0;
    F k1, k2, w3, w4, w8, wr, wn;
    const uint8_t* c0_point = nullptr; uint32_t aff_bytes = 64;
    const uint32_t* add_sig = nullptr; const F* add_fac = nullptr; const uint32_t* add_order = nullptr; std::vector<uint32_t> level_end;
    const uint32_t* map[3] = {nullptr, nullptr, nullptr};
    const F* q_coef[5] = {nullptr}; const F* q_ev[5] = {nullptr};     // QL QR QM QO QC (section order 7..11)
    const F* s_coef[3] = {nullptr}; const F* s_ev[3] = {nullptr};
    const F* lag = nullptr;                                            // max(nPublic, 1) arrays of 4n evaluations
    const F* c0 = nullptr;                                             // 8n coefficients
    bool c0_is_interleave = false;                                     // section 17 == CPolynomial(QL,QR,QO,QM,QC,S1,S2,S3) (checked at load)
    PlonkPow<F> wpow, w2pow, w4pow;                                    // powers of w_n, w_2n, w_4n
};

template <class F> struct FflonkWork {            // backend memory
    F *W = nullptr;
    F *bufA = nullptr, *bufB = nullptr, *bufC = nullptr, *bufZ = nullptr, *num = nullptr, *den = nullptr, *ratio = nullptr;   // n
    F *pA = nullptr, *pB = nullptr, *pC = nullptr;                                                                          // n
    F *cZ = nullptr;                                                                                                        // n + 8
    F *evA = nullptr, *evB = nullptr, *evC = nullptr, *evZ = nullptr, *T = nullptr, *Tz = nullptr, *s4a = nullptr, *s4b = nullptr;   // 4n
    F *pT0 = nullptr, *pT2 = nullptr;                                                                                      // 4n
    F *pT1 = nullptr;                                                                                                       // 2n
    F *C1 = nullptr;                                                                                                        // 8n
    F *C2 = nullptr, *Fq = nullptr, *F1 = nullptr, *F2 = nullptr, *G = nullptr, *P = nullptr, *scal = nullptr;              // 9n + 8
};

// Backend concept = plonk_flow.h's (upload, download, zero, copy, ntt, commit, commit_plain, additions, wires, blind, z,
// make_pow, eval) plus:
//   void wire_blind(F* A, F* B, F* C, uint64_t n, const F raw[6]);
//   void t0(const PlonkTIn&, uint64_t n4, F* T0);   void t1(uint64_t n2, const F* evZ, const F* lag1, const PlonkPow<F>&, const PlonkRound<F>&, F* T1, F* T1z);
//   void t2(const PlonkTIn&, uint64_t n4, const PlonkPow<F>&, const PlonkRound<F>&, F* T2, F* T2z);
//   int  divzh_n(uint64_t n, int blocks, const F* t, const F* tz, F* out, uint64_t bound);
//   void interleave(const FfParts&, uint64_t total, F* out);
//   int  quot_m(const F* f, uint64_t len, const FfSmall<F>& R, const F& scale, int m, uint64_t rows, const PlonkPow<F>& bpow, const PlonkPow<F>& ibpow, F* G, F* P, F* q);
//   void add3(uint64_t total, const F* a, const F* b, const F* c, F* out);
//   int  quot_l(uint64_t total, const F* C0, uint64_t l0, const F* C1, uint64_t l1, const F* C2, uint64_t l2, const F* Fp, uint64_t lf,
//               const FfLin<F>&, const PlonkPow<F>& ypow, const PlonkPow<F>& iypow, F* g, F* P, F* q_plain);
namespace ffhost {
template <class F> inline F horner(const std::vector<F>& c, const F& x) { F r = F::zero(); for (size_t i = c.size(); i-- > 0;) r = F::add(c[i], F::mul(r, x)); return r; }
// Polynomial.lagrangePolynomialInterpolation (polynomial.js:896-930)
template <class F> inline std::vector<F> interpolate(const std::vector<F>& xs, const std::vector<F>& ys) {
    const size_t m = xs.size();
    std::vector<F> res(m, F::zero());
    for (size_t i = 0; i < m; i++) {
        std::vector<F> basis(1, F::one());
        for (size_t j = 0; j < m; j++) {
            if (j == i) continue;
            std::vector<F> nxt(basis.size() + 1, F::zero());
            for (size_t k = 0; k < basis.size(); k++) { nxt[k] = F::sub(nxt[k], F::mul(basis[k], xs[j])); nxt[k + 1] = F::add(nxt[k + 1], basis[k]); }
            basis.swap(nxt);
        }
        const F f = F::mul(ys[i], F::inv(horner(basis, xs[i])));
        for (size_t k = 0; k < basis.size(); k++) res[k] = F::add(res[k], F::mul(basis[k], f));
    }
    return res;
}
}  // namespace ffhost

// ---------------------------------------------------------------------------------------------- per-proof scalar steps
// The host-side parts of one proof that both the single flow and the batched flow run.
// the reference's text for the flow's positive codes 3..8
inline const char* fflonk_error_text(int code) {
    switch (code) {
    case 3: return "Copy constraints does not match";
    case 4: return "Polynomial is not divisible";
    case 5: return "T0 Polynomial is not well calculated";
    case 6: return "T1 Polynomial is not well calculated";
    case 7: return "T2 Polynomial is not well calculated";
    case 8: return "Degree of L(X)/(ZTS2(y)(X-y)) remainder should be 0";
    default: return "";
    }
}
// fflonk_prove.js:79-81; 0 or 2 with err set
template <class F> inline int fflonk_witness_length(const FflonkKeyView<F>& k, uint64_t n_witness, std::string& err) {
    if (n_witness == (uint64_t)k.nVars - k.nAdditions) return 0;
    err = "Invalid witness length. Circuit: " + std::to_string(k.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k.nAdditions);
    return 2;
}
template <class F> inline void fflonk_round_init(const FflonkKeyView<F>& k, const uint8_t* blinders_mont /*9 x 32*/, PlonkRound<F>& r) {
    r.b[0] = F::zero(); r.b[10] = F::zero(); r.b[11] = F::zero();
    for (int i = 1; i <= 9; i++) memcpy(&r.b[i], blinders_mont + 32 * (i - 1), 32);
    r.k1 = k.k1; r.k2 = k.k2; r.wn = k.wn;
    for (int i = 0; i < 4; i++) { r.z1[i] = r.z2[i] = r.z3[i] = F::zero(); }
    r.beta = r.gamma = r.alpha = r.alpha2 = F::zero();
}
// the PlonkKeyView of the steps shared with PLONK (additions, wires, computeZ)
template <class F> inline PlonkKeyView<F> fflonk_plonk_view(const FflonkKeyView<F>& k) {
    PlonkKeyView<F> pk;
    pk.nVars = k.nVars; pk.nPublic = k.nPublic; pk.n = k.n; pk.nAdditions = k.nAdditions; pk.nConstraints = k.nConstraints; pk.power = k.power;
    pk.k1 = k.k1; pk.k2 = k.k2; pk.wn = k.wn;
    pk.add_sig = k.add_sig; pk.add_fac = k.add_fac; pk.add_order = k.add_order; pk.level_end = k.level_end;
    for (int j = 0; j < 3; j++) { pk.map[j] = k.map[j]; pk.s_ev[j] = k.s_ev[j]; pk.s_coef[j] = k.s_coef[j]; }
    pk.wpow = k.wpow;
    return pk;
}
// round 2 (:522-560): beta, gamma from C0, the public A values and C1
template <class PQ, class PR> inline void fflonk_beta_gamma(const FflonkKeyView<Fp<PR>>& k, const Fp<PR>* pubA, const uint8_t* pt_C1, PlonkRound<Fp<PR>>& r) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_point(k.c0_point);
    for (uint32_t i = 0; i < k.nPublic; i++) tr.add_scalar(pubA[i]);
    tr.add_point(pt_C1);
    r.beta = tr.challenge();
    tr.reset(); tr.add_scalar(r.beta);
    r.gamma = tr.challenge();
}
// round 3 (:832-850)
template <class PQ, class PR> inline Fp<PR> fflonk_xi_seed(const PlonkRound<Fp<PR>>& r, const uint8_t* pt_C2) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(r.gamma); tr.add_point(pt_C2);
    return tr.challenge();
}
// the opening sets S0, S1, S2, S2' (:852-880) and xi = S2[0]^3
template <class F> struct FfRoots { F S0[8], S1[4], S2[3], S2p[3], xi, xiw; };
template <class F> inline void fflonk_roots(const FflonkKeyView<F>& k, const F& xi_seed, FfRoots<F>& s) {
    const F seed2 = F::sqr(xi_seed);
    s.S0[0] = F::mul(seed2, xi_seed);
    F p = F::one(); for (int i = 1; i < 8; i++) { p = F::mul(p, k.w8); s.S0[i] = F::mul(s.S0[0], p); }
    s.S1[0] = F::sqr(s.S0[0]);
    p = F::one(); for (int i = 1; i < 4; i++) { p = F::mul(p, k.w4); s.S1[i] = F::mul(s.S1[0], p); }
    s.S2[0] = F::mul(s.S1[0], seed2); s.S2[1] = F::mul(s.S2[0], k.w3); s.S2[2] = F::mul(s.S2[0], F::sqr(k.w3));
    s.S2p[0] = F::mul(s.S2[0], k.wr); s.S2p[1] = F::mul(s.S2p[0], k.w3); s.S2p[2] = F::mul(s.S2p[0], F::sqr(k.w3));
    s.xi = F::mul(F::sqr(s.S2[0]), s.S2[0]);
    s.xiw = F::mul(s.xi, k.wn);
}
// round 4 (:933-940): ev = the 15 opening values
template <class PQ, class PR> inline Fp<PR> fflonk_alpha(const Fp<PR>& xi_seed, const Fp<PR>* ev) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(xi_seed);
    for (int j = 0; j < 15; j++) tr.add_scalar(ev[j]);
    return tr.challenge();
}
// R0, R1, R2 interpolate the combined polynomials on the opening sets (:987-1029).  The reference evaluates C0, C1, C2 at
// the 18 roots directly; because every root h of S0 / S1 / S2 / S2' satisfies h^8 = xi, h^4 = xi, h^3 = xi, h^3 = xi w, the
// same values follow from evaluations of the *parts* at xi / xi w (this is how the verifier rebuilds them,
// fflonk_verify.js:383-503):
//   C1(h) = a(xi) + h b(xi) + h^2 c(xi) + h^3 T0(xi)        C2(h) = z(x) + h T1(x) + h^2 T2(x),  x = xi or xi w
//   C0(h) = ql + h qr + h^2 qo + h^3 qm + h^4 qc + h^5 s1 + h^6 s2 + h^7 s3      (only if section 17 is that interleave)
// Same field elements, about 150 n fewer multiply-adds.  c0ys = C0(S0[i]) evaluated directly (read when C0 is not the interleave).
template <class F> inline void fflonk_interpolate(const FflonkKeyView<F>& k, const FfRoots<F>& s, const F* ev, const F& t0xi, const F& t1xi, const F& t2xi,
                                                  const F* c0ys, std::vector<F>& R0, std::vector<F>& R1, std::vector<F>& R2) {
    auto combine = [](const F* parts, int cnt, const F& h) { F acc = F::zero(); for (int j = cnt; j-- > 0;) acc = F::add(parts[j], F::mul(acc, h)); return acc; };
    std::vector<F> ys(8);
    if (k.c0_is_interleave) {
        const F parts[8] = {ev[0], ev[1], ev[3], ev[2], ev[4], ev[5], ev[6], ev[7]};            // ql qr qo qm qc s1 s2 s3
        for (int i = 0; i < 8; i++) ys[i] = combine(parts, 8, s.S0[i]);
    } else {
        for (int i = 0; i < 8; i++) ys[i] = c0ys[i];
    }
    R0 = ffhost::interpolate<F>(std::vector<F>(s.S0, s.S0 + 8), ys);
    ys.resize(4);
    { const F parts[4] = {ev[8], ev[9], ev[10], t0xi}; for (int i = 0; i < 4; i++) ys[i] = combine(parts, 4, s.S1[i]); }
    R1 = ffhost::interpolate<F>(std::vector<F>(s.S1, s.S1 + 4), ys);
    std::vector<F> xs6(s.S2, s.S2 + 3); xs6.insert(xs6.end(), s.S2p, s.S2p + 3);
    ys.resize(6);
    { const F parts[3] = {ev[11], t1xi, t2xi}; for (int i = 0; i < 3; i++) ys[i] = combine(parts, 3, s.S2[i]); }
    { const F parts[3] = {ev[12], ev[13], ev[14]}; for (int i = 0; i < 3; i++) ys[3 + i] = combine(parts, 3, s.S2p[i]); }
    R2 = ffhost::interpolate<F>(xs6, ys);
}
template <class F> inline FfSmall<F> fflonk_small(const std::vector<F>& v) {
    FfSmall<F> s; s.len = (int)v.size(); for (int i = 0; i < 8; i++) s.c[i] = i < s.len ? v[i] : F::zero(); return s;
}
// round 5 (:1059-1065)
template <class PQ, class PR> inline Fp<PR> fflonk_y(const Fp<PR>& alpha, const uint8_t* pt_W1) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(alpha); tr.add_point(pt_W1);
    return tr.challenge();
}
// the products (y - h) over S0, S1, S2 + S2'
template <class F> inline void fflonk_mul_l(const FfRoots<F>& s, const F& y, F& mulL0, F& mulL1, F& mulL2) {
    mulL0 = F::one(); mulL1 = F::one(); mulL2 = F::one();
    for (const F& x : s.S0) mulL0 = F::mul(mulL0, F::sub(y, x));
    for (const F& x : s.S1) mulL1 = F::mul(mulL1, F::sub(y, x));
    for (const F& x : s.S2) mulL2 = F::mul(mulL2, F::sub(y, x));
    for (const F& x : s.S2p) mulL2 = F::mul(mulL2, F::sub(y, x));
}
// the scalars of computeL (:1101-1180)
template <class F> inline FfLin<F> fflonk_lin(const FfRoots<F>& s, const F& alpha, const F& y, const std::vector<F>& R0, const std::vector<F>& R1,
                                              const std::vector<F>& R2) {
    F mulL0, mulL1, mulL2;
    fflonk_mul_l(s, y, mulL0, mulL1, mulL2);
    FfLin<F> L;
    L.pre0 = F::mul(mulL1, mulL2);
    L.pre1 = F::mul(alpha, F::mul(mulL0, mulL2));
    L.pre2 = F::mul(F::sqr(alpha), F::mul(mulL0, mulL1));
    L.r0y = ffhost::horner(R0, y); L.r1y = ffhost::horner(R1, y); L.r2y = ffhost::horner(R2, y);
    L.zty = F::mul(mulL0, F::mul(mulL1, mulL2));                 // ZT(y): the zerofier of all 18 roots (:1164-1172)
    L.zts2y_inv = F::inv(F::mul(mulL1, mulL2));                  // 1 / ZTS2(y) (:1174-1180)
    return L;
}
// the batched inverse (:1182-1285)
template <class F> inline F fflonk_inv(const FflonkKeyView<F>& k, const FfRoots<F>& s, const F& y) {
    F mulL0, mulL1, mulL2;
    fflonk_mul_l(s, y, mulL0, mulL1, mulL2);
    F acc = F::mul(mulL1, mulL2);                                // denH1, denH2
    acc = F::mul(acc, F::sub(fr_pow2k(s.xi, k.power), F::one()));  // zh
    auto li = [&](const F* roots, size_t ln) {
        F den1 = fr_from_u64<F>(ln), p = F::one();
        for (size_t i = 0; i + 2 < ln; i++) p = F::mul(p, roots[0]);
        den1 = F::mul(den1, p);
        for (size_t i = 0; i < ln; i++) acc = F::mul(acc, F::mul(F::mul(den1, roots[((ln - 1) * i) % ln]), F::sub(y, roots[i])));
    };
    li(s.S0, 8); li(s.S1, 4);
    const F three = fr_from_u64<F>(3);
    F den1 = F::mul(F::mul(three, s.S2[0]), F::sub(s.xi, s.xiw));
    for (int i = 0; i < 3; i++) acc = F::mul(acc, F::mul(den1, F::mul(s.S2[2 * i % 3], F::sub(y, s.S2[i]))));
    den1 = F::mul(F::mul(three, s.S2p[0]), F::sub(s.xiw, s.xi));
    for (int i = 0; i < 3; i++) acc = F::mul(acc, F::mul(den1, F::mul(s.S2p[2 * i % 3], F::sub(y, s.S2p[i]))));
    const F nf = fr_from_u64<F>(k.n);
    F wq = F::one();
    const uint32_t nl = k.nPublic > 1 ? k.nPublic : 1;
    for (uint32_t i = 0; i < nl; i++) { acc = F::mul(acc, F::mul(nf, F::sub(s.xi, wq))); wq = F::mul(wq, k.wn); }
    return F::inv(acc);
}

// Returns 0, a positive code for the reference's own errors (2 witness length, 3..8 as fflonk_error_text; err holds the
// reference's message) or the backend's negative code.
template <class PQ, class PR, class B>
int fflonk_prove_flow(B& be, const FflonkKeyView<Fp<PR>>& k, FflonkWork<Fp<PR>>& w, const uint8_t* witness_plain, uint64_t n_witness,
                      const uint8_t* blinders_mont /*9 x 32*/, uint8_t* proof_out, std::string& err) {
    typedef Fp<PR> F;
    const uint64_t n = k.n, n4 = 4 * n;
    const uint32_t aff = k.aff_bytes;
    if (fflonk_witness_length(k, n_witness, err)) return 2;
    auto fail = [&](int code) { err = fflonk_error_text(code); return code; };
    PlonkRound<F> r;
    fflonk_round_init(k, blinders_mont, r);
    uint8_t* pt_C1 = proof_out; uint8_t* pt_C2 = pt_C1 + aff; uint8_t* pt_W1 = pt_C2 + aff; uint8_t* pt_W2 = pt_W1 + aff;
    F* ev_out = (F*)(pt_W2 + aff);                                   // ql qr qm qo qc s1 s2 s3 a b c z zw t1w t2w inv

    const PlonkKeyView<F> pk = fflonk_plonk_view(k);
    PlonkWork<F> zw;                                                  // the buffers computeZ touches
    zw.bufA = w.bufA; zw.bufB = w.bufB; zw.bufC = w.bufC; zw.bufZ = w.bufZ; zw.num = w.num; zw.den = w.den; zw.ratio = w.ratio;

    // ---------------- round 1 (:319-520)
    be.upload(w.W, (const F*)witness_plain, n_witness);
    be.zero(w.W, 1);
    be.zero(w.W + n_witness, (size_t)k.nAdditions + 1);
    be.additions(pk, w.W);
    be.wires(pk, w.W, w.bufA, w.bufB, w.bufC);
    { F raw[6]; for (int i = 0; i < 6; i++) raw[i] = r.b[i + 1]; be.wire_blind(w.bufA, w.bufB, w.bufC, n, raw); }
    {
        F* bufs[3] = {w.bufA, w.bufB, w.bufC}; F* ps[3] = {w.pA, w.pB, w.pC}; F* evs[3] = {w.evA, w.evB, w.evC};
        for (int j = 0; j < 3; j++) {
            be.copy(w.num, bufs[j], n);
            F* res = be.ntt(w.num, w.den, n, true);
            be.copy(ps[j], res, n);
            be.zero(w.s4a + n, 3 * n); be.copy(w.s4a, ps[j], n);
            res = be.ntt(w.s4a, w.s4b, n4, false);
            be.copy(evs[j], res, n4);
        }
    }
    PlonkTIn tin;
    tin.A = w.evA; tin.B = w.evB; tin.C = w.evC; tin.Z = w.evZ;
    tin.QL = k.q_ev[0]; tin.QR = k.q_ev[1]; tin.QM = k.q_ev[2]; tin.QO = k.q_ev[3]; tin.QC = k.q_ev[4];
    tin.S1 = k.s_ev[0]; tin.S2 = k.s_ev[1]; tin.S3 = k.s_ev[2]; tin.LAG = k.lag; tin.pubA = w.bufA; tin.n_public = k.nPublic;
    {
        be.t0(tin, n4, w.T);
        F* ct = be.ntt(w.T, w.s4a, n4, true);
        int flag = be.divzh_n(n, 4, ct, nullptr, w.pT0, 2 * n - 2);
        if (flag & 1) return fail(4);
        if (flag & 2) return fail(5);
        FfParts parts; parts.m = 4;
        parts.p[0] = w.pA; parts.p[1] = w.pB; parts.p[2] = w.pC; parts.p[3] = w.pT0;
        parts.len[0] = parts.len[1] = parts.len[2] = n; parts.len[3] = 2 * n;
        be.interleave(parts, 8 * n, w.C1);
        int rc = be.commit(w.C1, 8 * n, pt_C1); if (rc) return rc;
    }
    be.mark(1);
    // ---------------- round 2 (:522-830)
    std::vector<F> pubA(k.nPublic);
    if (k.nPublic) be.download(pubA.data(), w.bufA, k.nPublic);
    fflonk_beta_gamma<PQ, PR>(k, pubA.data(), pt_C1, r);
    {
        int flag = be.z(pk, r, zw);
        if (flag) return fail(3);
        be.copy(w.num, w.bufZ, n);
        F* res = be.ntt(w.num, w.den, n, true);
        be.zero(w.cZ + n, PLONK_PAD); be.copy(w.cZ, res, n);
        be.zero(w.s4a + n, 3 * n); be.copy(w.s4a, w.cZ, n);
        res = be.ntt(w.s4a, w.s4b, n4, false);
        be.copy(w.evZ, res, n4);
        F bf[3] = {r.b[9], r.b[8], r.b[7]};
        be.blind(w.cZ, n, bf, 3);
        // T1 on the 2n domain
        be.t1(2 * n, w.evZ, k.lag, k.w2pow, r, w.T, w.Tz);
        F* c1 = be.ntt(w.T, w.s4a, 2 * n, true);
        F* c1z = be.ntt(w.Tz, w.s4b, 2 * n, true);
        flag = be.divzh_n(n, 2, c1, c1z, w.pT1, n + 2);
        if (flag & 1) return fail(4);
        if (flag & 2) return fail(6);
        // T2 on the 4n domain
        be.t2(tin, n4, k.w4pow, r, w.T, w.Tz);
        F* c2 = be.ntt(w.T, w.s4a, n4, true);
        F* c2z = be.ntt(w.Tz, w.s4b, n4, true);
        flag = be.divzh_n(n, 4, c2, c2z, w.pT2, 3 * n);
        if (flag & 1) return fail(4);
        if (flag & 2) return fail(7);
        FfParts parts; parts.m = 3;
        parts.p[0] = w.cZ; parts.p[1] = w.pT1; parts.p[2] = w.pT2; parts.p[3] = nullptr;
        parts.len[0] = n + 3; parts.len[1] = n + 2; parts.len[2] = 3 * n; parts.len[3] = 0;
        be.interleave(parts, 9 * n, w.C2);
        int rc = be.commit(w.C2, 9 * n, pt_C2); if (rc) return rc;
    }
    be.mark(2);
    // ---------------- round 3 (:832-931)
    const F xi_seed = fflonk_xi_seed<PQ, PR>(r, pt_C2);
    FfRoots<F> s;
    fflonk_roots(k, xi_seed, s);
    const uint64_t big = 9 * n + PLONK_PAD;
    PlonkPow<F> pxi, pxiw, ipxi, ipxiw;
    be.make_pow(s.xi, big, pxi, 0);
    be.make_pow(s.xiw, big, pxiw, 1);
    F ev[16];
    for (int j = 0; j < 5; j++) ev[j] = be.eval(k.q_coef[j], n, pxi, w.G, w.P);                     // ql qr qm qo qc
    for (int j = 0; j < 3; j++) ev[5 + j] = be.eval(k.s_coef[j], n, pxi, w.G, w.P);                 // s1 s2 s3
    ev[8] = be.eval(w.pA, n, pxi, w.G, w.P); ev[9] = be.eval(w.pB, n, pxi, w.G, w.P); ev[10] = be.eval(w.pC, n, pxi, w.G, w.P);
    ev[11] = be.eval(w.cZ, n + 3, pxi, w.G, w.P);
    ev[12] = be.eval(w.cZ, n + 3, pxiw, w.G, w.P);
    ev[13] = be.eval(w.pT1, 2 * n, pxiw, w.G, w.P);
    ev[14] = be.eval(w.pT2, 4 * n, pxiw, w.G, w.P);
    be.mark(3);
    // ---------------- round 4 (:933-1057)
    const F alpha = fflonk_alpha<PQ, PR>(xi_seed, ev);
    std::vector<F> R0, R1, R2;
    {
        const F t0xi = be.eval(w.pT0, 2 * n, pxi, w.G, w.P), t1xi = be.eval(w.pT1, 2 * n, pxi, w.G, w.P), t2xi = be.eval(w.pT2, 4 * n, pxi, w.G, w.P);
        F c0ys[8];
        if (!k.c0_is_interleave)
            for (int i = 0; i < 8; i++) { PlonkPow<F> ph; be.make_pow(s.S0[i], big, ph, 4); c0ys[i] = be.eval(k.c0, 8 * n, ph, w.G, w.P); }
        fflonk_interpolate(k, s, ev, t0xi, t1xi, t2xi, c0ys, R0, R1, R2);
    }
    be.make_pow(F::inv(s.xi), big, ipxi, 2);
    be.make_pow(F::inv(s.xiw), big, ipxiw, 3);
    {
        FfSmall<F> none; none.len = 0; for (auto& c : none.c) c = F::zero();
        // F = (C0 - R0)/(X^8 - xi) + alpha (C1 - R1)/(X^4 - xi) + alpha^2 (C2 - R2)/((X^3 - xi)(X^3 - xi w))   (:1031-1056)
        be.zero(w.Fq, big); be.zero(w.F1, big); be.zero(w.F2, big);
        int flag = be.quot_m(k.c0, 8 * n, fflonk_small(R0), F::one(), 8, n, pxi, ipxi, w.G, w.P, w.Fq);
        flag |= be.quot_m(w.C1, 8 * n, fflonk_small(R1), alpha, 4, 2 * n, pxi, ipxi, w.G, w.P, w.F1);
        flag |= be.quot_m(w.C2, 9 * n, fflonk_small(R2), F::sqr(alpha), 3, 3 * n, pxi, ipxi, w.G, w.P, w.scal);
        flag |= be.quot_m(w.scal, 9 * n, none, F::one(), 3, 3 * n, pxiw, ipxiw, w.G, w.P, w.F2);
        if (flag) return fail(4);
        be.add3(9 * n, w.Fq, w.F1, w.F2, w.Fq);
        int rc = be.commit(w.Fq, 9 * n, pt_W1); if (rc) return rc;
    }
    be.mark(4);
    // ---------------- round 5 (:1059-1180)
    const F y = fflonk_y<PQ, PR>(alpha, pt_W1);
    {
        const FfLin<F> L = fflonk_lin(s, alpha, y, R0, R1, R2);
        PlonkPow<F> py, ipy;
        be.make_pow(y, big, py, 4);
        be.make_pow(F::inv(y), big, ipy, 5);
        int flag = be.quot_l(9 * n, k.c0, 8 * n, w.C1, 8 * n, w.C2, 9 * n, w.Fq, 9 * n, L, py, ipy, w.G, w.P, w.scal);
        if (flag) return fail(8);
        int rc = be.commit_plain(w.scal, 9 * n, pt_W2); if (rc) return rc;
    }
    be.mark(5);
    ev[15] = fflonk_inv(k, s, y);
    memcpy(ev_out, ev, sizeof ev);
    return 0;
}

// ---------------------------------------------------------------------------------------------- batched flow
// K proofs against one key in lockstep, as plonk_prove_flow_batch.  Every work array holds the K proofs back to back at a
// fixed stride (array-major): a round's transforms are one strided NTT, its commitments one batch of MSM rows of the
// common length 9n (C1's zeros past 8n add nothing).  Arrays whose lifetimes do not overlap share memory: rounds 1-3 keep
// their polynomials in region U, which rounds 4-5 reuse for the divisions' scans; C1, C2, F and the MSM scalars live
// throughout.
inline uint64_t fflonk_batch_nz(uint64_t n) { return n + PLONK_PAD; }               // stride of cZ
// evaluation segments of round 3 per proof: the 15 opening values, T0, T1, T2 at xi, and C0 at S0[0..8) for a key whose
// section 17 is not the interleave of sections 7-14
inline int fflonk_batch_segs(bool c0_is_interleave) { return c0_is_interleave ? 18 : 26; }
inline uint64_t fflonk_batch_terms(uint64_t n, bool c0_is_interleave) { return 27 * n + 6 + (c0_is_interleave ? 0 : 64 * n); }
// per-proof elements of U's scratch S (rounds 1-3): the witness, the NTT data and scratch (16n), round 3's terms
inline uint64_t fflonk_batch_s(uint64_t n, uint64_t sW, bool c0_is_interleave) { return std::max({sW, 16 * n, fflonk_batch_terms(n, c0_is_interleave)}); }
// per-proof elements of U: rounds 1-3 (33n + 8 + S) or rounds 4-5 (two scans over 25n, two quotients of 9n)
inline uint64_t fflonk_batch_u(uint64_t n, uint64_t sW, bool c0_is_interleave) { return std::max(33 * n + 8 + fflonk_batch_s(n, sW, c0_is_interleave), 68 * n); }
// per-proof elements of all work arrays: U, then C1, C2, F, scal (9n each)
inline uint64_t fflonk_batch_elems(uint64_t n, uint64_t sW, bool c0_is_interleave) { return fflonk_batch_u(n, sW, c0_is_interleave) + 36 * n; }

template <class F> struct FflonkBatchWork {       // backend memory, F elements, K proofs
    uint64_t sW = 0;                              // stride of W: nVars + 2
    // rounds 1-3 (region U)
    F* wires = nullptr;                           // 3K x n: A of every proof, then B, then C (blinded evaluations)
    F* pABC = nullptr;                            // 3K x n coefficients, group-major like wires
    F* evABC = nullptr;                           // 3K x 4n
    F *pT0 = nullptr, *evZ = nullptr, *pT2 = nullptr;   // K x 4n each (T0 uses 2n, T2 3n)
    F* pT1 = nullptr;                             // K x 2n
    F* cZ = nullptr;                              // K x (n + 8)
    F* S = nullptr;                               // K x fflonk_batch_s: W, NTT data and scratch, the round-3 terms
    // rounds 4-5 (region U again)
    F *G = nullptr, *P = nullptr;                 // K x 25n each: the first three divisions' terms and sums
    F *F1 = nullptr, *F3 = nullptr, *F2 = nullptr;   // K x 9n each: alpha (C1 - R1)/(X^4 - xi), alpha^2 (C2 - R2)/(X^3 - xi), F3/(X^3 - xi w)
    // rounds 1-5
    F *C1 = nullptr, *C2 = nullptr, *Fq = nullptr, *scal = nullptr;   // K x 9n each; Fq: F (then W1's polynomial)
};
// the work arrays of K proofs at base (fflonk_batch_elems(...) x K elements)
template <class F> inline FflonkBatchWork<F> fflonk_batch_layout(F* base, uint64_t n, uint64_t sW, bool c0_is_interleave, uint64_t K) {
    FflonkBatchWork<F> w; w.sW = sW;
    const uint64_t u = fflonk_batch_u(n, sW, c0_is_interleave);
    auto at = [&](uint64_t per_proof_off) { return base + per_proof_off * K; };
    w.wires = at(0); w.pABC = at(3 * n); w.evABC = at(6 * n); w.pT0 = at(18 * n); w.evZ = at(22 * n); w.pT1 = at(26 * n); w.pT2 = at(28 * n);
    w.cZ = at(32 * n); w.S = at(33 * n + 8);
    w.G = at(0); w.P = at(25 * n); w.F1 = at(50 * n); w.F3 = at(59 * n); w.F2 = at(9 * n);   // F2: after the first scans, over G's tail
    w.C1 = at(u); w.C2 = at(u + 9 * n); w.Fq = at(u + 18 * n); w.scal = at(u + 27 * n);
    return w;
}
// one division f / (X^m - b) of every proof of a batch (K rows): f row q at f + q fs (len coefficients, zero after), R and
// scale from the quotient table's entry d, quotient row q at out + q * 9n (zero from rows m on)
template <class F> struct FfDiv { const F* f; uint64_t fs, len; int m; uint64_t rows; int d; PlonkPowK<F> bpow, ibpow; F* out; };

// Batch backend concept (BB) = plonk_flow.h's (zero, copy, copy2d, upload2d, zero2d, download2d, ntt, set_rounds, additions,
// wires, blind, make_pows, commit, commit_plain) plus:
//   void z_start(const PlonkKeyView<F>&, const PlonkBatchWork<F>&, uint32_t K);       // -> w.Z; flags bit 4 pending
//   void read_flags(int* flags);                                                       // flags[q] |= the pending flags, which clear
//   void wire_blind(F* wires, uint32_t K);                                            // ff_wire_blind on the 3K rows, b[1..6]
//   void t0(const FflonkKeyView<F>&, const F* evABC, const F* wires, F* T, uint32_t K);
//   void t1(const FflonkKeyView<F>&, const F* evZ, F* T /*K rows of 2n, then K of T1z*/, uint32_t K);
//   void t2(const FflonkKeyView<F>&, const F* evABC, const F* evZ, F* T /*K rows of 4n, then K of T2z*/, uint32_t K);
//   void divzh(uint64_t n, int blocks, const F* t, bool tz /*K more rows follow t*/, F* out, uint64_t ostride, uint64_t bound, int shift, uint32_t K);
//                                                                                       // ff_divzh; pending flags |= code << shift
//   void interleave(const FfParts& parts, const uint64_t strides[4], F* out /*K x 9n*/, uint32_t K);
//   void evals(const FflonkKeyView<F>&, const FflonkBatchWork<F>&, const PlonkPowK<F>* pw /*xi, xi w, and S0[0..8) unless the interleave*/, uint32_t K, F* out /*K x segs*/);
//   void set_quot(const FfQuot<F>* q /*4 x K, division-major*/, uint32_t K);   void set_lin(const FfLin<F>* L, uint32_t K);
//   void quot_m(const FfDiv<F>* divs, int cnt, F* G, F* P, uint32_t K);               // pending flags |= 1 on a remainder
//   void add3(uint64_t total, const F* a, const F* b, const F* c, F* out);
//   void quot_l(const FflonkKeyView<F>&, const FflonkBatchWork<F>&, const PlonkPowK<F>& py, const PlonkPowK<F>& ipy, uint32_t K);   // -> w.scal (plain); flags bit 1
// status[q] = 0 or the first code 3..8 of proof q (fflonk_error_text); a failing proof runs on with the others and its slot is
// zero-filled at the end.  Returns 0 or the backend's negative code.  The caller checks the witness length.
template <class PQ, class PR, class BB>
int fflonk_prove_flow_batch(BB& be, const FflonkKeyView<Fp<PR>>& k, const FflonkBatchWork<Fp<PR>>& w, uint32_t K, const uint8_t* witnesses_plain,
                            uint64_t n_witness, const uint8_t* blinders_mont /*K x 9 x 32*/, uint8_t* proofs_out, int32_t* status) {
    typedef Fp<PR> F;
    const uint64_t n = k.n, n4 = 4 * n, n9 = 9 * n, nz = fflonk_batch_nz(n), sW = w.sW;
    const uint32_t aff = k.aff_bytes;
    const size_t pb = 4 * (size_t)aff + 16 * 32;
    auto pt = [&](uint32_t q, int i) { return proofs_out + q * pb + (size_t)i * aff; };   // C1 C2 W1 W2
    std::vector<int> flags(K, 0);
    auto settle = [&](int bit_mask, int code) { for (uint32_t q = 0; q < K; q++) if ((flags[q] & bit_mask) && !status[q]) status[q] = code; };
    auto commit = [&](const F* coef, bool plain, int i) {
        std::vector<uint8_t> pts((size_t)K * aff);
        int rc = plain ? be.commit_plain(coef, K, pts.data()) : be.commit(coef, K, w.scal, pts.data());
        if (!rc) for (uint32_t q = 0; q < K; q++) memcpy(pt(q, i), pts.data() + (size_t)q * aff, aff);
        return rc;
    };
    const PlonkKeyView<F> pk = fflonk_plonk_view(k);
    std::vector<PlonkRound<F>> r(K);
    for (uint32_t q = 0; q < K; q++) { fflonk_round_init(k, blinders_mont + (size_t)q * 9 * 32, r[q]); status[q] = 0; }
    be.set_rounds(r.data(), K);

    // ---------------- round 1
    F* W = w.S;
    be.zero(W, (size_t)K * sW);                                                                      // W[0] = 0, additions start zeroed
    be.upload2d(W, sW, (const F*)witnesses_plain, n_witness, K);
    be.zero2d(W, sW, 1, K);
    be.additions(pk, W, sW, K);
    be.wires(pk, W, sW, w.wires, K);
    be.wire_blind(w.wires, K);
    be.copy(w.pABC, w.wires, (size_t)3 * K * n);
    F* res = be.ntt(w.pABC, w.S, 3ull * K, n, true);
    if (res != w.pABC) be.copy(w.pABC, res, (size_t)3 * K * n);
    be.zero(w.evABC, (size_t)3 * K * n4);
    be.copy2d(w.evABC, n4, w.pABC, n, n, 3ull * K);
    res = be.ntt(w.evABC, w.S, 3ull * K, n4, false);                                                // A, B, C on the 4n domain
    if (res != w.evABC) be.copy(w.evABC, res, (size_t)3 * K * n4);
    be.t0(k, w.evABC, w.wires, w.S, K);
    res = be.ntt(w.S, w.S + (size_t)K * n4, K, n4, true);
    be.divzh(n, 4, res, false, w.pT0, n4, 2 * n - 2, 0, K);
    be.read_flags(flags.data());
    settle(1, 4); settle(2, 5);
    {
        FfParts parts; parts.m = 4;
        parts.p[0] = w.pABC; parts.p[1] = w.pABC + (size_t)K * n; parts.p[2] = w.pABC + (size_t)2 * K * n; parts.p[3] = w.pT0;
        parts.len[0] = parts.len[1] = parts.len[2] = n; parts.len[3] = 2 * n;
        const uint64_t strides[4] = {n, n, n, n4};
        be.interleave(parts, strides, w.C1, K);
    }
    { int rc = commit(w.C1, false, 0); if (rc) return rc; }
    // ---------------- round 2
    {
        std::vector<F> pub((size_t)K * k.nPublic + 1);
        if (k.nPublic) be.download2d(pub.data(), w.wires, n, k.nPublic, K);
        for (uint32_t q = 0; q < K; q++) fflonk_beta_gamma<PQ, PR>(k, pub.data() + (size_t)q * k.nPublic, pt(q, 0), r[q]);
    }
    be.set_rounds(r.data(), K);
    {
        PlonkBatchWork<F> zw; zw.wires = w.wires;
        zw.num = w.S; zw.den = w.S + (size_t)K * n; zw.ratio = w.S + (size_t)2 * K * n; zw.Z = w.S + (size_t)3 * K * n;
        be.z_start(pk, zw, K);
        res = be.ntt(zw.Z, w.S + (size_t)4 * K * n, K, n, true);
    }
    be.zero(w.cZ, (size_t)K * nz);
    be.copy2d(w.cZ, nz, res, n, n, K);
    be.zero(w.evZ, (size_t)K * n4);
    be.copy2d(w.evZ, n4, w.cZ, nz, n, K);
    res = be.ntt(w.evZ, w.S, K, n4, false);
    if (res != w.evZ) be.copy(w.evZ, res, (size_t)K * n4);
    { const PlonkBlindIdx bi = {3, {{9, 8, 7}, {0, 0, 0}, {0, 0, 0}}}; be.blind(w.cZ, nz, n, 1, K, bi); }
    be.t1(k, w.evZ, w.S, K);                                                                         // T1 on the 2n domain
    res = be.ntt(w.S, w.S + (size_t)4 * K * n, 2ull * K, 2 * n, true);
    be.divzh(n, 2, res, true, w.pT1, 2 * n, n + 2, 0, K);
    be.t2(k, w.evABC, w.evZ, w.S, K);                                                                // T2 on the 4n domain
    res = be.ntt(w.S, w.S + (size_t)8 * K * n, 2ull * K, n4, true);
    be.divzh(n, 4, res, true, w.pT2, n4, 3 * n, 3, K);
    be.read_flags(flags.data());                                                                     // Z, T1, T2 in the single flow's order
    settle(4, 3); settle(1, 4); settle(2, 6); settle(8, 4); settle(16, 7);
    {
        FfParts parts; parts.m = 3;
        parts.p[0] = w.cZ; parts.p[1] = w.pT1; parts.p[2] = w.pT2; parts.p[3] = nullptr;
        parts.len[0] = n + 3; parts.len[1] = n + 2; parts.len[2] = 3 * n; parts.len[3] = 0;
        const uint64_t strides[4] = {nz, 2 * n, n4, 0};
        be.interleave(parts, strides, w.C2, K);
    }
    { int rc = commit(w.C2, false, 1); if (rc) return rc; }
    // ---------------- round 3: the 15 opening values and T0, T1, T2 at xi (and C0 at S0) in one reduction
    const int segs = fflonk_batch_segs(k.c0_is_interleave);
    std::vector<F> seeds(K), evs((size_t)segs * K);
    std::vector<FfRoots<F>> roots(K);
    PlonkPowK<F> pw[14];
    {
        std::vector<F> bases((size_t)8 * K);
        for (uint32_t q = 0; q < K; q++) {
            seeds[q] = fflonk_xi_seed<PQ, PR>(r[q], pt(q, 1));
            fflonk_roots(k, seeds[q], roots[q]);
            bases[q] = roots[q].xi; bases[K + q] = roots[q].xiw;
        }
        be.make_pows(bases.data(), 2, 0, K, pw);
        if (!k.c0_is_interleave) {
            for (int i = 0; i < 8; i++) for (uint32_t q = 0; q < K; q++) bases[(size_t)i * K + q] = roots[q].S0[i];
            be.make_pows(bases.data(), 8, 6, K, pw + 6);
        }
    }
    {
        PlonkPowK<F> epw[10];
        epw[0] = pw[0]; epw[1] = pw[1];
        for (int i = 0; i < 8; i++) epw[2 + i] = pw[6 + i];
        be.evals(k, w, epw, K, evs.data());
    }
    // ---------------- round 4
    std::vector<F> alphas(K);
    std::vector<std::vector<F>> R((size_t)3 * K);
    std::vector<FfQuot<F>> quot((size_t)4 * K);                                                      // alive for the whole call, as r
    {
        std::vector<F> ib((size_t)2 * K);
        for (uint32_t q = 0; q < K; q++) {
            const F* e = evs.data() + (size_t)q * segs;
            alphas[q] = fflonk_alpha<PQ, PR>(seeds[q], e);
            fflonk_interpolate(k, roots[q], e, e[15], e[16], e[17], e + 18, R[3 * q], R[3 * q + 1], R[3 * q + 2]);
            const F sc[4] = {F::one(), alphas[q], F::sqr(alphas[q]), F::one()};
            for (int d = 0; d < 4; d++) {
                quot[(size_t)d * K + q].R = fflonk_small(d < 3 ? R[3 * q + d] : std::vector<F>());
                quot[(size_t)d * K + q].scale = sc[d];
            }
            ib[q] = F::inv(roots[q].xi); ib[K + q] = F::inv(roots[q].xiw);
        }
        be.set_quot(quot.data(), K);
        be.make_pows(ib.data(), 2, 2, K, pw + 2);
    }
    {
        // F = (C0 - R0)/(X^8 - xi) + alpha (C1 - R1)/(X^4 - xi) + alpha^2 (C2 - R2)/((X^3 - xi)(X^3 - xi w))
        const FfDiv<F> first[3] = {{k.c0, 0, 8 * n, 8, n, 0, pw[0], pw[2], w.Fq},
                                   {w.C1, n9, 8 * n, 4, 2 * n, 1, pw[0], pw[2], w.F1},
                                   {w.C2, n9, n9, 3, 3 * n, 2, pw[0], pw[2], w.F3}};
        be.quot_m(first, 3, w.G, w.P, K);
        const FfDiv<F> second = {w.F3, n9, n9, 3, 3 * n, 3, pw[1], pw[3], w.F2};
        be.quot_m(&second, 1, w.G, w.P, K);
        be.read_flags(flags.data());
        settle(1, 4);
        be.add3((uint64_t)K * n9, w.Fq, w.F1, w.F2, w.Fq);
    }
    { int rc = commit(w.Fq, false, 2); if (rc) return rc; }
    // ---------------- round 5
    std::vector<F> ys(K);
    std::vector<FfLin<F>> L(K);
    {
        std::vector<F> yb((size_t)2 * K);
        for (uint32_t q = 0; q < K; q++) {
            ys[q] = fflonk_y<PQ, PR>(alphas[q], pt(q, 2));
            L[q] = fflonk_lin(roots[q], alphas[q], ys[q], R[3 * q], R[3 * q + 1], R[3 * q + 2]);
            yb[q] = ys[q]; yb[K + q] = F::inv(ys[q]);
        }
        be.set_lin(L.data(), K);
        be.make_pows(yb.data(), 2, 4, K, pw + 4);
    }
    be.quot_l(k, w, pw[4], pw[5], K);
    be.read_flags(flags.data());
    settle(1, 8);
    { int rc = commit(w.scal, true, 3); if (rc) return rc; }
    for (uint32_t q = 0; q < K; q++) {
        F* ev_out = (F*)(pt(q, 3) + aff);
        memcpy(ev_out, evs.data() + (size_t)q * segs, 15 * sizeof(F));
        ev_out[15] = fflonk_inv(k, roots[q], ys[q]);
    }
    for (uint32_t q = 0; q < K; q++) if (status[q]) memset(proofs_out + q * pb, 0, pb);
    return 0;
}

}  // namespace sb
