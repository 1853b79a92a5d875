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

template <class PQ, class PR, class B>
int fflonk_prove_flow(B& be, const FflonkKeyView<Fp<PR>>& k, FflonkWork<Fp<PR>>& w, const uint8_t* witness_plain, uint64_t n_witness,
                      const uint8_t* blinders_mont /*9 x 32*/, uint8_t* proof_out, std::string& err) {
    typedef Fp<PR> F;
    const uint64_t n = k.n, n4 = 4 * n;
    const uint32_t aff = k.aff_bytes;
    if (n_witness != (uint64_t)k.nVars - k.nAdditions) {                                             // fflonk_prove.js:79-81
        err = "Invalid witness length. Circuit: " + std::to_string(k.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k.nAdditions);
        return 2;
    }
    PlonkRound<F> r;
    r.b[0] = F::zero(); r.b[10] = F::zero(); r.b[11] = F::zero();
    for (int i = 1; i <= 9; i++) memcpy(&r.b[i], blinders_mont + 32 * (i - 1), 32);
    r.k1 = k.k1; r.k2 = k.k2; r.wn = k.wn;
    for (int i = 0; i < 4; i++) { r.z1[i] = r.z2[i] = r.z3[i] = F::zero(); }
    r.beta = r.gamma = r.alpha = r.alpha2 = F::zero();
    uint8_t* pt_C1 = proof_out; uint8_t* pt_C2 = pt_C1 + aff; uint8_t* pt_W1 = pt_C2 + aff; uint8_t* pt_W2 = pt_W1 + aff;
    F* ev_out = (F*)(pt_W2 + aff);                                   // ql qr qm qo qc s1 s2 s3 a b c z zw t1w t2w inv

    // PlonkKeyView for the steps shared with PLONK (additions, wires, computeZ)
    PlonkKeyView<F> pk;
    pk.nVars = k.nVars; pk.nPublic = k.nPublic; pk.n = k.n; pk.nAdditions = k.nAdditions; pk.nConstraints = k.nConstraints; pk.power = k.power;
    pk.k1 = k.k1; pk.k2 = k.k2; pk.wn = k.wn;
    pk.add_sig = k.add_sig; pk.add_fac = k.add_fac; pk.add_order = k.add_order; pk.level_end = k.level_end;
    for (int j = 0; j < 3; j++) { pk.map[j] = k.map[j]; pk.s_ev[j] = k.s_ev[j]; pk.s_coef[j] = k.s_coef[j]; }
    pk.wpow = k.wpow;
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
        if (flag & 1) { err = "Polynomial is not divisible"; return 4; }
        if (flag & 2) { err = "T0 Polynomial is not well calculated"; return 4; }
        FfParts parts; parts.m = 4;
        parts.p[0] = w.pA; parts.p[1] = w.pB; parts.p[2] = w.pC; parts.p[3] = w.pT0;
        parts.len[0] = parts.len[1] = parts.len[2] = n; parts.len[3] = 2 * n;
        be.interleave(parts, 8 * n, w.C1);
        int rc = be.commit(w.C1, 8 * n, pt_C1); if (rc) return rc;
    }
    be.mark(1);
    // ---------------- round 2 (:522-830)
    PlonkTranscript<PQ, PR> tr;
    std::vector<F> pubA(k.nPublic);
    if (k.nPublic) be.download(pubA.data(), w.bufA, k.nPublic);
    tr.add_point(k.c0_point);
    for (uint32_t i = 0; i < k.nPublic; i++) tr.add_scalar(pubA[i]);
    tr.add_point(pt_C1);
    r.beta = tr.challenge();
    tr.reset(); tr.add_scalar(r.beta);
    r.gamma = tr.challenge();
    {
        int flag = be.z(pk, r, zw);
        if (flag) { err = "Copy constraints does not match"; return 3; }
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
        if (flag & 1) { err = "Polynomial is not divisible"; return 4; }
        if (flag & 2) { err = "T1 Polynomial is not well calculated"; return 4; }
        // T2 on the 4n domain
        be.t2(tin, n4, k.w4pow, r, w.T, w.Tz);
        F* c2 = be.ntt(w.T, w.s4a, n4, true);
        F* c2z = be.ntt(w.Tz, w.s4b, n4, true);
        flag = be.divzh_n(n, 4, c2, c2z, w.pT2, 3 * n);
        if (flag & 1) { err = "Polynomial is not divisible"; return 4; }
        if (flag & 2) { err = "T2 Polynomial is not well calculated"; return 4; }
        FfParts parts; parts.m = 3;
        parts.p[0] = w.cZ; parts.p[1] = w.pT1; parts.p[2] = w.pT2; parts.p[3] = nullptr;
        parts.len[0] = n + 3; parts.len[1] = n + 2; parts.len[2] = 3 * n; parts.len[3] = 0;
        be.interleave(parts, 9 * n, w.C2);
        int rc = be.commit(w.C2, 9 * n, pt_C2); if (rc) return rc;
    }
    be.mark(2);
    // ---------------- round 3 (:832-931)
    tr.reset(); tr.add_scalar(r.gamma); tr.add_point(pt_C2);
    const F xi_seed = tr.challenge();
    std::vector<F> S0(8), S1(4), S2(3), S2p(3);
    {
        const F seed2 = F::sqr(xi_seed);
        S0[0] = F::mul(seed2, xi_seed);
        F p = F::one(); for (int i = 1; i < 8; i++) { p = F::mul(p, k.w8); S0[i] = F::mul(S0[0], p); }
        S1[0] = F::sqr(S0[0]);
        p = F::one(); for (int i = 1; i < 4; i++) { p = F::mul(p, k.w4); S1[i] = F::mul(S1[0], p); }
        S2[0] = F::mul(S1[0], seed2); S2[1] = F::mul(S2[0], k.w3); S2[2] = F::mul(S2[0], F::sqr(k.w3));
        S2p[0] = F::mul(S2[0], k.wr); S2p[1] = F::mul(S2p[0], k.w3); S2p[2] = F::mul(S2p[0], F::sqr(k.w3));
    }
    const F xi = F::mul(F::sqr(S2[0]), S2[0]);
    const F xiw = F::mul(xi, k.wn);
    const uint64_t big = 9 * n + PLONK_PAD;
    PlonkPow<F> pxi, pxiw, ipxi, ipxiw;
    be.make_pow(xi, big, pxi, 0);
    be.make_pow(xiw, big, pxiw, 1);
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
    tr.reset(); tr.add_scalar(xi_seed);
    for (int j = 0; j < 15; j++) tr.add_scalar(ev[j]);
    const F alpha = tr.challenge();
    // R0, R1, R2 interpolate the combined polynomials on the opening sets (:987-1029).  The reference evaluates C0, C1, C2 at
    // the 18 roots directly; because every root h of S0 / S1 / S2 / S2' satisfies h^8 = xi, h^4 = xi, h^3 = xi, h^3 = xi w, the
    // same values follow from evaluations of the *parts* at xi / xi w (this is how the verifier rebuilds them,
    // fflonk_verify.js:383-503):
    //   C1(h) = a(xi) + h b(xi) + h^2 c(xi) + h^3 T0(xi)        C2(h) = z(x) + h T1(x) + h^2 T2(x),  x = xi or xi w
    //   C0(h) = ql + h qr + h^2 qo + h^3 qm + h^4 qc + h^5 s1 + h^6 s2 + h^7 s3      (only if section 17 is that interleave)
    // Same field elements, about 150 n fewer multiply-adds.
    std::vector<F> R0, R1, R2;
    {
        const F t0xi = be.eval(w.pT0, 2 * n, pxi, w.G, w.P), t1xi = be.eval(w.pT1, 2 * n, pxi, w.G, w.P), t2xi = be.eval(w.pT2, 4 * n, pxi, w.G, w.P);
        auto combine = [](const F* parts, int cnt, const F& h) { F acc = F::zero(); for (int j = cnt; j-- > 0;) acc = F::add(parts[j], F::mul(acc, h)); return acc; };
        std::vector<F> ys(8);
        if (k.c0_is_interleave) {
            const F parts[8] = {ev[0], ev[1], ev[3], ev[2], ev[4], ev[5], ev[6], ev[7]};            // ql qr qo qm qc s1 s2 s3
            for (int i = 0; i < 8; i++) ys[i] = combine(parts, 8, S0[i]);
        } else {
            for (int i = 0; i < 8; i++) { PlonkPow<F> ph; be.make_pow(S0[i], big, ph, 4); ys[i] = be.eval(k.c0, 8 * n, ph, w.G, w.P); }
        }
        R0 = ffhost::interpolate<F>(S0, ys);
        ys.resize(4);
        { const F parts[4] = {ev[8], ev[9], ev[10], t0xi}; for (int i = 0; i < 4; i++) ys[i] = combine(parts, 4, S1[i]); }
        R1 = ffhost::interpolate<F>(S1, ys);
        std::vector<F> xs6(S2); xs6.insert(xs6.end(), S2p.begin(), S2p.end());
        ys.resize(6);
        { const F parts[3] = {ev[11], t1xi, t2xi}; for (int i = 0; i < 3; i++) ys[i] = combine(parts, 3, S2[i]); }
        { const F parts[3] = {ev[12], ev[13], ev[14]}; for (int i = 0; i < 3; i++) ys[3 + i] = combine(parts, 3, S2p[i]); }
        R2 = ffhost::interpolate<F>(xs6, ys);
    }
    be.make_pow(F::inv(xi), big, ipxi, 2);
    be.make_pow(F::inv(xiw), big, ipxiw, 3);
    {
        auto small = [](const std::vector<F>& v) { FfSmall<F> s; s.len = (int)v.size(); for (int i = 0; i < 8; i++) s.c[i] = i < s.len ? v[i] : F::zero(); return s; };
        FfSmall<F> none; none.len = 0; for (auto& c : none.c) c = F::zero();
        // F = (C0 - R0)/(X^8 - xi) + alpha (C1 - R1)/(X^4 - xi) + alpha^2 (C2 - R2)/((X^3 - xi)(X^3 - xi w))   (:1031-1056)
        be.zero(w.Fq, big); be.zero(w.F1, big); be.zero(w.F2, big);
        int flag = be.quot_m(k.c0, 8 * n, small(R0), F::one(), 8, n, pxi, ipxi, w.G, w.P, w.Fq);
        flag |= be.quot_m(w.C1, 8 * n, small(R1), alpha, 4, 2 * n, pxi, ipxi, w.G, w.P, w.F1);
        flag |= be.quot_m(w.C2, 9 * n, small(R2), F::sqr(alpha), 3, 3 * n, pxi, ipxi, w.G, w.P, w.scal);
        flag |= be.quot_m(w.scal, 9 * n, none, F::one(), 3, 3 * n, pxiw, ipxiw, w.G, w.P, w.F2);
        if (flag) { err = "Polynomial is not divisible"; return 4; }
        be.add3(9 * n, w.Fq, w.F1, w.F2, w.Fq);
        int rc = be.commit(w.Fq, 9 * n, pt_W1); if (rc) return rc;
    }
    be.mark(4);
    // ---------------- round 5 (:1059-1180)
    tr.reset(); tr.add_scalar(alpha); tr.add_point(pt_W1);
    const F y = tr.challenge();
    F mulL0 = F::one(), mulL1 = F::one(), mulL2 = F::one();
    for (const F& x : S0) mulL0 = F::mul(mulL0, F::sub(y, x));
    for (const F& x : S1) mulL1 = F::mul(mulL1, F::sub(y, x));
    for (const F& x : S2) mulL2 = F::mul(mulL2, F::sub(y, x));
    for (const F& x : S2p) mulL2 = F::mul(mulL2, F::sub(y, x));
    {
        FfLin<F> L;
        L.pre0 = F::mul(mulL1, mulL2);
        L.pre1 = F::mul(alpha, F::mul(mulL0, mulL2));
        L.pre2 = F::mul(F::sqr(alpha), F::mul(mulL0, mulL1));
        L.r0y = ffhost::horner(R0, y); L.r1y = ffhost::horner(R1, y); L.r2y = ffhost::horner(R2, y);
        L.zty = F::mul(mulL0, F::mul(mulL1, mulL2));                 // ZT(y): the zerofier of all 18 roots (:1164-1172)
        L.zts2y_inv = F::inv(F::mul(mulL1, mulL2));                  // 1 / ZTS2(y) (:1174-1180)
        PlonkPow<F> py, ipy;
        be.make_pow(y, big, py, 4);
        be.make_pow(F::inv(y), big, ipy, 5);
        int flag = be.quot_l(9 * n, k.c0, 8 * n, w.C1, 8 * n, w.C2, 9 * n, w.Fq, 9 * n, L, py, ipy, w.G, w.P, w.scal);
        if (flag) { err = "Degree of L(X)/(ZTS2(y)(X-y)) remainder should be 0"; return 4; }
        int rc = be.commit_plain(w.scal, 9 * n, pt_W2); if (rc) return rc;
    }
    be.mark(5);
    // ---------------- the batched inverse (:1182-1285)
    {
        F acc = F::mul(mulL1, mulL2);                                // denH1, denH2
        acc = F::mul(acc, F::sub(fr_pow2k(xi, k.power), F::one()));  // zh
        auto li = [&](const std::vector<F>& roots) {
            const size_t ln = roots.size();
            F den1 = fr_from_u64<F>(ln), p = F::one();
            for (size_t i = 0; i + 2 < ln; i++) p = F::mul(p, roots[0]);
            den1 = F::mul(den1, p);
            for (size_t i = 0; i < ln; i++) acc = F::mul(acc, F::mul(F::mul(den1, roots[((ln - 1) * i) % ln]), F::sub(y, roots[i])));
        };
        li(S0); li(S1);
        const F three = fr_from_u64<F>(3);
        F den1 = F::mul(F::mul(three, S2[0]), F::sub(xi, xiw));
        for (int i = 0; i < 3; i++) acc = F::mul(acc, F::mul(den1, F::mul(S2[2 * i % 3], F::sub(y, S2[i]))));
        den1 = F::mul(F::mul(three, S2p[0]), F::sub(xiw, xi));
        for (int i = 0; i < 3; i++) acc = F::mul(acc, F::mul(den1, F::mul(S2p[2 * i % 3], F::sub(y, S2p[i]))));
        const F nf = fr_from_u64<F>(n);
        F wq = F::one();
        const uint32_t nl = k.nPublic > 1 ? k.nPublic : 1;
        for (uint32_t i = 0; i < nl; i++) { acc = F::mul(acc, F::mul(nf, F::sub(xi, wq))); wq = F::mul(wq, k.wn); }
        ev[15] = F::inv(acc);
    }
    memcpy(ev_out, ev, sizeof ev);
    return 0;
}

}  // namespace sb
