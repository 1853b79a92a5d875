// verify_plonk.cuh — batched PLONK (src/plonk_verify.js:29-421) and fflonk (src/fflonk_verify.js:28-597) verification on the
// device pairing of pairing.cuh, templated on the base field (fflonk is instantiated for BN254 only).  Per call:
//   k_pv_prepare  thread 0 / 1: the Miller-loop lines of X_2 / of the G2 generator (the pairing target is 1, so nothing
//                 else is precomputed)
//   k_pv_scalars  one thread per proof: the reference's checks in its order (proof points on the curve, else status 3;
//                 evaluations below r as Montgomery bytes, else 4; public signals below r, else 2), the Keccak transcript,
//                 PI(xi) and every scalar the point sums need (plain, for gfft_mul)
//   k_pv_terms    one thread per (proof, term): s * P by gfft.cuh's per-thread scalar multiplication
//   k_pv_d4       PLONK only, one thread per proof: d4 = zh (T1 + xin T2 + xin^2 T3), nested as the reference nests it
//   k_pv_pair     one thread per proof: the pairing inputs summed from the terms, one two-pair Miller loop over the
//                 precomputed lines, one final exponentiation, compared with 1 (status 0, else 1)
// Every scalar multiplies the point the reference multiplies, by the reference's own scalar, and subtractions negate the
// point: on BLS12-381, where G1 has a cofactor and nothing checks subgroup membership, a proof point outside the
// r-subgroup gives the reference's point.  The per-proof code is __host__ __device__ so tests/host/plonk_verify_host.cpp
// runs it on the CPU.
#pragma once
#include <cstring>
#include "keccak.cuh"
#include "verify.cuh"

namespace sb {

template <class P> using FrF = Fp<typename FrOf<P>::T>;

// The verification key as the kernels read it, built on the host from the ABI's bytes (pv_key_host).
enum { PV_K1, PV_K2, PV_W, PV_W3, PV_W4, PV_W8, PV_WR, PV_WP };   // fr[]: PV_W = vk.w (fflonk), PV_WP = Fr.w[power]
template <class P> struct PvKey {
    Fp<P> pt[16];            // PLONK: Qm Ql Qr Qo Qc S1 S2 S3; fflonk: C0 in pt[0], pt[1]
    Fp<P> x2[4], g1[2], g2[4];
    FrF<P> fr[8];
    uint32_t n_public, power;
};

// plain <-> Montgomery scalars and small helpers
template <class P> SB_HD FrPlain fr_plain(const FrF<P>& a) { const FrF<P> p = FrF<P>::from_mont(a); FrPlain o; for (int i = 0; i < 8; i++) o.v[i] = p.v[i]; return o; }
template <class P> SB_HD FrF<P> fr_mont(const FrPlain& a) { FrF<P> p; for (int i = 0; i < 8; i++) p.v[i] = a.v[i]; return FrF<P>::to_mont(p); }
template <class R> SB_HD R fr_u32(uint32_t x) { R a = R::zero(); a.v[0] = x; return R::to_mont(a); }
template <class R> SB_HD R fr_div(const R& a, const R& b) { return R::mul(a, R::inv_binary(b)); }
template <class R> SB_HD R fr_powu(const R& a, int e) { R r = R::one(); for (int i = 0; i < e; i++) r = R::mul(r, a); return r; }

// Keccak256Transcript (src/Keccak256Transcript.js): points as G1.toRprUncompressed (x | y plain big-endian, infinity all
// zero), scalars as Fr.toRprBE, challenge = Fr.e(Scalar.fromRprBE(keccak_256(buffer))).  challenge() also resets.
template <class P> struct PvTranscript {
    typedef Fp<P> Q; typedef FrF<P> R;
    Keccak256 h;
    SB_HD PvTranscript() { h.reset(); }
    SB_HD void be(const uint32_t* v, int nw) { for (int i = 4 * nw - 1; i >= 0; i--) h.byte((uint8_t)(v[i >> 2] >> (8 * (i & 3)))); }
    SB_HD void point(const Q& x, const Q& y) { Q a = Q::from_mont(x); be(a.v, Q::N); a = Q::from_mont(y); be(a.v, Q::N); }
    SB_HD void scalar(const R& s) { const R a = R::from_mont(s); be(a.v, 8); }
    SB_HD void plain(const FrPlain& s) { be(s.v, 8); }
    SB_HD R challenge() {
        uint8_t d[32];
        h.finish(d); h.reset();
        FrPlain x;
        for (int i = 0; i < 8; i++) x.v[i] = (uint32_t)d[31 - 4 * i] | ((uint32_t)d[30 - 4 * i] << 8) | ((uint32_t)d[29 - 4 * i] << 16) | ((uint32_t)d[28 - 4 * i] << 24);
        while (!below_r<P>(x)) {   // r > 2^253: a few subtractions at most
            uint64_t borrow = 0;
            for (int i = 0; i < 8; i++) { const uint64_t t = (uint64_t)x.v[i] - FrOf<P>::T::p(i) - borrow; x.v[i] = (uint32_t)t; borrow = (t >> 32) & 1; }
        }
        return fr_mont<P>(x);
    }
};

// the reference's checks before the transcript: 3 (points), 4 (evaluations, as Montgomery bytes), 2 (public signals)
template <class P> SB_HD int pv_checks(const uint8_t* prf, int npts, int nchk, const FrPlain* pub, uint32_t n_public) {
    const Fp<P>* pt = (const Fp<P>*)prf;
    for (int i = 0; i < npts; i++) if (!Pairing<P>::g1_valid(pt[2 * i], pt[2 * i + 1])) return 3;
    const FrPlain* ev = (const FrPlain*)(prf + 2 * npts * sizeof(Fp<P>));
    for (int i = 0; i < nchk; i++) if (!below_r<P>(ev[i])) return 4;
    for (uint32_t i = 0; i < n_public; i++) if (!below_r<P>(pub[i])) return 2;
    return 0;
}

// L_1(xi) and PI(xi) = -sum s_i L_{i+1}(xi), L_i = w^(i-1) zh / (n (xi - w^(i-1))), n = 2^power.  PI is summed as one
// fraction, so the proof takes a single inversion however many public inputs it has.
template <class P> SB_HD void pv_pi(const FrF<P>& xi, const FrF<P>& zh, const FrF<P>& w, uint32_t power, const FrPlain* pub, uint32_t n_public,
                                    FrF<P>& l1, FrF<P>& pi) {
    typedef FrF<P> R;
    R nf = R::one();
    for (uint32_t i = 0; i < power; i++) nf = R::dbl(nf);
    const R den1 = R::mul(nf, R::sub(xi, R::one()));
    R num = R::zero(), den = R::one(), wq = R::one();
    for (uint32_t i = 0; i < n_public; i++) {
        const R a = R::mul(R::mul(wq, zh), fr_mont<P>(pub[i])), b = R::mul(nf, R::sub(xi, wq));
        num = R::sub(R::mul(num, b), R::mul(a, den));
        den = R::mul(den, b);
        wq = R::mul(wq, w);
    }
    const R inv = R::inv_binary(R::mul(den, den1));
    pi = R::mul(R::mul(num, den1), inv);
    l1 = R::mul(R::mul(zh, den), inv);
}

// ---------------------------------------------------------------------------------------------------------------- PLONK
// proof: A B C Z T1 T2 T3 Wxi Wxiw (affine Montgomery) || eval_a eval_b eval_c eval_s1 eval_s2 eval_zw (Montgomery)
// terms s[j] * base(j), j < 17; s[17] = zh:
//   0 Qm ea*eb  1 Ql ea  2 Qr eb  3 Qo ec  4 Z d2  5 S3 d3 (-)  6 A v1  7 B v2  8 C v3  9 S1 v4  10 S2 v5  11 G1 e (-)
//   12 Wxi xi  13 Wxiw u*xi*w  14 Wxiw u (into A1)  15 T2 xin  16 T3 xin^2 (into d4)
template <class R> struct PlonkVs { R beta, gamma, alpha, xi, v[6], u, xin, zh, l1, pi, r0; R s[18]; };

template <class P> SB_HD int plonk_vscalars(const PvKey<P>& vk, const uint8_t* prf, const FrPlain* pub, PlonkVs<FrF<P>>& o) {
    typedef FrF<P> R; typedef Fp<P> Q;
    const int st = pv_checks<P>(prf, 9, 6, pub, vk.n_public);
    if (st) return st;
    const Q* pt = (const Q*)prf;
    const R* ev = (const R*)(prf + 18 * sizeof(Q));
    PvTranscript<P> t;
    for (int i = 0; i < 8; i++) t.point(vk.pt[2 * i], vk.pt[2 * i + 1]);
    for (uint32_t i = 0; i < vk.n_public; i++) t.plain(pub[i]);
    for (int i = 0; i < 3; i++) t.point(pt[2 * i], pt[2 * i + 1]);
    o.beta = t.challenge();
    t.scalar(o.beta);
    o.gamma = t.challenge();
    t.scalar(o.beta); t.scalar(o.gamma); t.point(pt[6], pt[7]);
    o.alpha = t.challenge();
    t.scalar(o.alpha);
    for (int i = 4; i < 7; i++) t.point(pt[2 * i], pt[2 * i + 1]);
    o.xi = t.challenge();
    t.scalar(o.xi);
    for (int i = 0; i < 6; i++) t.scalar(ev[i]);
    o.v[0] = R::zero(); o.v[1] = t.challenge();
    for (int i = 2; i < 6; i++) o.v[i] = R::mul(o.v[i - 1], o.v[1]);
    t.point(pt[14], pt[15]); t.point(pt[16], pt[17]);
    o.u = t.challenge();
    o.xin = o.xi;
    for (uint32_t i = 0; i < vk.power; i++) o.xin = R::sqr(o.xin);
    o.zh = R::sub(o.xin, R::one());
    pv_pi<P>(o.xi, o.zh, vk.fr[PV_WP], vk.power, pub, vk.n_public, o.l1, o.pi);
    const R ea = ev[0], eb = ev[1], ec = ev[2], es1 = ev[3], es2 = ev[4], ezw = ev[5];
    const R alpha2 = R::sqr(o.alpha), l1a2 = R::mul(o.l1, alpha2);
    const R pa = R::add(R::add(ea, R::mul(o.beta, es1)), o.gamma), pb = R::add(R::add(eb, R::mul(o.beta, es2)), o.gamma);
    const R e3 = R::mul(R::mul(R::mul(R::mul(pa, pb), R::add(ec, o.gamma)), ezw), o.alpha);
    o.r0 = R::sub(R::sub(o.pi, l1a2), e3);
    const R betaxi = R::mul(o.beta, o.xi);
    R d2 = R::mul(R::add(R::add(ea, betaxi), o.gamma), R::add(R::add(eb, R::mul(betaxi, vk.fr[PV_K1])), o.gamma));
    d2 = R::mul(R::mul(d2, R::add(R::add(ec, R::mul(betaxi, vk.fr[PV_K2])), o.gamma)), o.alpha);
    d2 = R::add(R::add(d2, l1a2), o.u);
    const R d3 = R::mul(R::mul(pa, pb), R::mul(R::mul(o.alpha, o.beta), ezw));
    R e = R::neg(o.r0);
    for (int i = 1; i < 6; i++) e = R::add(e, R::mul(o.v[i], ev[i - 1]));
    e = R::add(e, R::mul(o.u, ezw));
    const R s13 = R::mul(R::mul(o.u, o.xi), vk.fr[PV_WP]);
    const R s[18] = {R::mul(ea, eb), ea, eb, ec, d2, d3, o.v[1], o.v[2], o.v[3], o.v[4], o.v[5], e, o.xi, s13, o.u, o.xin, R::sqr(o.xin), o.zh};
    for (int j = 0; j < 18; j++) o.s[j] = s[j];
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------- fflonk
// proof: C1 C2 W1 W2 (affine Montgomery) || ql qr qm qo qc s1 s2 s3 a b c z zw t1w t2w inv (Montgomery; inv is not read)
// terms: 0 C1 q1  1 C2 q2  2 G1 e (-)  3 W1 mulH0 (-)  4 W2 y
template <class R> struct FflonkVs { R beta, gamma, xi_seed, alpha, y, xi, xiw, zh, l1, pi, r0, r1, r2, q1, q2, mulH0, S0[8], S1[4], S2[3], S2p[3]; R s[5]; };

// computeLagrangeLiSi (fflonk_verify.js:545-561): the len Lagrange values at y of the roots of X^len = xi
template <class R> SB_HD R pv_li_si(const R* roots, int len, int i, const R& y, const R& xi) {
    const R num = R::sub(fr_powu(y, len), xi), den1 = R::mul(fr_u32<R>(len), fr_powu(roots[0], len - 2));
    return fr_div(num, R::mul(R::mul(den1, roots[((len - 1) * i) % len]), R::sub(y, roots[i])));
}

template <class P> SB_HD int fflonk_vscalars(const PvKey<P>& vk, const uint8_t* prf, const FrPlain* pub, FflonkVs<FrF<P>>& o) {
    typedef FrF<P> R; typedef Fp<P> Q;
    const int st = pv_checks<P>(prf, 4, 15, pub, vk.n_public);
    if (st) return st;
    const Q* pt = (const Q*)prf;
    const R* ev = (const R*)(prf + 8 * sizeof(Q));
    const R ql = ev[0], qr = ev[1], qm = ev[2], qo = ev[3], qc = ev[4], s1 = ev[5], s2 = ev[6], s3 = ev[7];
    const R a = ev[8], b = ev[9], c = ev[10], z = ev[11], zw = ev[12], t1w = ev[13], t2w = ev[14];
    PvTranscript<P> t;
    t.point(vk.pt[0], vk.pt[1]);
    for (uint32_t i = 0; i < vk.n_public; i++) t.plain(pub[i]);
    t.point(pt[0], pt[1]);
    o.beta = t.challenge();
    t.scalar(o.beta);
    o.gamma = t.challenge();
    t.scalar(o.gamma); t.point(pt[2], pt[3]);
    o.xi_seed = t.challenge();
    // roots (:225-277)
    const R seed2 = R::sqr(o.xi_seed), w3 = vk.fr[PV_W3], w3_2 = R::sqr(w3);
    o.S0[0] = R::mul(seed2, o.xi_seed);
    for (int i = 1; i < 8; i++) o.S0[i] = R::mul(o.S0[i - 1], vk.fr[PV_W8]);
    o.S1[0] = R::sqr(o.S0[0]);
    for (int i = 1; i < 4; i++) o.S1[i] = R::mul(o.S1[i - 1], vk.fr[PV_W4]);
    o.S2[0] = R::mul(o.S1[0], seed2); o.S2[1] = R::mul(o.S2[0], w3); o.S2[2] = R::mul(o.S2[0], w3_2);
    o.S2p[0] = R::mul(o.S2[0], vk.fr[PV_WR]); o.S2p[1] = R::mul(o.S2p[0], w3); o.S2p[2] = R::mul(o.S2p[0], w3_2);
    o.xi = R::mul(R::sqr(o.S2[0]), o.S2[0]);
    o.xiw = R::mul(o.xi, vk.fr[PV_WP]);
    R xin = o.xi;
    for (uint32_t i = 0; i < vk.power; i++) xin = R::sqr(xin);
    t.scalar(o.xi_seed);
    for (int i = 0; i < 15; i++) t.scalar(ev[i]);
    o.alpha = t.challenge();
    t.scalar(o.alpha); t.point(pt[4], pt[5]);
    o.y = t.challenge();
    o.zh = R::sub(xin, R::one());
    const R invzh = R::inv_binary(o.zh);
    pv_pi<P>(o.xi, o.zh, vk.fr[PV_W], vk.power, pub, vk.n_public, o.l1, o.pi);
    // r0 (:357-387)
    o.r0 = R::zero();
    for (int i = 0; i < 8; i++) {
        const R parts[8] = {ql, qr, qo, qm, qc, s1, s2, s3};
        R c0 = R::zero();
        for (int j = 7; j >= 0; j--) c0 = R::add(parts[j], R::mul(c0, o.S0[i]));
        o.r0 = R::add(o.r0, R::mul(c0, pv_li_si(o.S0, 8, i, o.y, o.xi)));
    }
    // r1 (:389-424)
    R t0 = R::add(R::add(R::mul(ql, a), R::mul(qr, b)), R::mul(qm, R::mul(a, b)));
    t0 = R::mul(R::add(R::add(R::add(t0, R::mul(qo, c)), qc), o.pi), invzh);
    o.r1 = R::zero();
    for (int i = 0; i < 4; i++) {
        const R h = o.S1[i], h2 = R::sqr(h);
        const R c1 = R::add(R::add(R::add(a, R::mul(h, b)), R::mul(h2, c)), R::mul(R::mul(h2, h), t0));
        o.r1 = R::add(o.r1, R::mul(c1, pv_li_si(o.S1, 4, i, o.y, o.xi)));
    }
    // r2 (:426-480)
    const R t1 = R::mul(R::mul(R::sub(z, R::one()), o.l1), invzh);
    const R betaxi = R::mul(o.beta, o.xi);
    const R t21 = R::mul(R::mul(R::add(a, R::add(betaxi, o.gamma)), R::add(b, R::add(R::mul(betaxi, vk.fr[PV_K1]), o.gamma))),
                         R::mul(R::add(c, R::add(R::mul(betaxi, vk.fr[PV_K2]), o.gamma)), z));
    const R t22 = R::mul(R::mul(R::add(a, R::add(R::mul(o.beta, s1), o.gamma)), R::add(b, R::add(R::mul(o.beta, s2), o.gamma))),
                         R::mul(R::add(c, R::add(R::mul(o.beta, s3), o.gamma)), zw));
    const R t2 = R::mul(R::sub(t21, t22), invzh);
    const R y3 = fr_powu(o.y, 3);
    const R num = R::add(R::sub(R::sqr(y3), R::mul(R::add(o.xi, o.xiw), y3)), R::mul(o.xi, o.xiw));
    o.r2 = R::zero();
    for (int half = 0; half < 2; half++) {
        const R* roots = half ? o.S2p : o.S2;
        const R den1 = R::mul(R::mul(fr_u32<R>(3), roots[0]), half ? R::sub(o.xiw, o.xi) : R::sub(o.xi, o.xiw));
        for (int i = 0; i < 3; i++) {
            const R h = roots[i];
            const R c2 = half ? R::add(R::add(zw, R::mul(h, t1w)), R::mul(R::sqr(h), t2w)) : R::add(R::add(z, R::mul(h, t1)), R::mul(R::sqr(h), t2));
            const R li = fr_div(num, R::mul(den1, R::mul(roots[(2 * i) % 3], R::sub(o.y, h))));
            o.r2 = R::add(o.r2, R::mul(c2, li));
        }
    }
    // F, E, J (:482-529)
    R mulH1 = R::one(), mulH2 = R::one();
    o.mulH0 = R::one();
    for (int i = 0; i < 8; i++) o.mulH0 = R::mul(o.mulH0, R::sub(o.y, o.S0[i]));
    for (int i = 0; i < 4; i++) mulH1 = R::mul(mulH1, R::sub(o.y, o.S1[i]));
    for (int i = 0; i < 3; i++) mulH2 = R::mul(R::mul(mulH2, R::sub(o.y, o.S2[i])), R::sub(o.y, o.S2p[i]));
    o.q1 = R::mul(o.alpha, fr_div(o.mulH0, mulH1));
    o.q2 = R::mul(R::sqr(o.alpha), fr_div(o.mulH0, mulH2));
    const R e = R::add(o.r0, R::add(R::mul(o.r1, o.q1), R::mul(o.r2, o.q2)));
    o.s[0] = o.q1; o.s[1] = o.q2; o.s[2] = e; o.s[3] = o.mulH0; o.s[4] = o.y;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------- protocols
// base(j): a key point index (< 16, pairs of pt[]), PV_PRF + a proof point index, or PV_GEN (the G1 generator)
enum { PV_PRF = 16, PV_GEN = 31 };
struct PvPlonk {
    static constexpr int NPTS = 9, NEV = 6, NT = 17, NS = 18;
    SB_CONSTEXPR_HD static constexpr int base(int j) {
        constexpr int v[NT] = {0, 1, 2, 3, PV_PRF + 3, 7, PV_PRF + 0, PV_PRF + 1, PV_PRF + 2, 5, 6, PV_GEN, PV_PRF + 7, PV_PRF + 8, PV_PRF + 8, PV_PRF + 5, PV_PRF + 6};
        return v[j];
    }
    template <class P> using Vs = PlonkVs<FrF<P>>;
    template <class P> SB_HD static int scalars(const PvKey<P>& k, const uint8_t* prf, const FrPlain* pub, Vs<P>& o) { return plonk_vscalars<P>(k, prf, pub, o); }
};
struct PvFflonk {
    static constexpr int NPTS = 4, NEV = 16, NT = 5, NS = 5;
    SB_CONSTEXPR_HD static constexpr int base(int j) { constexpr int v[NT] = {PV_PRF + 0, PV_PRF + 1, PV_GEN, PV_PRF + 2, PV_PRF + 3}; return v[j]; }
    template <class P> using Vs = FflonkVs<FrF<P>>;
    template <class P> SB_HD static int scalars(const PvKey<P>& k, const uint8_t* prf, const FrPlain* pub, Vs<P>& o) { return fflonk_vscalars<P>(k, prf, pub, o); }
};
template <class P, class V> SB_HD uint64_t pv_proof_bytes() { return 2 * V::NPTS * sizeof(Fp<P>) + 32 * V::NEV; }

template <class F> SB_HD XYZZ<F> pv_affine(const F& x, const F& y) {
    XYZZ<F> p = XYZZ<F>::inf();
    if (!(x.is_zero() && y.is_zero())) { p.x = x; p.y = y; p.zz = F::one(); p.zzz = F::one(); }
    return p;
}
template <class F> SB_HD XYZZ<F> pv_neg(XYZZ<F> p) { p.y = F::neg(p.y); return p; }

// d4 = zh (T1 + xin T2 + xin^2 T3) with t = the proof's terms: written over term 15, term 16 cleared.  mul(P, plain s) = s P.
template <class P, class M> SB_HD void plonk_d4(const uint8_t* prf, XYZZ<Fp<P>>* t, const FrPlain& zh, M mul) {
    const Fp<P>* pt = (const Fp<P>*)prf;
    XYZZ<Fp<P>> acc = pv_affine(pt[8], pt[9]);
    acc.add(t[15]); acc.add(t[16]);
    t[15] = mul(acc, zh);
    t[16] = XYZZ<Fp<P>>::inf();
}

// The pairing's G1 inputs from a proof's terms: p1 pairs with X_2, p2 with the G2 generator, and the proof verifies when
// e(p1, X_2) e(p2, G2) = 1.
//   PLONK  (:402-421):  p1 = -A1, A1 = Wxi + u Wxiw;   p2 = B1 = Qc + sum of terms 0..13 (5 and 11 negated) - d4
//   fflonk (:531-542):  p1 = W2;   p2 = -A1, A1 = C0 + q1 C1 + q2 C2 - e G1 - mulH0 W1 + y W2
template <class P, class V> SB_HD void pv_inputs(const PvKey<P>& vk, const uint8_t* prf, const XYZZ<Fp<P>>* t, XYZZ<Fp<P>>& p1, XYZZ<Fp<P>>& p2) {
    typedef Fp<P> F;
    const F* pt = (const F*)prf;
    if constexpr (V::NT == PvPlonk::NT) {
        XYZZ<F> a1 = pv_affine(pt[14], pt[15]);
        a1.add(t[14]);
        XYZZ<F> b1 = pv_affine(vk.pt[8], vk.pt[9]);
        for (int j = 0; j < 14; j++) b1.add(j == 5 || j == 11 ? pv_neg(t[j]) : t[j]);
        b1.add(pv_neg(t[15]));
        p1 = pv_neg(a1); p2 = b1;
    } else {
        XYZZ<F> a1 = pv_affine(vk.pt[0], vk.pt[1]);
        for (int j = 0; j < 5; j++) a1.add(j == 2 || j == 3 ? pv_neg(t[j]) : t[j]);
        p1 = pv_affine(pt[6], pt[7]); p2 = pv_neg(a1);
    }
}

// ---------------------------------------------------------------------------------------------------------------- kernels
#ifdef __CUDACC__
template <class P> __global__ void k_pv_prepare(const PvKey<P>* __restrict__ vk, PairLine<P>* __restrict__ lines) {
    typedef Pairing<P> T;
    typedef Fp2<P> F2;
    const Fp<P>* q = threadIdx.x ? vk->g2 : vk->x2;
    F2 x, y; x.a = q[0]; x.b = q[1]; y.a = q[2]; y.b = q[3];
    if (threadIdx.x < 2 && !(x.is_zero() && y.is_zero())) T::prepare(x, y, lines + threadIdx.x * T::NLINES);
}

template <class P, class V> __global__ void __launch_bounds__(VERIFY_THREADS)
k_pv_scalars(const PvKey<P>* __restrict__ vk, const FrPlain* __restrict__ pubs, const uint8_t* __restrict__ proofs, uint32_t count,
             FrPlain* __restrict__ sc, int32_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    typename V::template Vs<P> o;
    const int st = V::template scalars<P>(*vk, proofs + k * pv_proof_bytes<P, V>(), pubs + (uint64_t)k * vk->n_public, o);
    status[k] = st;
    if (st) return;
    for (int j = 0; j < V::NS; j++) sc[(uint64_t)k * V::NS + j] = fr_plain<P>(o.s[j]);
}

template <class P, class V> __global__ void __launch_bounds__(GFFT_THREADS)
k_pv_terms(const PvKey<P>* __restrict__ vk, const uint8_t* __restrict__ proofs, const FrPlain* __restrict__ sc, const int32_t* __restrict__ status,
           uint64_t n, XYZZ<Fp<P>>* __restrict__ terms) {
    typedef Fp<P> F;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint64_t k = t / V::NT;
    const int j = (int)(t % V::NT);
    if (status[k]) return;
    const int b = V::base(j);
    const uint8_t* src = b == PV_GEN ? (const uint8_t*)vk->g1 : b >= PV_PRF ? proofs + k * pv_proof_bytes<P, V>() + (b - PV_PRF) * 2 * sizeof(F)
                                                                            : (const uint8_t*)(vk->pt + 2 * b);
    terms[t] = gfft_mul<F>(gfft_get<F>(src, 0, 0), sc[k * V::NS + j]);
}

template <class P> __global__ void __launch_bounds__(GFFT_THREADS)
k_pv_d4(const uint8_t* __restrict__ proofs, const FrPlain* __restrict__ sc, const int32_t* __restrict__ status, uint32_t count, XYZZ<Fp<P>>* __restrict__ terms) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count || status[k]) return;
    plonk_d4<P>(proofs + k * pv_proof_bytes<P, PvPlonk>(), terms + (uint64_t)k * PvPlonk::NT, sc[(uint64_t)k * PvPlonk::NS + 17],
                [](const XYZZ<Fp<P>>& p, const FrPlain& s) { return gfft_mul<Fp<P>>(p, s); });
}

template <class P, class V> __global__ void __launch_bounds__(VERIFY_THREADS)
k_pv_pair(const PvKey<P>* __restrict__ vk, const PairLine<P>* __restrict__ lines, const uint8_t* __restrict__ proofs,
          const XYZZ<Fp<P>>* __restrict__ terms, uint32_t count, int32_t* __restrict__ status) {
    typedef Pairing<P> T;
    typedef Fp<P> F;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count || status[k]) return;
    XYZZ<F> p[2];
    pv_inputs<P, V>(*vk, proofs + k * pv_proof_bytes<P, V>(), terms + (uint64_t)k * V::NT, p[0], p[1]);
    F x[2], y[2];
    for (int i = 0; i < 2; i++) {
        x[i] = F::zero(); y[i] = F::zero();
        if (!p[i].is_inf()) {
            const F s = F::inv_binary(p[i].zzz), u = F::mul(p[i].zz, s);
            x[i] = F::mul(p[i].x, F::sqr(u)); y[i] = F::mul(p[i].y, s);
        }
    }
    Fp2<P> qx, qy; qx.a = vk->x2[0]; qx.b = vk->x2[1]; qy.a = vk->x2[2]; qy.b = vk->x2[3];
    const bool live1 = !p[0].is_inf() && !(qx.is_zero() && qy.is_zero()), live2 = !p[1].is_inf();
    const typename T::F12 f = T::miller(x[0], y[0], qx, qy, false, x[0], y[0], lines, live1, x[1], y[1], lines + T::NLINES, live2);
    status[k] = T::eq(T::final_exp(f), T::one()) ? 0 : 1;
}

#endif  // __CUDACC__

// host: the kernels' key from the ABI's bytes (include/snarkb200.h) and the context's generators and Fr.w[power] (all
// Montgomery); false when a key point is off its curve or has a coordinate >= q
template <class P, class V> bool pv_key_host(const uint8_t* vk, uint32_t n_public, uint32_t power, const uint8_t* gen1, const uint8_t* gen2,
                                             const uint8_t* wpow, PvKey<P>& k) {
    typedef Fp<P> F;
    typedef Pairing<P> T;
    memset(&k, 0, sizeof k);
    const int npts = V::NT == PvPlonk::NT ? 8 : 1, nfr = V::NT == PvPlonk::NT ? 2 : 7;
    memcpy(k.pt, vk, 2 * npts * sizeof(F));
    memcpy(k.x2, vk + 2 * npts * sizeof(F), 4 * sizeof(F));
    const uint8_t* fr = vk + (2 * npts + 4) * sizeof(F);
    if (V::NT == PvPlonk::NT) { memcpy(&k.fr[PV_K1], fr, 32); memcpy(&k.fr[PV_K2], fr + 32, 32); }
    else memcpy(&k.fr[PV_K1], fr, 32 * nfr);
    memcpy(&k.fr[PV_WP], wpow, 32);
    memcpy(k.g1, gen1, sizeof k.g1); memcpy(k.g2, gen2, sizeof k.g2);
    k.n_public = n_public; k.power = power;
    bool ok = true;
    for (int i = 0; i < npts; i++) ok = ok && T::g1_valid(k.pt[2 * i], k.pt[2 * i + 1]);
    Fp2<P> x, y; x.a = k.x2[0]; x.b = k.x2[1]; y.a = k.x2[2]; y.b = k.x2[3];
    return ok && T::g2_valid(x, y);
}

}  // namespace sb
