// fflonk.cuh — the per-element work of snarkjs' fflonk prover (src/fflonk_prove.js) between its NTTs and MSMs, in the
// style of plonk.cuh: every loop body of the reference is an SB_HD function of the element index (one CUDA thread per
// index on the device, a plain loop in tests/host/host_fflonk.cpp), and its recurrences become scans:
//
//   f / (X^m - b)   (Polynomial.divByZerofier, polynomial.js:617-660) — with f(X) = sum_j X^j f_j(X^m) this is m independent
//                   divisions f_j(Y) / (Y - b) on the stride-m subsequences: g = f[k] b^(k div m) stored class-major,
//                   a segmented inclusive sum scan P, q[k] = (P_last(class) - P[k]) b^-(k div m + 1); the class totals
//                   are the remainder and must vanish.
//   f / (X - y)     (Polynomial.divBy, :341-360) — the m = 1 case, shared with plonk.cuh (pl_quot_coef).
#pragma once
#include "plonk.cuh"

namespace sb {

// ---------------------------------------------------------------------------------------------- round 1
// computeT0 (fflonk_prove.js:415-504): T0 * Z_H on the 4n domain.  PlonkTIn carries A B C QM QL QR QO QC LAG pubA n_public.
template <class F> SB_HD void ff_t0(uint64_t i, uint64_t n4, const PlonkTIn& in, F* T0) {
    const F a = pl_ld((const F*)in.A + i), b = pl_ld((const F*)in.B + i), c = pl_ld((const F*)in.C + i);
    F pi = F::zero();
    for (uint32_t j = 0; j < in.n_public; j++)
        pi = F::sub(pi, F::mul(pl_ld((const F*)in.LAG + (uint64_t)j * n4 + i), pl_ld((const F*)in.pubA + j)));
    F t = F::mul(a, pl_ld((const F*)in.QL + i));
    t = F::add(t, F::mul(b, pl_ld((const F*)in.QR + i)));
    t = F::add(t, F::mul(F::mul(a, b), pl_ld((const F*)in.QM + i)));
    t = F::add(t, F::mul(c, pl_ld((const F*)in.QO + i)));
    t = F::add(t, F::add(pl_ld((const F*)in.QC + i), pi));
    pl_st(T0 + i, t);
}
// wire blinding (:375-380): the reference writes the blinders' Montgomery bytes into the *plain* evaluation buffer before
// batchToMontgomery, so the evaluation is toMontgomery(raw bytes)
template <class F> SB_HD void ff_wire_blind(F* buf, uint64_t n, const F& b_lo_raw, const F& b_hi_raw) {
    pl_st(buf + n - 2, F::to_mont(b_lo_raw));
    pl_st(buf + n - 1, F::to_mont(b_hi_raw));
}

// ---------------------------------------------------------------------------------------------- round 2
// computeT1 (:667-718) on the 2n domain: (z - 1) L1 and its blinding part.  evZ and lag1 are 4n-point arrays (stride 2).
template <class F> SB_HD void ff_t1(uint64_t i, const F* evZ, const F* lag1, const PlonkPow<F>& w2pow, const PlonkRound<F>& r, F* T1, F* T1z) {
    const F om = pl_pow(w2pow, i);
    const F zp = F::add(F::mul(F::add(F::mul(r.b[7], om), r.b[8]), om), r.b[9]);
    const F l1 = pl_ld(lag1 + 2 * i);
    pl_st(T1 + i, F::mul(F::sub(pl_ld(evZ + 2 * i), F::one()), l1));
    pl_st(T1z + i, F::mul(zp, l1));
}
// computeT2 (:720-815) on the 4n domain.  PlonkTIn carries A B C Z S1 S2 S3.
template <class F> SB_HD void ff_t2(uint64_t i, uint64_t n4, const PlonkTIn& in, const PlonkPow<F>& w4pow, const PlonkRound<F>& r, F* T2, F* T2z) {
    const F a = pl_ld((const F*)in.A + i), b = pl_ld((const F*)in.B + i), c = pl_ld((const F*)in.C + i);
    const F z = pl_ld((const F*)in.Z + i), zw = pl_ld((const F*)in.Z + ((i + 4) & (n4 - 1)));
    const F om = pl_pow(w4pow, i), omW = F::mul(om, r.wn);
    const F zp = F::add(F::mul(F::add(F::mul(r.b[7], om), r.b[8]), om), r.b[9]);
    const F zWp = F::add(F::mul(F::add(F::mul(r.b[7], omW), r.b[8]), omW), r.b[9]);
    const F betaX = F::mul(r.beta, om);
    F e1 = F::mul(F::add(F::add(a, betaX), r.gamma), F::add(F::add(b, F::mul(betaX, r.k1)), r.gamma));
    e1 = F::mul(e1, F::add(F::add(c, F::mul(betaX, r.k2)), r.gamma));
    F e2 = F::mul(F::add(F::add(a, F::mul(r.beta, pl_ld((const F*)in.S1 + i))), r.gamma), F::add(F::add(b, F::mul(r.beta, pl_ld((const F*)in.S2 + i))), r.gamma));
    e2 = F::mul(e2, F::add(F::add(c, F::mul(r.beta, pl_ld((const F*)in.S3 + i))), r.gamma));
    pl_st(T2 + i, F::sub(F::mul(e1, z), F::mul(e2, zw)));
    pl_st(T2z + i, F::sub(F::mul(e1, zp), F::mul(e2, zWp)));
}
// divByZerofier(n, 1) (polynomial.js:617-660) on a polynomial of `blocks` * n coefficients, then add the blinding part tz
// (may be null) and check the degree bound: coefficients at index >= bound must be zero afterwards.
// Thread i < n owns coefficients i, n+i, 2n+i, ...  Returns 1 ("Polynomial is not divisible") or 2 (degree) or 0.
template <class F> SB_HD int ff_divzh(uint64_t i, uint64_t n, int blocks, const F* t, const F* tz, F* out, uint64_t bound) {
    int bad = 0;
    F c = F::neg(pl_ld(t + i));
    for (int k = 0; k < blocks; k++) {
        if (k) c = F::sub(c, pl_ld(t + (uint64_t)k * n + i));
        if (k == blocks - 1 && !c.is_zero()) bad = 1;                 // the top n coefficients must vanish
        F o = tz ? F::add(c, pl_ld(tz + (uint64_t)k * n + i)) : c;
        if ((uint64_t)k * n + i >= bound && !o.is_zero() && !bad) bad = 2;
        pl_st(out + (uint64_t)k * n + i, o);
    }
    return bad;
}
// CPolynomial.getPolynomial (cpolynomial.js:52-72): out[i m + j] = p_j[i]
struct FfParts { const void* p[4]; uint64_t len[4]; int m; };
template <class F> SB_HD void ff_interleave(uint64_t k, const FfParts& parts, F* out) {
    const uint64_t j = k % parts.m, i = k / parts.m;
    pl_st(out + k, i < parts.len[j] ? pl_ld((const F*)parts.p[j] + i) : F::zero());
}

// ---------------------------------------------------------------------------------------------- round 4
template <class F> struct FfSmall { F c[8]; int len; };               // R0 / R1 / R2: at most 8 coefficients
// per proof and division of a batch: the interpolant to subtract and the scale (1, alpha, alpha^2, 1)
template <class F> struct FfQuot { FfSmall<F> R; F scale; };
// numerator coefficient k of (f - R) * scale, times b^(k div m), stored class-major: G[(k mod m) rows + k div m]
template <class F> SB_HD void ff_qm_g(uint64_t k, const F* f, uint64_t len, const FfSmall<F>& R, const F& scale, int m, uint64_t rows,
                                      const PlonkPow<F>& bpow, F* G) {
    F x = k < len ? pl_ld(f + k) : F::zero();
    if (k < (uint64_t)R.len) x = F::sub(x, R.c[k]);
    x = F::mul(x, scale);
    const uint64_t j = k % m, t = k / m;
    pl_st(G + j * rows + t, F::mul(x, pl_pow(bpow, t)));
}
// quotient coefficient k from the segmented inclusive sums P (class-major); the top row is zero.
// Returns nonzero when class k mod m leaves a remainder (checked once per class, by the thread of its first element).
template <class F> SB_HD int ff_qm_q(uint64_t k, int m, uint64_t rows, const F* P, const PlonkPow<F>& ibpow, F* q) {
    const uint64_t j = k % m, t = k / m;
    const F total = pl_ld(P + j * rows + rows - 1);
    int bad = (t == 0 && !total.is_zero()) ? 1 : 0;
    pl_st(q + k, t + 1 >= rows ? F::zero() : F::mul(F::sub(total, pl_ld(P + j * rows + t)), pl_pow(ibpow, t + 1)));
    return bad;
}

// ---------------------------------------------------------------------------------------------- round 5
template <class F> struct FfLin { F pre0, pre1, pre2, r0y, r1y, r2y, zty, zts2y_inv; };
// computeL (:1101-1162) then mulScalar(1 / ZTS2(y)) (:1077-1079): coefficient k of
//   [preL0 (C0 - R0(y)) + preL1 (C1 - R1(y)) + preL2 (C2 - R2(y)) - ZT(y) F] / ZTS2(y)
template <class F> SB_HD F ff_l_coef(uint64_t k, const F* C0, uint64_t l0, const F* C1, uint64_t l1, const F* C2, uint64_t l2, const F* Fp, uint64_t lf,
                                     const FfLin<F>& L) {
    F c0 = pl_at<F>(C0, k, l0), c1 = pl_at<F>(C1, k, l1), c2 = pl_at<F>(C2, k, l2);
    if (k == 0) { c0 = F::sub(c0, L.r0y); c1 = F::sub(c1, L.r1y); c2 = F::sub(c2, L.r2y); }
    F x = F::mul(c0, L.pre0);
    x = F::add(x, F::mul(c1, L.pre1));
    x = F::add(x, F::mul(c2, L.pre2));
    x = F::sub(x, F::mul(pl_at<F>(Fp, k, lf), L.zty));
    return F::mul(x, L.zts2y_inv);
}

// ---------------------------------------------------------------------------------------------- batches
// Round 3 of a batch evaluates 18 polynomials per proof (26 when C0 is not the interleave of its parts): segment e of
// proof q is polynomial f_e (len_e coefficients) at power table pw_e (0 = xi, 1 = xi w, 2 + i = S0[i]).  Segments
// 0-14 are the proof's 15 opening values, 15-17 T0, T1, T2 at xi, 18 + i C0 at S0[i].
struct FfEvalIn {
    const void* key[9];                      // ql qr qm qo qc s1 s2 s3 (n coefficients each), C0 (8n)
    const void *pABC, *cZ, *pT0, *pT1, *pT2;  // batch rows: 3K x n (group-major), K x nz, K x 4n, K x 2n, K x 4n
    uint64_t n, K, nz;
};
template <class F> SB_HD const F* ff_eval_seg(const FfEvalIn& in, uint64_t q, int e, uint64_t& len, int& pw) {
    const uint64_t n = in.n;
    len = n; pw = 0;
    if (e < 8) return (const F*)in.key[e];
    if (e < 11) return (const F*)in.pABC + ((e - 8) * in.K + q) * n;
    switch (e) {
    case 11: len = n + 3; return (const F*)in.cZ + q * in.nz;
    case 12: len = n + 3; pw = 1; return (const F*)in.cZ + q * in.nz;
    case 13: len = 2 * n; pw = 1; return (const F*)in.pT1 + q * 2 * n;
    case 14: len = 4 * n; pw = 1; return (const F*)in.pT2 + q * 4 * n;
    case 15: len = 2 * n; return (const F*)in.pT0 + q * 4 * n;
    case 16: len = 2 * n; return (const F*)in.pT1 + q * 2 * n;
    case 17: len = 4 * n; return (const F*)in.pT2 + q * 4 * n;
    default: len = 8 * n; pw = 2 + (e - 18); return (const F*)in.key[8];
    }
}
// offset of segment e in a proof's terms (segment e's offset + its length = segment e + 1's)
SB_HD uint64_t ff_eval_off(uint64_t n, int e) {
    if (e <= 11) return e * n;
    if (e == 12) return 12 * n + 3;
    if (e == 13) return 13 * n + 6;
    const uint64_t at[5] = {15, 19, 21, 23, 27};   // e = 14..18: n multiples (+ 6)
    if (e <= 18) return at[e - 14] * n + 6;
    return 27 * n + 6 + 8 * n * (e - 18);
}

#ifdef __CUDACC__
template <class F> __global__ void __launch_bounds__(128) k_ff_t0(uint64_t n4, PlonkTIn in, F* T0) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n4) ff_t0<F>(i, n4, in, T0);
}
template <class F> struct FfBlind6 { F raw[6]; };
template <class F> __global__ void k_ff_wire_blind(F* A, F* B, F* C, uint64_t n, FfBlind6<F> b) {
    if (blockIdx.x == 0 && threadIdx.x < 3) { F* bufs[3] = {A, B, C}; ff_wire_blind<F>(bufs[threadIdx.x], n, b.raw[2 * threadIdx.x], b.raw[2 * threadIdx.x + 1]); }
}
template <class F> __global__ void k_ff_t1(uint64_t n2, const F* evZ, const F* lag1, PlonkPow<F> w2pow, PlonkRound<F> r, F* T1, F* T1z) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n2) ff_t1<F>(i, evZ, lag1, w2pow, r, T1, T1z);
}
template <class F> __global__ void __launch_bounds__(128) k_ff_t2(uint64_t n4, PlonkTIn in, PlonkPow<F> w4pow, PlonkRound<F> r, F* T2, F* T2z) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n4) ff_t2<F>(i, n4, in, w4pow, r, T2, T2z);
}
template <class F> __global__ void k_ff_divzh(uint64_t n, int blocks, const F* t, const F* tz, F* out, uint64_t bound, int* flag) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) { int bad = ff_divzh<F>(i, n, blocks, t, tz, out, bound); if (bad) atomicOr(flag, bad); }
}
template <class F> __global__ void k_ff_interleave(uint64_t total, FfParts parts, F* out) {
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total) ff_interleave<F>(k, parts, out);
}
template <class F> struct FfOne { F x; };
template <class F> __global__ void k_ff_qm_g(uint64_t total, const F* f, uint64_t len, FfSmall<F> R, FfOne<F> scale, int m, uint64_t rows, PlonkPow<F> bpow, F* G) {
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total) ff_qm_g<F>(k, f, len, R, scale.x, m, rows, bpow, G);
}
template <class F> __global__ void k_ff_qm_q(uint64_t total, int m, uint64_t rows, const F* P, PlonkPow<F> ibpow, F* q, int* flag) {
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total && ff_qm_q<F>(k, m, rows, P, ibpow, q)) atomicOr(flag, 1);
}
template <class F> __global__ void k_ff_add3(uint64_t total, const F* a, const F* b, const F* c, F* out) {
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total) pl_st(out + k, F::add(F::add(pl_ld(a + k), pl_ld(b + k)), pl_ld(c + k)));
}
template <class F> __global__ void k_ff_l(uint64_t total, const F* C0, uint64_t l0, const F* C1, uint64_t l1, const F* C2, uint64_t l2, const F* Fp, uint64_t lf,
                                          FfLin<F> L, PlonkPow<F> ypow, F* g) {
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total) pl_st(g + k, F::mul(ff_l_coef<F>(k, C0, l0, C1, l1, C2, l2, Fp, lf, L), pl_pow(ypow, k)));
}

// ------------------------------------------------------------------------------------------------ batched kernels
// The kernels above with the proof on blockIdx.y, as plonk.cuh's k_plb_*: work arrays hold the K proofs back to back at a
// fixed stride, per-proof scalars (PlonkRound, FfQuot, FfLin, power tables) come from small device arrays, and a block
// stages its proof's scalars in shared memory where every element reads them.
// wires: 3K rows of n (A rows, then B, then C); thread j < 3K blinds row j with b[2 (j / K) + 1], b[2 (j / K) + 2]
template <class F> __global__ void k_ffb_wire_blind(F* wires, uint64_t n, uint32_t K, const PlonkRound<F>* rs) {
    uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= 3 * K) return;
    const uint32_t j = row / K, q = row % K;
    ff_wire_blind<F>(wires + row * n, n, pl_ld(&rs[q].b[2 * j + 1]), pl_ld(&rs[q].b[2 * j + 2]));
}
// ev: 3K rows of 4n (A, B, C evaluations); wires: A's rows give the public inputs; T: K rows of 4n
template <class F> __global__ void __launch_bounds__(128) k_ffb_t0(uint64_t n4, uint64_t n, PlonkTIn in, const F* ev, const F* wires, F* T) {
    const uint64_t q = blockIdx.y, K = gridDim.y;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n4) return;
    in.A = ev + q * n4; in.B = ev + (K + q) * n4; in.C = ev + (2 * K + q) * n4; in.pubA = wires + q * n;
    ff_t0<F>(i, n4, in, T + q * n4);
}
// evZ: K rows of 4n; T: K rows of 2n (T1), then K rows of 2n (T1z)
template <class F> __global__ void __launch_bounds__(128) k_ffb_t1(uint64_t n2, const F* evZ, const F* lag1, PlonkPow<F> w2pow, const PlonkRound<F>* rs, F* T) {
    __shared__ __align__(16) uint32_t sh[sizeof(PlonkRound<F>) / 4];
    const uint64_t q = blockIdx.y, K = gridDim.y;
    const PlonkRound<F>& r = pl_stage(sh, rs + q);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n2) ff_t1<F>(i, evZ + q * 2 * n2, lag1, w2pow, r, T + q * n2, T + (K + q) * n2);
}
// ev: 3K rows of 4n, evZ: K rows of 4n; T: K rows of 4n (T2), then K rows of 4n (T2z)
template <class F> __global__ void __launch_bounds__(128) k_ffb_t2(uint64_t n4, PlonkTIn in, const F* ev, const F* evZ, PlonkPow<F> w4pow,
                                                                   const PlonkRound<F>* rs, F* T) {
    __shared__ __align__(16) uint32_t sh[sizeof(PlonkRound<F>) / 4];
    const uint64_t q = blockIdx.y, K = gridDim.y;
    const PlonkRound<F>& r = pl_stage(sh, rs + q);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n4) return;
    in.A = ev + q * n4; in.B = ev + (K + q) * n4; in.C = ev + (2 * K + q) * n4; in.Z = evZ + q * n4;
    ff_t2<F>(i, n4, in, w4pow, r, T + q * n4, T + (K + q) * n4);
}
// t: K rows of blocks x n (then K rows of its blinding part when tz); out row q at q * ostride; flag[q] |= code << shift
template <class F> __global__ void k_ffb_divzh(uint64_t n, int blocks, const F* t, int tz, F* out, uint64_t ostride, uint64_t bound, int shift, int* flag) {
    const uint64_t q = blockIdx.y, K = gridDim.y, len = (uint64_t)blocks * n;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int bad = ff_divzh<F>(i, n, blocks, t + q * len, tz ? t + (K + q) * len : nullptr, out + q * ostride, bound);
    if (bad) atomicOr(flag + q, bad << shift);
}
// part j of proof q at parts.p[j] + q * strides[j]; out: K rows of `total`
struct FfStrides { uint64_t s[4]; };
template <class F> __global__ void k_ffb_interleave(uint64_t total, FfParts parts, FfStrides st, F* out) {
    const uint64_t q = blockIdx.y;
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k >= total) return;
    for (int j = 0; j < parts.m; j++) parts.p[j] = (const F*)parts.p[j] + q * st.s[j];
    ff_interleave<F>(k, parts, out + q * total);
}
// round 3's terms: row e + segs q of the grid (segment e of proof q, ff_eval_seg) -> g[q * T + ff_eval_off(e) + i] = f_e[i] x^i
template <class F> struct FfEvalPows { PlonkPowK<F> p[10]; };
template <class F> __global__ void k_ffb_eval_terms(FfEvalIn in, int segs, uint64_t T, FfEvalPows<F> pw, F* g) {
    const uint64_t row = blockIdx.y, q = row / segs; const int e = (int)(row % segs);
    uint64_t len; int p;
    const F* f = ff_eval_seg<F>(in, q, e, len, p);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < len) pl_st(g + q * T + ff_eval_off(in.n, e) + i, F::mul(pl_ld(f + i), pl_pow(pw.p[p].at(q), i)));
}
// numerator terms of one division of every proof (ff_qm_g): f row q at f + q * fs, G: K blocks of rows * m (class-major)
template <class F> __global__ void k_ffb_qm_g(uint64_t total, const F* f, uint64_t fs, uint64_t len, const FfQuot<F>* qt, int m, uint64_t rows,
                                              PlonkPowK<F> bpow, F* G) {
    __shared__ __align__(16) uint32_t sh[sizeof(FfQuot<F>) / 4];
    const uint64_t q = blockIdx.y;
    const FfQuot<F>& d = pl_stage(sh, qt + q);
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < total) ff_qm_g<F>(k, f + q * fs, len, d.R, d.scale, m, rows, bpow.at(q), G + q * total);
}
// quotients from the keyed sums (ff_qm_q): out row q at out + q * ostride, zero from rows * m to ostride; flag[q] |= 1 on a remainder
template <class F> __global__ void k_ffb_qm_q(uint64_t total, uint64_t ostride, int m, uint64_t rows, const F* P, PlonkPowK<F> ibpow, F* out, int* flag) {
    const uint64_t q = blockIdx.y;
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k >= ostride) return;
    if (k >= total) { pl_st(out + q * ostride + k, F::zero()); return; }
    if (ff_qm_q<F>(k, m, rows, P + q * total, ibpow.at(q), out + q * ostride)) atomicOr(flag + q, 1);
}
// round 5's numerator of every proof (ff_l_coef times y^k): C1, C2, Fp, g: K rows of m
template <class F> __global__ void __launch_bounds__(128) k_ffb_l(uint64_t m, const F* C0, uint64_t l0, const F* C1, uint64_t l1, const F* C2,
                                                                  const F* Fp, const FfLin<F>* Ls, PlonkPowK<F> ypow, F* g) {
    __shared__ __align__(16) uint32_t sh[sizeof(FfLin<F>) / 4];
    const uint64_t q = blockIdx.y;
    const FfLin<F>& L = pl_stage(sh, Ls + q);
    uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (k < m) pl_st(g + q * m + k, F::mul(ff_l_coef<F>(k, C0, l0, C1 + q * m, l1, C2 + q * m, m, Fp + q * m, m, L), pl_pow(ypow.at(q), k)));
}
// f / (X - y) of every proof from the keyed sums P (K rows of m): plain scalars; flag[q] |= 1 when the remainder is not zero
template <class F> __global__ void k_ffb_quot(uint64_t m, const F* P, PlonkPowK<F> ipow, F* q_plain, int* flag) {
    const uint64_t q = blockIdx.y;
    uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const F* Pr = P + q * m;
    if (j == 0 && !pl_ld(Pr + m - 1).is_zero()) atomicOr(flag + q, 1);
    pl_st(q_plain + q * m + j, F::from_mont(pl_quot_coef<F>(j, m, Pr, ipow.at(q))));
}
#endif  // __CUDACC__

}  // namespace sb
