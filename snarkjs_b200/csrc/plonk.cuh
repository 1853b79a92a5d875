// plonk.cuh — the per-element work of snarkjs' PLONK prover (src/plonk_prove.js) between its NTTs and MSMs.
//
// The reference runs these as JavaScript loops over BigBuffers, one field operation per WASM call
// (computeZ :376-458, computeT :486-684, divZh polynomial.js:592-614, computeR :752-856, computeWxi/Wxiw :858-888,
// Polynomial.evaluate polynomial.js:174-184, divByZerofier :617-660).  Here every loop body is a function of the
// element index, so a kernel is just "one thread per index"; the two recurrences become scans:
//
//   z[i+1] = z[i] * num[i] / den[i]                 -> batch inversion + exclusive product scan
//   q = f / (X - b):  q[j] = sum_{k>j} f[k] b^(k-j-1)  -> g[k] = f[k] b^k, inclusive sum scan P, q[j] = (P[last] - P[j]) b^-(j+1)
//                                                      (P[last] = f(b) is the remainder: must be 0)
//   f(x) = sum f[k] x^k                             -> the same products, reduced
//
// All element functions are SB_HD (host + device): tests/host/host_plonk.cpp compiles them with g++ and
// tests/test_host_plonk.py checks them against the CPU oracle without a GPU.  Field elements are canonical
// Montgomery everywhere except the witness (plain, as in the wtns file).
#pragma once
#include "fp.cuh"

namespace sb {

// base^i = lo[i mod 2^h] * hi[i >> h]
template <class F> struct PlonkPow { const F* lo = nullptr; const F* hi = nullptr; int h = 0; };

template <class F> struct PlonkRound {         // challenges and constants of rounds 2-3
    F beta, gamma, alpha, alpha2, k1, k2, wn;  // wn = Fr.w[power]
    F b[12];                                   // blinders b[1..11] (b[0] unused)
    F z1[4], z2[4], z3[4];                     // MulZ tables (src/mul_z.js:21-47)
};

template <class F> struct PlonkLin {           // scalars of round 5 (computeR / computeWxi)
    F coef_ab, ea, eb, ec, e24, e3beta, zh, xin, xin2, r0, v[6], wsub;
};

template <class F> SB_HD F pl_ld(const F* p) {
#ifdef __CUDA_ARCH__
    F x; const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
    return x;
#else
    return *p;
#endif
}
template <class F> SB_HD void pl_st(F* p, const F& x) {
#ifdef __CUDA_ARCH__
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
    q[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
#else
    *p = x;
#endif
}
template <class F> SB_HD F pl_pow(const PlonkPow<F>& t, uint64_t i) {
    return F::mul(pl_ld(t.lo + (i & ((1ull << t.h) - 1))), pl_ld(t.hi + (i >> t.h)));
}
// one power table per proof of a batch: proof q's tables start at lo + q * slo and hi + q * shi
template <class F> struct PlonkPowK {
    const F* lo = nullptr; const F* hi = nullptr; int h = 0; uint64_t slo = 0, shi = 0;
    SB_HD PlonkPow<F> at(uint64_t q) const { PlonkPow<F> p; p.lo = lo + q * slo; p.hi = hi + q * shi; p.h = h; return p; }
};
// which blinders b[idx[j][0..cnt)] go onto the rows of group j (a batch blinds groups x K rows, group-major)
struct PlonkBlindIdx { int cnt; int idx[3][3]; };

// ---------------------------------------------------------------------------------------------- round 1
// calculateAdditions (plonk_prove.js:166-195): w[n_wit + i] = f1 * w[s1] + f2 * w[s2].  Factors are Montgomery, the witness
// plain, so the Montgomery product is the plain value.  sig = (s1, s2) pairs, fac = (f1, f2) pairs, original order.
template <class F> SB_HD void pl_addition(uint32_t i, const uint32_t* sig, const F* fac, F* w, uint32_t n_wit, uint32_t n_vars) {
    uint32_t s1 = sig[2 * i], s2 = sig[2 * i + 1];
    // getWitness :203-211.  An addition that names itself or a later addition reads the reference's still-zero
    // internalWitness slot (:178-180 allocate it zeroed); here that slot may be written concurrently, so it is forced to 0.
    F a = (s1 < n_vars && (s1 < n_wit || s1 - n_wit < i)) ? pl_ld(w + s1) : F::zero();
    F b = (s2 < n_vars && (s2 < n_wit || s2 - n_wit < i)) ? pl_ld(w + s2) : F::zero();
    pl_st(w + n_wit + i, F::add(F::mul(pl_ld(fac + 2 * i), a), F::mul(pl_ld(fac + 2 * i + 1), b)));
}
// computeWirePolynomials (:256-280): out[i] = toMontgomery(w[map[i]]) for i < n_cons, 0 up to n
template <class F> SB_HD void pl_wire(uint64_t i, const uint32_t* map, const F* w, uint32_t n_vars, uint64_t n_cons, F* out) {
    F x = F::zero();
    if (i < n_cons) { uint32_t s = map[i]; if (s < n_vars) x = F::to_mont(pl_ld(w + s)); }
    pl_st(out + i, x);
}
// Polynomial.blindCoefficients (polynomial.js:68-93) on a coefficient array with >= n + cnt slots whose tail is zero
template <class F> SB_HD void pl_blind(F* p, uint64_t n, const F* bf, int cnt) {
    for (int i = 0; i < cnt; i++) {
        pl_st(p + n + i, F::add(pl_ld(p + n + i), bf[i]));
        pl_st(p + i, F::sub(pl_ld(p + i), bf[i]));
    }
}

// ---------------------------------------------------------------------------------------------- round 2
// computeZ (:381-420): the i-th numerator and denominator factor.  sigma evaluations live on the 4n domain (stride 4).
template <class F> SB_HD void pl_z_terms(uint64_t i, const F* A, const F* B, const F* C, const F* s1, const F* s2, const F* s3,
                                         const PlonkPow<F>& wpow, const PlonkRound<F>& r, F* num, F* den) {
    F a = pl_ld(A + i), b = pl_ld(B + i), c = pl_ld(C + i);
    F betaw = F::mul(r.beta, pl_pow(wpow, i));
    F n1 = F::add(F::add(a, betaw), r.gamma);
    F n2 = F::add(F::add(b, F::mul(r.k1, betaw)), r.gamma);
    F n3 = F::add(F::add(c, F::mul(r.k2, betaw)), r.gamma);
    pl_st(num + i, F::mul(n1, F::mul(n2, n3)));
    F d1 = F::add(F::add(a, F::mul(pl_ld(s1 + 4 * i), r.beta)), r.gamma);
    F d2 = F::add(F::add(b, F::mul(pl_ld(s2 + 4 * i), r.beta)), r.gamma);
    F d3 = F::add(F::add(c, F::mul(pl_ld(s3 + 4 * i), r.beta)), r.gamma);
    pl_st(den + i, F::mul(d1, F::mul(d2, d3)));
}
// Montgomery's simultaneous inversion over one chunk [lo, hi): out[j] = mul[j] / in[j]  (in != out; zeros give zeros)
template <class F> SB_HD void pl_ratio_chunk(const F* in, const F* mul, F* out, uint64_t lo, uint64_t hi) {
    F acc = F::one();
    for (uint64_t j = lo; j < hi; j++) { pl_st(out + j, acc); F x = pl_ld(in + j); if (!x.is_zero()) acc = F::mul(acc, x); }
    F inv = F::inv(acc);
    for (uint64_t j = hi; j-- > lo;) {
        F x = pl_ld(in + j);
        if (x.is_zero()) { pl_st(out + j, F::zero()); continue; }
        F xi = F::mul(inv, pl_ld(out + j));
        inv = F::mul(inv, x);
        pl_st(out + j, F::mul(xi, pl_ld(mul + j)));
    }
}

// ---------------------------------------------------------------------------------------------- round 3
// MulZ.mul4 (src/mul_z.js:104-147): product of four (value, blinding-part) pairs modulo Z_H on coset p of the 4n domain
template <class F> SB_HD void pl_mul4(const F& a, const F& b, const F& c, const F& d, const F& ap, const F& bp, const F& cp, const F& dp,
                                      int p, const PlonkRound<F>& r, F& res, F& resz) {
    F a_b = F::mul(a, b), a_bp = F::mul(a, bp), ap_b = F::mul(ap, b), ap_bp = F::mul(ap, bp);
    F c_d = F::mul(c, d), c_dp = F::mul(c, dp), cp_d = F::mul(cp, d), cp_dp = F::mul(cp, dp);
    res = F::mul(a_b, c_d);
    F a0 = F::mul(F::add(ap_b, a_bp), c_d);
    a0 = F::add(a0, F::mul(a_b, F::add(cp_d, c_dp)));
    resz = a0;
    if (p) {
        F a1 = F::mul(ap_bp, c_d);
        a1 = F::add(a1, F::mul(F::add(ap_b, a_bp), F::add(cp_d, c_dp)));
        a1 = F::add(a1, F::mul(a_b, cp_dp));
        F a2 = F::mul(F::add(a_bp, ap_b), cp_dp);
        a2 = F::add(a2, F::mul(ap_bp, F::add(c_dp, cp_d)));
        F a3 = F::mul(ap_bp, cp_dp);
        resz = F::add(resz, F::mul(r.z1[p], a1));
        resz = F::add(resz, F::mul(r.z2[p], a2));
        resz = F::add(resz, F::mul(r.z3[p], a3));
    }
}
struct PlonkTIn {      // 4n-point evaluation arrays (device pointers), untyped so that the struct is curve-independent
    const void *A, *B, *C, *Z, *QM, *QL, *QR, *QO, *QC, *S1, *S2, *S3, *LAG;   // LAG: n_public arrays of 4n, back to back
    const void* pubA;                                                           // A evaluations (first n_public used)
    uint32_t n_public;
};
// computeT (:512-627): one evaluation of T and of its blinding part Tz
template <class F> SB_HD void pl_t_eval(uint64_t i, uint64_t n4, const PlonkTIn& in, const PlonkPow<F>& w4pow, const PlonkRound<F>& r, F* T, F* Tz) {
    const F a = pl_ld((const F*)in.A + i), b = pl_ld((const F*)in.B + i), c = pl_ld((const F*)in.C + i), z = pl_ld((const F*)in.Z + i);
    const F zw = pl_ld((const F*)in.Z + ((i + 4) & (n4 - 1)));
    const F w = pl_pow(w4pow, i);
    const F ap = F::add(r.b[2], F::mul(r.b[1], w));
    const F bp = F::add(r.b[4], F::mul(r.b[3], w));
    const F cp = F::add(r.b[6], F::mul(r.b[5], w));
    const F zp = F::add(F::mul(F::add(F::mul(r.b[7], w), r.b[8]), w), r.b[9]);
    const F wW = F::mul(w, r.wn);
    const F zWp = F::add(F::mul(F::add(F::mul(r.b[7], wW), r.b[8]), wW), r.b[9]);
    const int p = (int)(i & 3);
    F pi = F::zero();
    for (uint32_t j = 0; j < in.n_public; j++)
        pi = F::sub(pi, F::mul(pl_ld((const F*)in.LAG + (uint64_t)j * n4 + i), pl_ld((const F*)in.pubA + j)));
    // e1 (MulZ.mul2, mul_z.js:49-70)
    const F qm = pl_ld((const F*)in.QM + i), ql = pl_ld((const F*)in.QL + i), qr = pl_ld((const F*)in.QR + i), qo = pl_ld((const F*)in.QO + i);
    F e1 = F::mul(a, b);
    F e1z = F::add(F::mul(a, bp), F::mul(ap, b));
    if (p) e1z = F::add(e1z, F::mul(r.z1[p], F::mul(ap, bp)));
    e1 = F::mul(e1, qm); e1z = F::mul(e1z, qm);
    e1 = F::add(e1, F::mul(a, ql)); e1z = F::add(e1z, F::mul(ap, ql));
    e1 = F::add(e1, F::mul(b, qr)); e1z = F::add(e1z, F::mul(bp, qr));
    e1 = F::add(e1, F::mul(c, qo)); e1z = F::add(e1z, F::mul(cp, qo));
    e1 = F::add(F::add(e1, pi), pl_ld((const F*)in.QC + i));
    // e2, e3
    const F betaw = F::mul(r.beta, w);
    F e2, e2z, e3, e3z;
    pl_mul4(F::add(F::add(a, betaw), r.gamma), F::add(F::add(b, F::mul(betaw, r.k1)), r.gamma), F::add(F::add(c, F::mul(betaw, r.k2)), r.gamma), z,
            ap, bp, cp, zp, p, r, e2, e2z);
    pl_mul4(F::add(F::add(a, F::mul(r.beta, pl_ld((const F*)in.S1 + i))), r.gamma), F::add(F::add(b, F::mul(r.beta, pl_ld((const F*)in.S2 + i))), r.gamma),
            F::add(F::add(c, F::mul(r.beta, pl_ld((const F*)in.S3 + i))), r.gamma), zw, ap, bp, cp, zWp, p, r, e3, e3z);
    // e4
    const F l1 = pl_ld((const F*)in.LAG + i);
    const F e4 = F::mul(F::mul(F::sub(z, F::one()), l1), r.alpha2);
    const F e4z = F::mul(F::mul(zp, l1), r.alpha2);
    pl_st(T + i, F::add(F::add(e1, F::mul(F::sub(e2, e3), r.alpha)), e4));
    pl_st(Tz + i, F::add(F::add(e1z, F::mul(F::sub(e2z, e3z), r.alpha)), e4z));
}
// Polynomial.divZh (polynomial.js:592-614) + T.add(Tz) (:645) for the four coefficients i, n+i, 2n+i, 3n+i.
// Returns nonzero when the reference would throw: 1 = "Polynomial is not divisible", 2 = "T Polynomial is not well calculated".
template <class F> SB_HD int pl_divzh(uint64_t i, uint64_t n, const F* t, const F* tz, F* out) {
    int bad = 0;
    F c0 = F::neg(pl_ld(t + i));
    F c1 = F::sub(c0, pl_ld(t + n + i));
    F c2 = F::sub(c1, pl_ld(t + 2 * n + i));
    F c3 = F::sub(c2, pl_ld(t + 3 * n + i));
    if (2 * n + i > 3 * n - 4 && !c2.is_zero()) bad = 1;
    if (!c3.is_zero()) bad = 1;                                  // 3n + i > 3n - 4 always
    F o2 = F::add(c2, pl_ld(tz + 2 * n + i)), o3 = F::add(c3, pl_ld(tz + 3 * n + i));
    if (i >= 6 && !o3.is_zero() && !bad) bad = 2;                // degree < 3n + 6 (:648-650)
    pl_st(out + i, F::add(c0, pl_ld(tz + i)));
    pl_st(out + n + i, F::add(c1, pl_ld(tz + n + i)));
    pl_st(out + 2 * n + i, o2);
    pl_st(out + 3 * n + i, o3);
    return bad;
}
// the split of T into T1 | T2 | T3 with b10, b11 (:660-682); i < n + 6
template <class F> SB_HD void pl_tsplit(uint64_t i, uint64_t n, const F* t, const F& b10, const F& b11, F* T1, F* T2, F* T3) {
    if (i < n) {
        pl_st(T1 + i, pl_ld(t + i));
        F x = pl_ld(t + n + i); if (i == 0) x = F::sub(x, b10);
        pl_st(T2 + i, x);
    } else if (i == n) { pl_st(T1 + i, b10); pl_st(T2 + i, b11); }
    F y = pl_ld(t + 2 * n + i); if (i == 0) y = F::sub(y, b11);
    pl_st(T3 + i, y);
}

// ---------------------------------------------------------------------------------------------- rounds 4-5
struct PlonkLinIn {    // coefficient arrays; lengths: Q*, S* n; A, B, C n+2; Z n+3; T1, T2 n+1; T3 n+6
    const void *QM, *QL, *QR, *QO, *QC, *S1, *S2, *S3, *A, *B, *C, *Z, *T1, *T2, *T3;
};
template <class F> SB_HD F pl_at(const void* p, uint64_t i, uint64_t len) { return i < len ? pl_ld((const F*)p + i) : F::zero(); }
// computeR (:752-856) and the numerator of computeWxi (:858-878), coefficient i < n + 6
template <class F> SB_HD F pl_wxi_coef(uint64_t i, uint64_t n, const PlonkLinIn& in, const PlonkLin<F>& k) {
    F r = F::mul(k.coef_ab, pl_at<F>(in.QM, i, n));
    r = F::add(r, F::mul(k.ea, pl_at<F>(in.QL, i, n)));
    r = F::add(r, F::mul(k.eb, pl_at<F>(in.QR, i, n)));
    r = F::add(r, F::mul(k.ec, pl_at<F>(in.QO, i, n)));
    r = F::add(r, pl_at<F>(in.QC, i, n));
    r = F::add(r, F::mul(k.e24, pl_at<F>(in.Z, i, n + 3)));
    r = F::sub(r, F::mul(k.e3beta, pl_at<F>(in.S3, i, n)));
    F t = F::mul(k.xin2, pl_at<F>(in.T3, i, n + 6));
    t = F::add(t, F::mul(k.xin, pl_at<F>(in.T2, i, n + 1)));
    t = F::add(t, pl_at<F>(in.T1, i, n + 1));
    r = F::sub(r, F::mul(k.zh, t));
    if (i == 0) r = F::add(r, k.r0);
    r = F::add(r, F::mul(k.v[1], pl_at<F>(in.A, i, n + 2)));
    r = F::add(r, F::mul(k.v[2], pl_at<F>(in.B, i, n + 2)));
    r = F::add(r, F::mul(k.v[3], pl_at<F>(in.C, i, n + 2)));
    r = F::add(r, F::mul(k.v[4], pl_at<F>(in.S1, i, n)));
    r = F::add(r, F::mul(k.v[5], pl_at<F>(in.S2, i, n)));
    if (i == 0) r = F::sub(r, k.wsub);
    return r;
}
// quotient coefficient j of f / (X - b) from the inclusive sums P of g[k] = f[k] b^k:  q[j] = (P[m-1] - P[j]) * (1/b)^(j+1); q[m-1] = 0.
// to_plain: the result leaves Montgomery form (it is an MSM scalar).
template <class F> SB_HD F pl_quot_coef(uint64_t j, uint64_t m, const F* P, const PlonkPow<F>& ipow) {
    if (j + 1 >= m) return F::zero();
    return F::mul(F::sub(pl_ld(P + m - 1), pl_ld(P + j)), pl_pow(ipow, j + 1));
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------ kernels
template <class F> __global__ void k_pl_additions(const uint32_t* __restrict__ order, uint32_t lo, uint32_t hi, const uint32_t* __restrict__ sig,
                                                  const F* __restrict__ fac, F* w, uint32_t n_wit, uint32_t n_vars) {
    uint32_t j = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (j < hi) pl_addition<F>(order[j], sig, fac, w, n_wit, n_vars);
}
struct PlonkMaps { const uint32_t* m[3]; void* out[3]; };
template <class F> __global__ void k_pl_wires(PlonkMaps mp, const F* __restrict__ w, uint32_t n_vars, uint64_t n_cons, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) pl_wire<F>(i, mp.m[blockIdx.y], w, n_vars, n_cons, (F*)mp.out[blockIdx.y]);
}
template <class F> struct PlonkBlind { F bf[3]; int cnt; };
template <class F> __global__ void k_pl_blind(F* p, uint64_t n, PlonkBlind<F> b) {
    if (blockIdx.x == 0 && threadIdx.x == 0) pl_blind<F>(p, n, b.bf, b.cnt);
}
template <class F> __global__ void k_pl_z_terms(uint64_t n, const F* A, const F* B, const F* C, const F* s1, const F* s2, const F* s3,
                                                PlonkPow<F> wpow, PlonkRound<F> r, F* num, F* den) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) pl_z_terms<F>(i, A, B, C, s1, s2, s3, wpow, r, num, den);
}
static constexpr int PL_INV_CHUNK = 16;
template <class F> __global__ void k_pl_ratio(const F* in, const F* mul, F* out, uint64_t n) {
    uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint64_t lo = t * PL_INV_CHUNK, hi = lo + PL_INV_CHUNK < n ? lo + PL_INV_CHUNK : n;
    if (lo < n) pl_ratio_chunk<F>(in, mul, out, lo, hi);
}
// flag |= 4 unless z[n-1] * ratio[n-1] == 1  ("Copy constraints does not match", :436-438)
template <class F> __global__ void k_pl_z_check(const F* z, const F* ratio, uint64_t n, int* flag) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { F t = F::mul(pl_ld(z + n - 1), pl_ld(ratio + n - 1)); if (!(t == F::one())) atomicOr(flag, 4); }
}
template <class F> __global__ void __launch_bounds__(128) k_pl_t(uint64_t n4, PlonkTIn in, PlonkPow<F> w4pow, PlonkRound<F> r, F* T, F* Tz) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n4) pl_t_eval<F>(i, n4, in, w4pow, r, T, Tz);
}
template <class F> __global__ void k_pl_divzh(uint64_t n, const F* t, const F* tz, F* out, int* flag) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) { int bad = pl_divzh<F>(i, n, t, tz, out); if (bad) atomicOr(flag, bad); }
}
template <class F> struct PlonkB2 { F b10, b11; };
template <class F> __global__ void k_pl_tsplit(uint64_t n, const F* t, PlonkB2<F> b, F* T1, F* T2, F* T3) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n + 6) pl_tsplit<F>(i, n, t, b.b10, b.b11, T1, T2, T3);
}
// g[k] = f[k] * x^k (f shorter than m is zero-extended); sub0 is subtracted from f[0] first
template <class F> struct PlonkOne { F x; };
template <class F> __global__ void k_pl_mul_pow(const F* f, uint64_t len, uint64_t m, PlonkPow<F> pw, PlonkOne<F> sub0, F* g) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    F x = i < len ? pl_ld(f + i) : F::zero();
    if (i == 0) x = F::sub(x, sub0.x);
    pl_st(g + i, F::mul(x, pl_pow(pw, i)));
}
template <class F> __global__ void k_pl_wxi(uint64_t n, PlonkLinIn in, PlonkLin<F> k, PlonkPow<F> pw, F* g) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n + 6) pl_st(g + i, F::mul(pl_wxi_coef<F>(i, n, in, k), pl_pow(pw, i)));
}
// q (Montgomery) and its plain copy for the MSM; flag |= 1 when the remainder P[m-1] is not zero
template <class F> __global__ void k_pl_quot(uint64_t m, const F* P, PlonkPow<F> ipow, F* q_plain, int* flag) {
    uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    if (j == 0 && !pl_ld(P + m - 1).is_zero()) atomicOr(flag, 1);
    pl_st(q_plain + j, F::from_mont(pl_quot_coef<F>(j, m, P, ipow)));
}

// ------------------------------------------------------------------------------------------------ batched kernels
// The kernels above with a proof axis (blockIdx.y = proof q, or row of a group-major array): every work array holds the K
// proofs back to back at a fixed stride, and per-proof scalars (PlonkRound, PlonkLin, power tables) come from small device
// arrays indexed by the proof.  A block never spans two proofs, so a block stages its proof's scalars in shared memory once.
template <class T> __device__ __forceinline__ const T& pl_stage(uint32_t* sh, const T* src) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
    for (unsigned t = threadIdx.x; t < sizeof(T) / 4; t += blockDim.x) sh[t] = s[t];
    __syncthreads();
    return *reinterpret_cast<const T*>(sh);
}
template <class F> __global__ void k_plb_additions(const uint32_t* __restrict__ order, uint32_t lo, uint32_t hi, const uint32_t* __restrict__ sig,
                                                   const F* __restrict__ fac, F* w, uint64_t sw, uint32_t n_wit, uint32_t n_vars) {
    uint32_t j = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (j < hi) pl_addition<F>(order[j], sig, fac, w + blockIdx.y * sw, n_wit, n_vars);
}
// grid (., K, 3): wire j of proof q goes to row j K + q of out (rows of n)
template <class F> __global__ void k_plb_wires(PlonkMaps mp, const F* __restrict__ w, uint64_t sw, uint32_t n_vars, uint64_t n_cons, uint64_t n, F* out) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) pl_wire<F>(i, mp.m[blockIdx.z], w + blockIdx.y * sw, n_vars, n_cons, out + ((uint64_t)blockIdx.z * gridDim.y + blockIdx.y) * n);
}
// one thread per row of groups x K rows of `stride` elements
template <class F> __global__ void k_plb_blind(F* p, uint64_t stride, uint64_t n, uint32_t rows, uint32_t K, const PlonkRound<F>* rs, PlonkBlindIdx bi) {
    uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    const uint32_t j = row / K, q = row % K;
    F bf[3];
    for (int t = 0; t < bi.cnt; t++) bf[t] = pl_ld(&rs[q].b[bi.idx[j][t]]);
    pl_blind<F>(p + row * stride, n, bf, bi.cnt);
}
// wires: 3K rows of n (A rows, then B, then C)
template <class F> __global__ void __launch_bounds__(128) k_plb_z_terms(uint64_t n, const F* wires, const F* s1, const F* s2, const F* s3,
                                                                        PlonkPow<F> wpow, const PlonkRound<F>* rs, F* num, F* den) {
    __shared__ __align__(16) uint32_t sh[sizeof(PlonkRound<F>) / 4];
    const uint64_t q = blockIdx.y, K = gridDim.y;
    const PlonkRound<F>& r = pl_stage(sh, rs + q);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) pl_z_terms<F>(i, wires + q * n, wires + (K + q) * n, wires + (2 * K + q) * n, s1, s2, s3, wpow, r, num + q * n, den + q * n);
}
// one thread per proof: flag[q] |= 4 unless z[n-1] * ratio[n-1] == 1 in proof q's rows
template <class F> __global__ void k_plb_z_check(const F* z, const F* ratio, uint64_t n, uint32_t K, int* flag) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= K) return;
    F t = F::mul(pl_ld(z + q * n + n - 1), pl_ld(ratio + q * n + n - 1));
    if (!(t == F::one())) flag[q] |= 4;
}
// ev: 3K rows of 4n (A, B, C evaluations), evZ: K rows of 4n, wires: A's rows give the public inputs; T, Tz: K rows of 4n
template <class F> __global__ void __launch_bounds__(128) k_plb_t(uint64_t n4, uint64_t n, PlonkTIn in, const F* ev, const F* evZ, const F* wires,
                                                                  PlonkPow<F> w4pow, const PlonkRound<F>* rs, F* T, F* Tz) {
    __shared__ __align__(16) uint32_t sh[sizeof(PlonkRound<F>) / 4];
    const uint64_t q = blockIdx.y, K = gridDim.y;
    const PlonkRound<F>& r = pl_stage(sh, rs + q);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n4) return;
    in.A = ev + q * n4; in.B = ev + (K + q) * n4; in.C = ev + (2 * K + q) * n4; in.Z = evZ + q * n4; in.pubA = wires + q * n;
    pl_t_eval<F>(i, n4, in, w4pow, r, T + q * n4, Tz + q * n4);
}
// t: T rows then Tz rows (K each, 4n); out: K rows of 4n
template <class F> __global__ void k_plb_divzh(uint64_t n, const F* t, F* out, int* flag) {
    const uint64_t q = blockIdx.y, K = gridDim.y, n4 = 4 * n;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) { int bad = pl_divzh<F>(i, n, t + q * n4, t + (K + q) * n4, out + q * n4); if (bad) atomicOr(flag + q, bad); }
}
// cT: 3K rows of stride p (T1 rows, T2 rows, T3 rows)
template <class F> __global__ void k_plb_tsplit(uint64_t n, uint64_t p, const F* t, const PlonkRound<F>* rs, F* cT) {
    const uint64_t q = blockIdx.y, K = gridDim.y;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n + 6) pl_tsplit<F>(i, n, t + q * 4 * n, pl_ld(&rs[q].b[10]), pl_ld(&rs[q].b[11]), cT + q * p, cT + (K + q) * p, cT + (2 * K + q) * p);
}
// round 4's six evaluations of every proof: row 6q + e of g (stride p) holds f_e[i] x^i, zero from the polynomial's length on.
// e = A, B, C (n + 2 coefficients), S1, S2 (n, the key's), Z (n + 3, at xi w); cABC: 3K rows, cZ: K rows, stride p.
template <class F> __global__ void k_plb_eval_terms(uint64_t n, uint64_t p, const F* cABC, const F* s1, const F* s2, const F* cZ,
                                                    PlonkPowK<F> pxi, PlonkPowK<F> pxiw, F* g) {
    const uint64_t row = blockIdx.y, q = row / 6, K = gridDim.y / 6; const int e = (int)(row % 6);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= p) return;
    const F* f; uint64_t len = n;
    if (e < 3) { f = cABC + (e * K + q) * p; len = n + 2; }
    else if (e == 3) f = s1;
    else if (e == 4) f = s2;
    else { f = cZ + q * p; len = n + 3; }
    pl_st(g + row * p + i, i < len ? F::mul(pl_ld(f + i), pl_pow(e == 5 ? pxiw.at(q) : pxi.at(q), i)) : F::zero());
}
// round 5's two divisions of every proof: row q of g (stride p = n + 6) is Wxi's numerator (computeR + computeWxi) times
// xi^i, row K + q is (Z - eval_zw) times (xi w)^i for i < n + 3 and zero after.  kin: the key's coefficient arrays.
template <class F> __global__ void __launch_bounds__(128) k_plb_wxi(uint64_t n, uint64_t p, PlonkLinIn kin, const F* cABC, const F* cZ, const F* cT,
                                                                    const PlonkLin<F>* Ls, const F* ezw, PlonkPowK<F> pxi, PlonkPowK<F> pxiw, F* g) {
    __shared__ __align__(16) uint32_t sh[sizeof(PlonkLin<F>) / 4];
    const uint64_t K = gridDim.y / 2, row = blockIdx.y, q = row % K;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (row < K) {
        const PlonkLin<F>& L = pl_stage(sh, Ls + q);
        if (i >= p) return;
        kin.A = cABC + q * p; kin.B = cABC + (K + q) * p; kin.C = cABC + (2 * K + q) * p; kin.Z = cZ + q * p;
        kin.T1 = cT + q * p; kin.T2 = cT + (K + q) * p; kin.T3 = cT + (2 * K + q) * p;
        pl_st(g + row * p + i, F::mul(pl_wxi_coef<F>(i, n, kin, L), pl_pow(pxi.at(q), i)));
    } else {
        if (i >= p) return;
        F x = i < n + 3 ? pl_ld(cZ + q * p + i) : F::zero();
        if (i == 0) x = F::sub(x, pl_ld(ezw + q));
        pl_st(g + row * p + i, F::mul(x, pl_pow(pxiw.at(q), i)));
    }
}
// quotient rows from their inclusive sums P (stride p): row q divides by X - xi (m = n + 6), row K + q by X - xi w (m = n + 3);
// plain scalars, zero from m on; flag[q] |= 1 when a remainder is not zero
template <class F> __global__ void k_plb_quot(uint64_t n, uint64_t p, const F* P, PlonkPowK<F> ipxi, PlonkPowK<F> ipxiw, F* q_plain, int* flag) {
    const uint64_t K = gridDim.y / 2, row = blockIdx.y, q = row % K;
    const uint64_t m = row < K ? n + 6 : n + 3;
    uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (j >= p) return;
    const F* Pr = P + row * p;
    if (j == 0 && !pl_ld(Pr + m - 1).is_zero()) atomicOr(flag + q, 1);
    pl_st(q_plain + row * p + j, j < m ? F::from_mont(pl_quot_coef<F>(j, m, Pr, row < K ? ipxi.at(q) : ipxiw.at(q))) : F::zero());
}
// segment id of an array-major batch: element idx belongs to row idx / len
struct PlbRowKey {
    uint64_t len;
    __host__ __device__ __forceinline__ uint32_t operator()(uint64_t idx) const { return (uint32_t)(idx / len); }
};
struct PlbRowOff {
    uint64_t len;
    __host__ __device__ __forceinline__ int64_t operator()(uint64_t row) const { return (int64_t)(row * len); }
};

struct FrAddOp { template <class F> __host__ __device__ __forceinline__ F operator()(const F& a, const F& b) const { return F::add(a, b); } };
struct FrMulOp { template <class F> __host__ __device__ __forceinline__ F operator()(const F& a, const F& b) const { return F::mul(a, b); } };
#endif  // __CUDACC__

}  // namespace sb
