// ec.cuh — Fp2 and short-Weierstrass (a = 0) point arithmetic for the MSM kernels.
//
// The reference accumulates buckets in Jacobian coordinates (wasmcurves build_curve_jacobian_a0,
// build/snarkjs.js:5944-7430; addMixed 6576-6678).  MSM results are only defined up to the projective
// representative (SURVEY.md §3.3), so the GPU path uses extended Jacobian "XYZZ" coordinates
// (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2): mixed add 8M+2S instead of 7M+4S, no field inversion, and
// infinity is ZZ == 0.  All the reference's special cases are kept: base at infinity (all-zero bytes),
// empty accumulator, P + P (doubling) and P + (-P) (infinity).
#pragma once
#include "fp.cuh"

namespace sb {

// Fp2 = Fp[u]/(u^2+1)  (reference build_f2m 4028; mul 4157; square 4216).  Byte order c0 || c1.
template <class P> struct Fp2 {
    typedef Fp<P> B;
    static constexpr bool HAS_MUL2 = false;
    B a, b;
    SB_HD static Fp2 one() { Fp2 r; r.a = B::one(); r.b = B::zero(); return r; }
    SB_HD static Fp2 inv(const Fp2& x) {   // (a - bu)/(a^2 + b^2)
        B t = B::inv_binary(B::add(B::sqr(x.a), B::sqr(x.b)));
        Fp2 r; r.a = B::mul(x.a, t); r.b = B::neg(B::mul(x.b, t)); return r;
    }
    SB_HD static Fp2 zero() { Fp2 r; r.a = B::zero(); r.b = B::zero(); return r; }
    SB_HD bool is_zero() const { return a.is_zero() & b.is_zero(); }
    SB_HD bool operator==(const Fp2& o) const { return (a == o.a) & (b == o.b); }
    SB_HD static Fp2 add(const Fp2& x, const Fp2& y) { Fp2 r; r.a = B::add(x.a, y.a); r.b = B::add(x.b, y.b); return r; }
    SB_HD static Fp2 sub(const Fp2& x, const Fp2& y) { Fp2 r; r.a = B::sub(x.a, y.a); r.b = B::sub(x.b, y.b); return r; }
    SB_HD static Fp2 dbl(const Fp2& x) { Fp2 r; r.a = B::dbl(x.a); r.b = B::dbl(x.b); return r; }
    SB_HD static Fp2 neg(const Fp2& x) { Fp2 r; r.a = B::neg(x.a); r.b = B::neg(x.b); return r; }
    SB_HD static Fp2 cneg(const Fp2& x, bool f) { Fp2 r; r.a = B::cneg(x.a, f); r.b = B::cneg(x.b, f); return r; }
    // Karatsuba, 3 base multiplies
    SB_HD_NOINLINE static Fp2 mul(const Fp2& x, const Fp2& y) { return mul_i(x, y); }
    SB_HD_NOINLINE static Fp2 sqr(const Fp2& x) { return sqr_i(x); }
    // force-inlined variants for the hot bucket-accumulation loop (everything else calls the out-of-line ones to keep
    // code size and compile time down)
    SB_HD static Fp2 mul_i(const Fp2& x, const Fp2& y) {
#if defined(__CUDA_ARCH__) && defined(SB_FP2_LAZY)   // off by default: fewer MACs, but more live registers in the G2 accumulation
        return mul_lazy(x, y);          // 5 N^2 wide MACs
#endif
        if constexpr (B::HAS_MUL2) {
            // schoolbook with two dual-product multiplies (one reduction each): c0 = a0 b0 + a1 (-b1), c1 = a0 b1 + a1 b0.
            // Same 6 N^2 wide MACs as Karatsuba's three multiplies, but none of its five additions/subtractions.
            Fp2 r; r.a = B::mul2(x.a, y.a, x.b, B::neg(y.b)); r.b = B::mul2(x.a, y.b, x.b, y.a); return r;
        } else {
            B A = B::mul(x.a, y.a), Bb = B::mul(x.b, y.b);
            B C = B::mul(B::add(x.a, x.b), B::add(y.a, y.b));
            Fp2 r; r.a = B::sub(A, Bb); r.b = B::sub(B::sub(C, A), Bb); return r;
        }
    }
    // Karatsuba on double-width products with lazy reduction: 3 N^2 (products) + 2 N^2 (two reductions) wide MACs
    // instead of 6 N^2.  v2 - v0 - v1 = a0 b1 + a1 b0 >= 0 and < 2p^2 < pR; v0 - v1 is made non-negative by adding p*R.
    SB_HD static Fp2 mul_lazy(const Fp2& x, const Fp2& y) {
        constexpr int N = B::N;
        uint32_t v0[2 * N], v1[2 * N], v2[2 * N], sa[N], sb[N];
        B::mul_wide(x.a.v, y.a.v, v0);
        B::mul_wide(x.b.v, y.b.v, v1);
        B::add_noreduce(x.a, x.b, sa); B::add_noreduce(y.a, y.b, sb);
        B::mul_wide(sa, sb, v2);
        B::wide_sub(v2, v0); B::wide_sub(v2, v1);
        uint32_t bw = B::wide_sub(v0, v1);
        B::wide_add_p_high(v0, bw);
        Fp2 r; r.a = B::redc_wide(v0); r.b = B::redc_wide(v2); return r;
    }
    // complex squaring, 2 base multiplies
    SB_HD static Fp2 sqr_i(const Fp2& x) {
        B AB = B::mul(x.a, x.b);
        Fp2 r; r.a = B::mul(B::add(x.a, x.b), B::sub(x.a, x.b)); r.b = B::dbl(AB); return r;
    }
};

// Affine point (x, y); infinity = (0, 0) (reference 6068-6086).
template <class F> struct Affine {
    F x, y;
    SB_HD bool is_inf() const { return x.is_zero() & y.is_zero(); }
};

// Extended Jacobian point.
template <class F> struct XYZZ {
    F x, y, zz, zzz;
    SB_HD static XYZZ inf() { XYZZ r; r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero(); return r; }
    SB_HD bool is_inf() const { return zz.is_zero(); }

    // 2 * (affine p), p not infinity   (mdbl-2008-s-1)
    SB_HD_NOINLINE static XYZZ dbl_affine(const F& px, const F& py, const F& one) {
        XYZZ r;
        if (py.is_zero()) return inf();
        F U = F::dbl(py), V = F::sqr(U), W = F::mul(U, V), S = F::mul(px, V);
        F M = F::sqr(px); M = F::add(F::dbl(M), M);
        r.x = F::sub(F::sqr(M), F::dbl(S));
        r.y = F::sub(F::mul(M, F::sub(S, r.x)), F::mul(W, py));
        r.zz = V; r.zzz = W;
        (void)one;
        return r;
    }
    // 2 * p   (dbl-2008-s-1, a = 0)
    SB_HD_NOINLINE static XYZZ dbl(const XYZZ& p) {
        if (p.is_inf() || p.y.is_zero()) return inf();
        XYZZ r;
        F U = F::dbl(p.y), V = F::sqr(U), W = F::mul(U, V), S = F::mul(p.x, V);
        F M = F::sqr(p.x); M = F::add(F::dbl(M), M);
        r.x = F::sub(F::sqr(M), F::dbl(S));
        r.y = F::sub(F::mul(M, F::sub(S, r.x)), F::mul(W, p.y));
        r.zz = F::mul(V, p.zz); r.zzz = F::mul(W, p.zzz);
        return r;
    }
    // acc += (qx, qy) affine, q not infinity (madd-2008-s), `one` = Montgomery 1.
    SB_HD void add_affine(const F& qx, const F& qy, const F& one) {
        if (is_inf()) { x = qx; y = qy; zz = one; zzz = one; return; }
        F U2 = F::mul_i(qx, zz), S2 = F::mul_i(qy, zzz);
        F Pp = F::sub(U2, x), R = F::sub(S2, y);
        if (Pp.is_zero()) {            // same x: doubling or cancellation (reference 6620-6640 special cases)
            if (R.is_zero()) *this = dbl_affine(qx, qy, one);
            else *this = inf();
            return;
        }
        F PP = F::sqr_i(Pp), PPP = F::mul_i(Pp, PP), Q = F::mul_i(x, PP);
        F X3 = F::sub(F::sub(F::sqr_i(R), PPP), F::dbl(Q));
        F Y3;
        if constexpr (F::HAS_MUL2) Y3 = F::mul2_i(R, F::sub(Q, X3), F::neg(y), PPP);   // R(Q - X3) - Y1*PPP, one reduction
        else Y3 = F::sub(F::mul_i(R, F::sub(Q, X3)), F::mul_i(y, PPP));
        x = X3; y = Y3; zz = F::mul_i(zz, PP); zzz = F::mul_i(zzz, PPP);
    }
    // acc += q   (add-2008-s), for the device reduction kernels: the same formulas and special cases as add() below, hence
    // the same bytes, with the force-inlined multiplies.  q's zz and zzz enter their last products first, so they die
    // before the bulk of the addition.
    SB_HD void add_i(const XYZZ& q) {
        if (q.is_inf()) return;
        if (is_inf()) { *this = q; return; }
        F U1 = F::mul_i(x, q.zz), S1 = F::mul_i(y, q.zzz);
        F ZZ = F::mul_i(zz, q.zz), ZZZ = F::mul_i(zzz, q.zzz);
        F Pp = F::sub(F::mul_i(q.x, zz), U1), R = F::sub(F::mul_i(q.y, zzz), S1);
        if (Pp.is_zero()) {
            if (R.is_zero()) *this = dbl(*this);
            else *this = inf();
            return;
        }
        F PP = F::sqr_i(Pp), PPP = F::mul_i(Pp, PP), Q = F::mul_i(U1, PP);
        F X3 = F::sub(F::sub(F::sqr_i(R), PPP), F::dbl(Q));
        F Y3;
        if constexpr (F::HAS_MUL2) Y3 = F::mul2_i(R, F::sub(Q, X3), F::neg(S1), PPP);   // R(Q - X3) - S1*PPP, one reduction
        else Y3 = F::sub(F::mul_i(R, F::sub(Q, X3)), F::mul_i(S1, PPP));
        x = X3; y = Y3; zz = F::mul_i(ZZ, PP); zzz = F::mul_i(ZZZ, PPP);
    }
    // acc += q   (add-2008-s): host code and the group FFT
    SB_HD void add(const XYZZ& q) {
        if (q.is_inf()) return;
        if (is_inf()) { *this = q; return; }
        F U1 = F::mul(x, q.zz), U2 = F::mul(q.x, zz);
        F S1 = F::mul(y, q.zzz), S2 = F::mul(q.y, zzz);
        F Pp = F::sub(U2, U1), R = F::sub(S2, S1);
        if (Pp.is_zero()) {
            if (R.is_zero()) *this = dbl(*this);
            else *this = inf();
            return;
        }
        F PP = F::sqr(Pp), PPP = F::mul(Pp, PP), Q = F::mul(U1, PP);
        F X3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
        F Y3 = F::sub(F::mul(R, F::sub(Q, X3)), F::mul(S1, PPP));
        x = X3; y = Y3;
        zz = F::mul(F::mul(zz, q.zz), PP); zzz = F::mul(F::mul(zzz, q.zzz), PPP);
    }
};

}  // namespace sb
