// field_eval.cuh — per-record dispatch of the fp.cuh / ec.cuh primitives for sb_field_eval, a test hook that runs one
// primitive over an array of operand records.  The kernel (field_eval.cu) and the CPU driver of the same code
// (tests/host/field_eval_host.cpp) both call field_eval_record; nothing on the proving path does.
//
// Fields (the oracle's F_* ids, then the two Fq2): 0 BN254 Fq, 1 BN254 Fr, 2 BLS12-381 Fq, 3 BLS12-381 Fr, 4 BN254 Fq2,
// 5 BLS12-381 Fq2.  A record is k little-endian elements of N 32-bit limbs (N of the base field); an Fq2 element is c0 || c1.
// The point ops name a group by its base field: 0 BN254 G1, 2 BLS12-381 G1, 4 BN254 G2, 5 BLS12-381 G2; a point is its
// coordinates in that order (x y for affine, x y zz zzz for XYZZ), each one element of the base field.
#pragma once
#include "ec.cuh"

namespace sb {

enum { FE_BN_FQ = 0, FE_BN_FR, FE_BLS_FQ, FE_BLS_FR, FE_BN_FQ2, FE_BLS_FQ2, FE_NFIELDS };
enum {
    // Fp (fields 0-3)                                 record in -> out, in elements
    FE_ADD = 0, FE_SUB, FE_NEG, FE_DBL,             // a b -> a+b, a b -> a-b, a -> -a, a -> 2a
    FE_MUL,                                          // a b -> a*b*R^-1
    FE_MUL2,                                         // x y u v -> (x*y + u*v)*R^-1; fields with Fp::HAS_MUL2 only
    FE_MUL_WIDE,                                     // a b -> a*b (2 elements: 2N limbs)
    FE_REDC_WIDE,                                    // T (2N limbs, T < p*R) -> T*R^-1
    FE_TO_MONT, FE_FROM_MONT,                        // a -> a*R, a -> a*R^-1 (any a < 2^(32N))
    FE_INV_BINARY, FE_INV,                           // a -> R^2*a^-1 (0 -> 0): Kaliski, Fermat
    // Fq2 (fields 4-5)
    FE_FP2_MUL_I, FE_FP2_MUL_LAZY,                   // x y -> x*y: dual-product schoolbook, lazy Karatsuba
    FE_FP2_SQR_I, FE_FP2_INV,                        // x -> x^2, x -> x^-1 (0 -> 0)
    // XYZZ points (fields 0, 2, 4, 5)
    FE_EC_ADD_AFFINE,                                // acc q -> acc.add_affine(q) (acc XYZZ, q affine, not infinity)
    FE_EC_ADD_I, FE_EC_ADD,                          // acc q -> acc.add_i(q), acc.add(q) (both XYZZ)
    FE_EC_DBL, FE_EC_DBL_AFFINE,                     // p -> dbl(p) (XYZZ), p -> dbl_affine(p) (affine)
    FE_NOPS
};

SB_CONSTEXPR_HD constexpr bool field_eval_has_mul2(int field) {
    return field == FE_BN_FQ ? Fp<BnFq>::HAS_MUL2 : field == FE_BN_FR ? Fp<BnFr>::HAS_MUL2
         : field == FE_BLS_FQ ? Fp<BlsFq>::HAS_MUL2 : field == FE_BLS_FR ? Fp<BlsFr>::HAS_MUL2 : false;
}
// 32-bit words of one input record (out == false) or one output record (out == true); 0 if the pair does not exist
SB_CONSTEXPR_HD constexpr int field_eval_words(int field, int op, bool out) {
    if (field < 0 || field >= FE_NFIELDS) return 0;
    const int n = (field == FE_BLS_FQ || field == FE_BLS_FQ2) ? 12 : 8;
    if (op >= FE_EC_ADD_AFFINE && op < FE_NOPS) {
        if (field == FE_BN_FR || field == FE_BLS_FR) return 0;
        const int e = field >= FE_BN_FQ2 ? 2 * n : n;   // words per coordinate
        switch (op) {
        case FE_EC_ADD_AFFINE: return out ? 4 * e : 6 * e;
        case FE_EC_ADD_I: case FE_EC_ADD: return out ? 4 * e : 8 * e;
        case FE_EC_DBL: return 4 * e;
        default: return out ? 4 * e : 2 * e;       // FE_EC_DBL_AFFINE
        }
    }
    if (field >= FE_BN_FQ2) {
        if (op == FE_FP2_MUL_I || op == FE_FP2_MUL_LAZY) return out ? 2 * n : 4 * n;
        if (op == FE_FP2_SQR_I || op == FE_FP2_INV) return 2 * n;
        return 0;
    }
    switch (op) {
    case FE_ADD: case FE_SUB: case FE_MUL: return out ? n : 2 * n;
    case FE_NEG: case FE_DBL: case FE_TO_MONT: case FE_FROM_MONT: case FE_INV_BINARY: case FE_INV: return n;
    case FE_MUL2: return field_eval_has_mul2(field) ? (out ? n : 4 * n) : 0;
    case FE_MUL_WIDE: return 2 * n;
    case FE_REDC_WIDE: return out ? n : 2 * n;
    default: return 0;
    }
}

template <class P> SB_HD Fp<P> fe_ld(const uint32_t* w) {
    Fp<P> x;
_Pragma("unroll")
    for (int i = 0; i < P::N; i++) x.v[i] = w[i];
    return x;
}
template <class P> SB_HD void fe_st(uint32_t* w, const Fp<P>& x) {
_Pragma("unroll")
    for (int i = 0; i < P::N; i++) w[i] = x.v[i];
}

template <class P> SB_HD void field_eval_fp(int op, const uint32_t* in, uint32_t* out) {
    typedef Fp<P> F;
    constexpr int N = P::N;
    switch (op) {
    case FE_ADD: fe_st(out, F::add(fe_ld<P>(in), fe_ld<P>(in + N))); break;
    case FE_SUB: fe_st(out, F::sub(fe_ld<P>(in), fe_ld<P>(in + N))); break;
    case FE_NEG: fe_st(out, F::neg(fe_ld<P>(in))); break;
    case FE_DBL: fe_st(out, F::dbl(fe_ld<P>(in))); break;
    case FE_MUL: fe_st(out, F::mul(fe_ld<P>(in), fe_ld<P>(in + N))); break;
    case FE_MUL2:
        if constexpr (F::HAS_MUL2) fe_st(out, F::mul2(fe_ld<P>(in), fe_ld<P>(in + N), fe_ld<P>(in + 2 * N), fe_ld<P>(in + 3 * N)));
        break;
    case FE_MUL_WIDE: {
        F a = fe_ld<P>(in), b = fe_ld<P>(in + N);
        uint32_t T[2 * N];
        F::mul_wide(a.v, b.v, T);
_Pragma("unroll")
        for (int i = 0; i < 2 * N; i++) out[i] = T[i];
        break;
    }
    case FE_REDC_WIDE: {
        uint32_t T[2 * N];
_Pragma("unroll")
        for (int i = 0; i < 2 * N; i++) T[i] = in[i];
        fe_st(out, F::redc_wide(T));
        break;
    }
    case FE_TO_MONT: fe_st(out, F::to_mont(fe_ld<P>(in))); break;
    case FE_FROM_MONT: fe_st(out, F::from_mont(fe_ld<P>(in))); break;
    case FE_INV_BINARY: fe_st(out, F::inv_binary(fe_ld<P>(in))); break;
    case FE_INV: fe_st(out, F::inv(fe_ld<P>(in))); break;
    default: break;
    }
}

template <class P> SB_HD void field_eval_fp2(int op, const uint32_t* in, uint32_t* out) {
    typedef Fp2<P> F2;
    constexpr int N = P::N;
    F2 x, y, r;
    x.a = fe_ld<P>(in); x.b = fe_ld<P>(in + N);
    switch (op) {
    case FE_FP2_MUL_I: y.a = fe_ld<P>(in + 2 * N); y.b = fe_ld<P>(in + 3 * N); r = F2::mul_i(x, y); break;
    case FE_FP2_MUL_LAZY: y.a = fe_ld<P>(in + 2 * N); y.b = fe_ld<P>(in + 3 * N); r = F2::mul_lazy(x, y); break;
    case FE_FP2_SQR_I: r = F2::sqr_i(x); break;
    case FE_FP2_INV: r = F2::inv(x); break;
    default: return;
    }
    fe_st(out, r.a); fe_st(out + N, r.b);
}

// coordinates of an Fp or Fp2 point
template <class P> SB_HD void ec_ld(Fp<P>& x, const uint32_t* w) { x = fe_ld<P>(w); }
template <class P> SB_HD void ec_ld(Fp2<P>& x, const uint32_t* w) { x.a = fe_ld<P>(w); x.b = fe_ld<P>(w + P::N); }
template <class P> SB_HD void ec_st(uint32_t* w, const Fp<P>& x) { fe_st(w, x); }
template <class P> SB_HD void ec_st(uint32_t* w, const Fp2<P>& x) { fe_st(w, x.a); fe_st(w + P::N, x.b); }
template <class F> SB_HD XYZZ<F> ec_ld_xyzz(const uint32_t* w) {
    constexpr int E = sizeof(F) / 4;
    XYZZ<F> p;
    ec_ld(p.x, w); ec_ld(p.y, w + E); ec_ld(p.zz, w + 2 * E); ec_ld(p.zzz, w + 3 * E);
    return p;
}

// The point formulas as the MSM and group FFT kernels call them.  add_affine is handed `one` = F::one() as k_accumulate
// hands it; its q is never infinity there (k_accumulate drops (0, 0) bases before the addition), so no record may be.
template <class F> SB_HD void field_eval_ec(int op, const uint32_t* in, uint32_t* out) {
    constexpr int E = sizeof(F) / 4;                 // words per coordinate
    static_assert(E * 4 == sizeof(F), "a coordinate is whole 32-bit words");
    XYZZ<F> r;
    F qx, qy;
    switch (op) {
    case FE_EC_ADD_AFFINE:
        r = ec_ld_xyzz<F>(in); ec_ld(qx, in + 4 * E); ec_ld(qy, in + 5 * E);
        r.add_affine(qx, qy, F::one());
        break;
    case FE_EC_ADD_I: r = ec_ld_xyzz<F>(in); r.add_i(ec_ld_xyzz<F>(in + 4 * E)); break;
    case FE_EC_ADD: r = ec_ld_xyzz<F>(in); r.add(ec_ld_xyzz<F>(in + 4 * E)); break;
    case FE_EC_DBL: r = XYZZ<F>::dbl(ec_ld_xyzz<F>(in)); break;
    case FE_EC_DBL_AFFINE: ec_ld(qx, in); ec_ld(qy, in + E); r = XYZZ<F>::dbl_affine(qx, qy, F::one()); break;
    default: return;
    }
    ec_st(out, r.x); ec_st(out + E, r.y); ec_st(out + 2 * E, r.zz); ec_st(out + 3 * E, r.zzz);
}

// one record of (field, op); the caller has checked field_eval_words(field, op, ...) != 0
SB_HD void field_eval_record(int field, int op, const uint32_t* in, uint32_t* out) {
    if (op >= FE_EC_ADD_AFFINE) {
        switch (field) {
        case FE_BN_FQ: field_eval_ec<Fp<BnFq>>(op, in, out); break;
        case FE_BLS_FQ: field_eval_ec<Fp<BlsFq>>(op, in, out); break;
        case FE_BN_FQ2: field_eval_ec<Fp2<BnFq>>(op, in, out); break;
        case FE_BLS_FQ2: field_eval_ec<Fp2<BlsFq>>(op, in, out); break;
        default: break;
        }
        return;
    }
    switch (field) {
    case FE_BN_FQ: field_eval_fp<BnFq>(op, in, out); break;
    case FE_BN_FR: field_eval_fp<BnFr>(op, in, out); break;
    case FE_BLS_FQ: field_eval_fp<BlsFq>(op, in, out); break;
    case FE_BLS_FR: field_eval_fp<BlsFr>(op, in, out); break;
    case FE_BN_FQ2: field_eval_fp2<BnFq>(op, in, out); break;
    case FE_BLS_FQ2: field_eval_fp2<BlsFq>(op, in, out); break;
    default: break;
    }
}

}  // namespace sb
