// fp.cuh — prime-field arithmetic for sm_90a: N x 32-bit limbs, Montgomery form, R = 2^(32N).
//
// Replaces wasmcurves' build_f1m (reference build/snarkjs.js:2861-3830; mul 3072-3273) on the GPU.
// The reference multiplies by product scanning with 64-bit WASM accumulators; here the multiply is a
// word-serial CIOS with two column-aligned accumulator rows ("even"/"odd"), so every
// mad.lo.cc / madc.hi.cc pair lands on one aligned 64-bit column and ptxas can fuse the pair into
// a single IMAD.WIDE.U32 with carry.  All results are fully reduced to [0,p) — byte-identical to the
// reference's canonical representation.
#pragma once
#include <cstdint>

namespace sb {

// ---------------------------------------------------------------------------------------------
// Field parameter tags.  p(i)/r2(i)/one(i) are constexpr so that, after unrolling, every limb
// becomes an immediate or constant-bank operand (no registers spent on the modulus).
// np0 = -p^-1 mod 2^32 (reference build/snarkjs.js:3092).
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
#define SB_CONSTEXPR_HD __host__ __device__
#else
#define SB_CONSTEXPR_HD
#endif
#define SB_L(...) {__VA_ARGS__}
#define SB_FIELD_TAG(NAME, NLIMBS, NP0, PL, ONEL, R2L)                                          \
    struct NAME {                                                                             \
        static constexpr int N = NLIMBS;                                                      \
        static constexpr uint32_t np0 = NP0;                                                  \
        SB_CONSTEXPR_HD static constexpr uint32_t p(int i)   { constexpr uint32_t v[NLIMBS] = PL;   return v[i]; } \
        SB_CONSTEXPR_HD static constexpr uint32_t one(int i) { constexpr uint32_t v[NLIMBS] = ONEL; return v[i]; } \
        SB_CONSTEXPR_HD static constexpr uint32_t r2(int i)  { constexpr uint32_t v[NLIMBS] = R2L;  return v[i]; } \
    };

// BN254 base field q (build/snarkjs.js:9394); limbs: p, R mod p, R^2 mod p
SB_FIELD_TAG(BnFq, 8, 0xe4866389u,
    SB_L(0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u),
    SB_L(0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u),
    SB_L(0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u))
// BN254 scalar field r (build/snarkjs.js:9395)
SB_FIELD_TAG(BnFr, 8, 0xefffffffu,
    SB_L(0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u),
    SB_L(0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u),
    SB_L(0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u))
// BLS12-381 base field q (build/snarkjs.js:10797-10815)
SB_FIELD_TAG(BlsFq, 12, 0xfffcfffdu,
    SB_L(0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau),
    SB_L(0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u, 0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u),
    SB_L(0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u, 0x4c95b6d5u, 0x8de5476cu, 0x939d83c0u, 0x67eb88a9u, 0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u))
// BLS12-381 scalar field r
SB_FIELD_TAG(BlsFr, 8, 0xffffffffu,
    SB_L(0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u),
    SB_L(0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau, 0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u),
    SB_L(0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u, 0x0748d9d9u))

// ---------------------------------------------------------------------------------------------
// carry-chain PTX primitives
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
#define SB_HD __host__ __device__ __forceinline__
#define SB_HD_NOINLINE __host__ __device__ __noinline__
#else
#define SB_HD inline
#define SB_HD_NOINLINE inline
#endif

// On the device these are single PTX instructions sharing the hardware carry flag.  On the host
// (unit tests of the exact same template code, tests/host_fp_check.cpp) the flag is emulated.
namespace ptx {
#ifdef __CUDA_ARCH__
#define SB_ASM(...) asm volatile(__VA_ARGS__)
SB_HD uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; SB_ASM("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SB_HD uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; SB_ASM("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SB_HD void mad_lo_cc(uint32_t& acc, uint32_t a, uint32_t b)  { SB_ASM("mad.lo.cc.u32 %0, %1, %2, %0;"  : "+r"(acc) : "r"(a), "r"(b)); }
SB_HD void madc_lo_cc(uint32_t& acc, uint32_t a, uint32_t b) { SB_ASM("madc.lo.cc.u32 %0, %1, %2, %0;" : "+r"(acc) : "r"(a), "r"(b)); }
SB_HD void madc_hi_cc(uint32_t& acc, uint32_t a, uint32_t b) { SB_ASM("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(acc) : "r"(a), "r"(b)); }
SB_HD void madc_lo_cc3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { SB_ASM("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
SB_HD void madc_hi_cc3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { SB_ASM("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
SB_HD void madc_hi3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c)    { SB_ASM("madc.hi.u32 %0, %1, %2, %3;"    : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
SB_HD void add_cc(uint32_t& r, uint32_t a, uint32_t b)  { SB_ASM("add.cc.u32 %0, %1, %2;"  : "=r"(r) : "r"(a), "r"(b)); }
SB_HD void addc_cc(uint32_t& r, uint32_t a, uint32_t b) { SB_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
SB_HD void addc(uint32_t& r, uint32_t a, uint32_t b)    { SB_ASM("addc.u32 %0, %1, %2;"    : "=r"(r) : "r"(a), "r"(b)); }
SB_HD void sub_cc(uint32_t& r, uint32_t a, uint32_t b)  { SB_ASM("sub.cc.u32 %0, %1, %2;"  : "=r"(r) : "r"(a), "r"(b)); }
SB_HD void subc_cc(uint32_t& r, uint32_t a, uint32_t b) { SB_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
SB_HD void subc(uint32_t& r, uint32_t a, uint32_t b)    { SB_ASM("subc.u32 %0, %1, %2;"    : "=r"(r) : "r"(a), "r"(b)); }
#else
static thread_local uint32_t g_cc = 0;   // emulated carry/borrow flag
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t emu_add(uint32_t a, uint32_t b, uint32_t cin, bool setcc) { uint64_t t = (uint64_t)a + b + cin; if (setcc) g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t emu_sub(uint32_t a, uint32_t b, uint32_t bin, bool setcc) { uint64_t t = (uint64_t)a - b - bin; if (setcc) g_cc = (uint32_t)((t >> 32) & 1); return (uint32_t)t; }
inline void mad_lo_cc(uint32_t& acc, uint32_t a, uint32_t b)  { acc = emu_add(mul_lo(a, b), acc, 0, true); }
inline void madc_lo_cc(uint32_t& acc, uint32_t a, uint32_t b) { acc = emu_add(mul_lo(a, b), acc, g_cc, true); }
inline void madc_hi_cc(uint32_t& acc, uint32_t a, uint32_t b) { acc = emu_add(mul_hi(a, b), acc, g_cc, true); }
inline void madc_lo_cc3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { r = emu_add(mul_lo(a, b), c, g_cc, true); }
inline void madc_hi_cc3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { r = emu_add(mul_hi(a, b), c, g_cc, true); }
inline void madc_hi3(uint32_t& r, uint32_t a, uint32_t b, uint32_t c)    { r = emu_add(mul_hi(a, b), c, g_cc, false); }
inline void add_cc(uint32_t& r, uint32_t a, uint32_t b)  { r = emu_add(a, b, 0, true); }
inline void addc_cc(uint32_t& r, uint32_t a, uint32_t b) { r = emu_add(a, b, g_cc, true); }
inline void addc(uint32_t& r, uint32_t a, uint32_t b)    { r = emu_add(a, b, g_cc, false); }
inline void sub_cc(uint32_t& r, uint32_t a, uint32_t b)  { r = emu_sub(a, b, 0, true); }
inline void subc_cc(uint32_t& r, uint32_t a, uint32_t b) { r = emu_sub(a, b, g_cc, true); }
inline void subc(uint32_t& r, uint32_t a, uint32_t b)    { r = emu_sub(a, b, g_cc, false); }
#endif
}  // namespace ptx

// ---------------------------------------------------------------------------------------------
// Fp<P>
// ---------------------------------------------------------------------------------------------
template <class P> struct Fp {
    static constexpr int N = P::N;
    static constexpr bool HAS_MUL2 = P::p(P::N - 1) < 0x55555555u;   // 3p < R: the dual-product multiply applies
    uint32_t v[N];

    SB_HD static Fp zero() { Fp r;
_Pragma("unroll")
        for (int i = 0; i < N; i++) r.v[i] = 0;
        return r; }
    SB_HD static Fp one() { Fp r;
_Pragma("unroll")
        for (int i = 0; i < N; i++) r.v[i] = P::one(i);
        return r; }
    SB_HD static Fp r2() { Fp r;
_Pragma("unroll")
        for (int i = 0; i < N; i++) r.v[i] = P::r2(i);
        return r; }
    SB_HD bool is_zero() const { uint32_t o = 0;
_Pragma("unroll")
        for (int i = 0; i < N; i++) o |= v[i];
        return o == 0; }
    SB_HD bool operator==(const Fp& b) const { uint32_t o = 0;
_Pragma("unroll")
        for (int i = 0; i < N; i++) o |= v[i] ^ b.v[i];
        return o == 0; }

    // r = (x >= p) ? x - p : x      (x < 2p)
    SB_HD static void final_sub(uint32_t* x) {
        uint32_t d[N], bw;
        ptx::sub_cc(d[0], x[0], P::p(0));
_Pragma("unroll")
        for (int i = 1; i < N; i++) ptx::subc_cc(d[i], x[i], P::p(i));
        ptx::subc(bw, 0, 0);   // 0 if no borrow, 0xffffffff if borrow
_Pragma("unroll")
        for (int i = 0; i < N; i++) x[i] = bw ? x[i] : d[i];
    }

    // f1m_add (reference 2902-2920)
    SB_HD static Fp add(const Fp& a, const Fp& b) {
        Fp r;
        ptx::add_cc(r.v[0], a.v[0], b.v[0]);
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.v[i], a.v[i], b.v[i]);
        ptx::addc(r.v[N - 1], a.v[N - 1], b.v[N - 1]);   // p < 2^(32N-1): no carry out
        final_sub(r.v);
        return r;
    }
    SB_HD static Fp dbl(const Fp& a) { return add(a, a); }
    // f1m_sub (reference 2922-2936)
    SB_HD static Fp sub(const Fp& a, const Fp& b) {
        Fp r; uint32_t bw;
        ptx::sub_cc(r.v[0], a.v[0], b.v[0]);
_Pragma("unroll")
        for (int i = 1; i < N; i++) ptx::subc_cc(r.v[i], a.v[i], b.v[i]);
        ptx::subc(bw, 0, 0);
        ptx::add_cc(r.v[0], r.v[0], bw & P::p(0));
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.v[i], r.v[i], bw & P::p(i));
        ptx::addc(r.v[N - 1], r.v[N - 1], bw & P::p(N - 1));
        return r;
    }
    SB_HD static Fp neg(const Fp& a) {
        Fp r; uint32_t nz = a.is_zero() ? 0u : 0xffffffffu;
        ptx::sub_cc(r.v[0], nz & P::p(0), a.v[0]);
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::subc_cc(r.v[i], nz & P::p(i), a.v[i]);
        ptx::subc(r.v[N - 1], nz & P::p(N - 1), a.v[N - 1]);
        return r;
    }
    // conditional negate: (flag ? -a : a)
    SB_HD static Fp cneg(const Fp& a, bool flag) {
        Fp n = neg(a), r;
_Pragma("unroll")
        for (int i = 0; i < N; i++) r.v[i] = flag ? n.v[i] : a.v[i];
        return r;
    }

    // One CIOS row.  On entry X holds columns 0..N-1 with X[0] already cancelled by the previous
    // reduction, Y holds columns 1..N.  Shift one word right, add a*bi, add m*p.
    // On exit the roles are swapped: Y holds columns 0..N-1 with Y[0] cancelled, X holds columns 1..N.
    SB_HD static void row(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
        ptx::add_cc(Y[0], Y[0], X[1]);
_Pragma("unroll")
        for (int j = 0; j < N - 2; j += 2) {
            ptx::madc_lo_cc3(X[j], a[j + 1], bi, X[j + 2]);
            ptx::madc_hi_cc3(X[j + 1], a[j + 1], bi, X[j + 3]);
        }
        ptx::madc_lo_cc3(X[N - 2], a[N - 1], bi, 0);
        ptx::madc_hi3(X[N - 1], a[N - 1], bi, 0);
        ptx::mad_lo_cc(Y[0], a[0], bi);
        ptx::madc_hi_cc(Y[1], a[0], bi);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(Y[j], a[j], bi);
            ptx::madc_hi_cc(Y[j + 1], a[j], bi);
        }
        ptx::addc(X[N - 1], X[N - 1], 0);
        reduce(X, Y);
    }
    // m = Y[0]*np0 ; X += m*p_odd ; Y += m*p_even (Y[0] becomes 0)
    SB_HD static void reduce(uint32_t* X, uint32_t* Y) {
        uint32_t m = Y[0] * P::np0;
        ptx::mad_lo_cc(X[0], P::p(1), m);
        ptx::madc_hi_cc(X[1], P::p(1), m);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(X[j], P::p(j + 1), m);
            ptx::madc_hi_cc(X[j + 1], P::p(j + 1), m);
        }
        ptx::mad_lo_cc(Y[0], P::p(0), m);
        ptx::madc_hi_cc(Y[1], P::p(0), m);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(Y[j], P::p(j), m);
            ptx::madc_hi_cc(Y[j + 1], P::p(j), m);
        }
        ptx::addc(X[N - 1], X[N - 1], 0);
    }

    // f1m_mul (reference 3072-3273): a*b*R^-1 mod p, canonical.
    SB_HD static Fp mul(const Fp& a, const Fp& b) {
#if !defined(__CUDA_ARCH__) && !defined(SB_HOST_EMULATE_PTX)
        return host_mul(a, b);
#else
        uint32_t E[N], O[N];
_Pragma("unroll")
        for (int j = 0; j < N; j += 2) {
            E[j] = ptx::mul_lo(a.v[j], b.v[0]);     E[j + 1] = ptx::mul_hi(a.v[j], b.v[0]);
            O[j] = ptx::mul_lo(a.v[j + 1], b.v[0]); O[j + 1] = ptx::mul_hi(a.v[j + 1], b.v[0]);
        }
        reduce(O, E);
_Pragma("unroll")
        for (int i = 1; i < N; i += 2) {
            row(E, O, a.v, b.v[i]);
            if (i + 1 < N) row(O, E, a.v, b.v[i + 1]);
        }
        // N is even: the last row was row(E, O, ...): O holds columns 0..N-1 (O[0]==0), E holds columns 1..N
        Fp r;
        ptx::add_cc(r.v[0], E[0], O[1]);
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.v[i], E[i], O[i + 1]);
        ptx::addc(r.v[N - 1], E[N - 1], 0);
        final_sub(r.v);
        return r;
#endif
    }
    SB_HD static Fp sqr(const Fp& a) { return mul(a, a); }

    // Dual-product Montgomery multiply: (x*y + u*v) * R^-1 mod p with ONE interleaved reduction — 3N^2 wide MACs instead
    // of the 4N^2 of two multiplies.  Requires 3p < R so that the running sum (< 3p) fits N limbs; result < p(1 + 2p/R).
    SB_HD static void row2(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi, const uint32_t* u, uint32_t vi) {
        ptx::add_cc(Y[0], Y[0], X[1]);
_Pragma("unroll")
        for (int j = 0; j < N - 2; j += 2) {
            ptx::madc_lo_cc3(X[j], a[j + 1], bi, X[j + 2]);
            ptx::madc_hi_cc3(X[j + 1], a[j + 1], bi, X[j + 3]);
        }
        ptx::madc_lo_cc3(X[N - 2], a[N - 1], bi, 0);
        ptx::madc_hi3(X[N - 1], a[N - 1], bi, 0);
        ptx::mad_lo_cc(Y[0], a[0], bi);
        ptx::madc_hi_cc(Y[1], a[0], bi);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(Y[j], a[j], bi);
            ptx::madc_hi_cc(Y[j + 1], a[j], bi);
        }
        ptx::addc(X[N - 1], X[N - 1], 0);
        add_product(X, Y, u, vi);
        reduce(X, Y);
    }
    // X (columns 1..N) += u_odd * vi ; Y (columns 0..N-1) += u_even * vi, carry of Y into X[N-1]
    SB_HD static void add_product(uint32_t* X, uint32_t* Y, const uint32_t* u, uint32_t vi) {
        ptx::mad_lo_cc(X[0], u[1], vi);
        ptx::madc_hi_cc(X[1], u[1], vi);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(X[j], u[j + 1], vi);
            ptx::madc_hi_cc(X[j + 1], u[j + 1], vi);
        }
        ptx::mad_lo_cc(Y[0], u[0], vi);
        ptx::madc_hi_cc(Y[1], u[0], vi);
_Pragma("unroll")
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(Y[j], u[j], vi);
            ptx::madc_hi_cc(Y[j + 1], u[j], vi);
        }
        ptx::addc(X[N - 1], X[N - 1], 0);
    }
    SB_HD static Fp mul2(const Fp& x, const Fp& y, const Fp& u, const Fp& v) {
        static_assert(P::p(N - 1) < 0x55555555u, "mul2 needs 3p < R");
#if !defined(__CUDA_ARCH__) && !defined(SB_HOST_EMULATE_PTX)
        return add(host_mul(x, y), host_mul(u, v));
#else
        uint32_t E[N], O[N];
_Pragma("unroll")
        for (int j = 0; j < N; j += 2) {
            E[j] = ptx::mul_lo(x.v[j], y.v[0]);     E[j + 1] = ptx::mul_hi(x.v[j], y.v[0]);
            O[j] = ptx::mul_lo(x.v[j + 1], y.v[0]); O[j + 1] = ptx::mul_hi(x.v[j + 1], y.v[0]);
        }
        add_product(O, E, u.v, v.v[0]);
        reduce(O, E);
_Pragma("unroll")
        for (int i = 1; i < N; i += 2) {
            row2(E, O, x.v, y.v[i], u.v, v.v[i]);
            if (i + 1 < N) row2(O, E, x.v, y.v[i + 1], u.v, v.v[i + 1]);
        }
        Fp r;
        ptx::add_cc(r.v[0], E[0], O[1]);
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.v[i], E[i], O[i + 1]);
        ptx::addc(r.v[N - 1], E[N - 1], 0);
        final_sub(r.v);
        return r;
#endif
    }
    // ---- double-width product and stand-alone Montgomery reduction (for lazily reduced Fq2 arithmetic) -------------
    // T[0..2N) = a * b.  Two column-aligned accumulator arrays E (even columns) / O (O[k] = column k+1) as in mul();
    // every chain's carry-out lands in a limb that so far only holds earlier carry bits.  N^2 wide MACs.
    SB_HD static void mul_wide(const uint32_t* a, const uint32_t* b, uint32_t* T) {
        uint32_t E[2 * N], O[2 * N];
_Pragma("unroll")
        for (int k = 0; k < 2 * N; k++) { E[k] = 0; O[k] = 0; }
_Pragma("unroll")
        for (int i = 0; i < N; i++) {
            const uint32_t bi = b[i];
            if ((i & 1) == 0) {
                // even row: even j -> E[i+j], odd j -> O[i+j-1]
                ptx::mad_lo_cc(E[i], a[0], bi); ptx::madc_hi_cc(E[i + 1], a[0], bi);
_Pragma("unroll")
                for (int j = 2; j < N; j += 2) { ptx::madc_lo_cc(E[i + j], a[j], bi); ptx::madc_hi_cc(E[i + j + 1], a[j], bi); }
                ptx::addc(E[i + N], E[i + N], 0);
                ptx::mad_lo_cc(O[i], a[1], bi); ptx::madc_hi_cc(O[i + 1], a[1], bi);
_Pragma("unroll")
                for (int j = 3; j < N; j += 2) { ptx::madc_lo_cc(O[i + j - 1], a[j], bi); ptx::madc_hi_cc(O[i + j], a[j], bi); }
                ptx::addc(O[i + N], O[i + N], 0);
            } else {
                // odd row: odd j -> E[i+j], even j -> O[i+j-1]
                ptx::mad_lo_cc(E[i + 1], a[1], bi); ptx::madc_hi_cc(E[i + 2], a[1], bi);
_Pragma("unroll")
                for (int j = 3; j < N; j += 2) { ptx::madc_lo_cc(E[i + j], a[j], bi); ptx::madc_hi_cc(E[i + j + 1], a[j], bi); }
                if (i + N + 1 < 2 * N) ptx::addc(E[i + N + 1], E[i + N + 1], 0);
                ptx::mad_lo_cc(O[i - 1], a[0], bi); ptx::madc_hi_cc(O[i], a[0], bi);
_Pragma("unroll")
                for (int j = 2; j < N; j += 2) { ptx::madc_lo_cc(O[i + j - 1], a[j], bi); ptx::madc_hi_cc(O[i + j], a[j], bi); }
                ptx::addc(O[i + N - 1], O[i + N - 1], 0);
            }
        }
        T[0] = E[0];
        ptx::add_cc(T[1], E[1], O[0]);
_Pragma("unroll")
        for (int k = 2; k < 2 * N - 1; k++) ptx::addc_cc(T[k], E[k], O[k - 1]);
        ptx::addc(T[2 * N - 1], E[2 * N - 1], O[2 * N - 2]);
    }
    // one REDC step's shift: X (even columns, X[0] cancelled) / Y (odd columns) -> Y even, X odd, new top limb t enters
    SB_HD static void shift_in(uint32_t* X, uint32_t* Y, uint32_t t) {
        ptx::add_cc(Y[0], Y[0], X[1]);
_Pragma("unroll")
        for (int j = 0; j < N - 2; j++) ptx::addc_cc(X[j], X[j + 2], 0);
        ptx::addc_cc(X[N - 2], t, 0);
        ptx::addc(X[N - 1], 0, 0);
    }
    // T (2N limbs, T < p*R) -> T * R^-1 mod p, canonical.  N^2 wide MACs.
    SB_HD static Fp redc_wide(const uint32_t* T) {
        uint32_t E[N], O[N];
_Pragma("unroll")
        for (int k = 0; k < N; k++) { E[k] = T[k]; O[k] = 0; }
        reduce(O, E);
_Pragma("unroll")
        for (int i = 1; i < N; i += 2) {
            shift_in(E, O, T[N + i - 1]); reduce(E, O);
            if (i + 1 < N) { shift_in(O, E, T[N + i]); reduce(O, E); }
        }
        Fp r;
        ptx::add_cc(r.v[0], E[0], O[1]);
_Pragma("unroll")
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.v[i], E[i], O[i + 1]);
        ptx::addc(r.v[N - 1], E[N - 1], T[2 * N - 1]);
        final_sub(r.v);
        return r;
    }
    // 2N-limb helpers: x -= y (returns borrow mask), x += y, high half += p under mask
    SB_HD static uint32_t wide_sub(uint32_t* x, const uint32_t* y) {
        uint32_t bw;
        ptx::sub_cc(x[0], x[0], y[0]);
_Pragma("unroll")
        for (int k = 1; k < 2 * N; k++) ptx::subc_cc(x[k], x[k], y[k]);
        ptx::subc(bw, 0, 0);
        return bw;
    }
    SB_HD static void wide_add_p_high(uint32_t* x, uint32_t mask) {
        ptx::add_cc(x[N], x[N], mask & P::p(0));
_Pragma("unroll")
        for (int k = 1; k < N - 1; k++) ptx::addc_cc(x[N + k], x[N + k], mask & P::p(k));
        ptx::addc(x[2 * N - 1], x[2 * N - 1], mask & P::p(N - 1));
    }
    // plain N-limb sum without reduction (operands < p, p < 2^(32N-1))
    SB_HD static void add_noreduce(const Fp& a, const Fp& b, uint32_t* out) {
        ptx::add_cc(out[0], a.v[0], b.v[0]);
_Pragma("unroll")
        for (int k = 1; k < N - 1; k++) ptx::addc_cc(out[k], a.v[k], b.v[k]);
        ptx::addc(out[N - 1], a.v[N - 1], b.v[N - 1]);
    }

    // x*y + u*v for the hot loop: dual product where the modulus allows it, two multiplies otherwise
    SB_HD static Fp mul2_i(const Fp& x, const Fp& y, const Fp& u, const Fp& v) {
        if constexpr (P::p(N - 1) < 0x55555555u) return mul2(x, y, u, v);
        else return add(mul(x, y), mul(u, v));
    }
    SB_HD static Fp mul_i(const Fp& a, const Fp& b) { return mul(a, b); }
    SB_HD static Fp sqr_i(const Fp& a) { return mul(a, a); }
    // a*R mod p for any a < R, not only a < p: the conversion kernels take the caller's bytes unchecked.  The CIOS rows
    // multiply the first operand by one word of the second, and their running value stays below first + p; with
    // R^2 mod p first that is < 2p < R, while a first operand near R would carry out of the top limb.
    SB_HD static Fp to_mont(const Fp& a) { return mul(r2(), a); }

#ifndef __CUDA_ARCH__
    // Host-side multiply (final proof assembly, window Horner): plain word-serial Montgomery with 64-bit
    // accumulators.  Same canonical result as the device path.
    static inline Fp host_mul(const Fp& a, const Fp& b) {
        constexpr int M = N / 2;                       // 64-bit limbs
        typedef unsigned __int128 u128;
        uint64_t A[M], B[M], Pm[M], t[M + 2];
        for (int i = 0; i < M; i++) {
            A[i] = a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32);
            B[i] = b.v[2 * i] | ((uint64_t)b.v[2 * i + 1] << 32);
            Pm[i] = P::p(2 * i) | ((uint64_t)P::p(2 * i + 1) << 32);
        }
        for (int i = 0; i < M + 2; i++) t[i] = 0;
        uint64_t inv = (uint32_t)(0u - P::np0);        // p^-1 mod 2^32, one Newton step -> mod 2^64
        inv *= 2 - Pm[0] * inv;
        const uint64_t n0 = 0 - inv;
        for (int i = 0; i < M; i++) {
            u128 c = 0;
            for (int j = 0; j < M; j++) { c += (u128)A[j] * B[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
            c += t[M]; t[M] = (uint64_t)c; t[M + 1] = (uint64_t)(c >> 64);
            const uint64_t m = t[0] * n0;
            c = ((u128)m * Pm[0] + t[0]) >> 64;
            for (int j = 1; j < M; j++) { c += (u128)m * Pm[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
            c += t[M]; t[M - 1] = (uint64_t)c; t[M] = t[M + 1] + (uint64_t)(c >> 64);
        }
        bool ge = t[M] != 0;
        if (!ge) { ge = true; for (int i = M - 1; i >= 0; i--) { if (t[i] > Pm[i]) break; if (t[i] < Pm[i]) { ge = false; break; } } }
        if (ge) { u128 bw = 0; for (int i = 0; i < M; i++) { u128 d = (u128)t[i] - Pm[i] - bw; t[i] = (uint64_t)d; bw = (d >> 64) & 1; } }
        Fp r;
        for (int i = 0; i < M; i++) { r.v[2 * i] = (uint32_t)t[i]; r.v[2 * i + 1] = (uint32_t)(t[i] >> 32); }
        return r;
    }
#endif
    // a^e for a plain little-endian exponent of nw 32-bit words
    SB_HD static Fp pow(const Fp& a, const uint32_t* e, int nw) {
        Fp r = one();
        for (int i = nw * 32 - 1; i >= 0; i--) {
            r = sqr(r);
            if ((e[i >> 5] >> (i & 31)) & 1) r = mul(r, a);
        }
        return r;
    }
    // Inverse by Kaliski's "almost Montgomery inverse" (binary extended Euclid on plain limbs: shifts, adds and
    // compares only — ~15-20 k ALU instructions instead of the ~65 k IMAD-heavy ones of a^(p-2)).  Input and output in
    // Montgomery form; inverse of 0 is 0.  phase 1: r = a^-1 * 2^k (n <= k <= 2n), phase 2: 2n-k modular doublings
    // give a^-1 * 2^(2n) = (x R)^-1 * R^2 = x^-1 R for the Montgomery input a = x R.
    SB_HD static Fp inv_binary(const Fp& a) {
        if (a.is_zero()) return a;
        uint32_t u[N], v[N], r[N], s[N];
_Pragma("unroll")
        for (int i = 0; i < N; i++) { u[i] = P::p(i); v[i] = a.v[i]; r[i] = 0; s[i] = 0; }
        s[0] = 1;
        int k = 0;
        auto shr1 = [](uint32_t* x) {
_Pragma("unroll")
            for (int i = 0; i < N - 1; i++) x[i] = (x[i] >> 1) | (x[i + 1] << 31);
            x[N - 1] >>= 1; };
        auto shl1 = [](uint32_t* x) {
_Pragma("unroll")
            for (int i = N - 1; i > 0; i--) x[i] = (x[i] << 1) | (x[i - 1] >> 31);
            x[0] <<= 1; };
        auto sub = [](uint32_t* x, const uint32_t* y) { uint32_t bw = 0;
_Pragma("unroll")
            for (int i = 0; i < N; i++) { uint32_t xi = x[i], yi = y[i]; uint32_t d = xi - yi - bw; bw = (xi < yi) | ((xi == yi) & bw); x[i] = d; } };
        auto add = [](uint32_t* x, const uint32_t* y) { uint32_t c = 0;
_Pragma("unroll")
            for (int i = 0; i < N; i++) { uint32_t xi = x[i]; uint32_t t = xi + y[i]; uint32_t c1 = t < xi; uint32_t t2 = t + c; c = c1 | (t2 < t); x[i] = t2; } };
        auto gt = [](const uint32_t* x, const uint32_t* y) { bool g = false, decided = false;
_Pragma("unroll")
            for (int i = N - 1; i >= 0; i--) { bool ne = x[i] != y[i]; g = (!decided && ne) ? (x[i] > y[i]) : g; decided = decided || ne; }
            return g; };
        auto is0 = [](const uint32_t* x) { uint32_t o = 0;
_Pragma("unroll")
            for (int i = 0; i < N; i++) o |= x[i];
            return o == 0; };
        while (!is0(v)) {
            if (!(u[0] & 1)) { shr1(u); shl1(s); }
            else if (!(v[0] & 1)) { shr1(v); shl1(r); }
            else if (gt(u, v)) { sub(u, v); shr1(u); add(r, s); shl1(s); }
            else { sub(v, u); shr1(v); add(s, r); shl1(r); }
            k++;
        }
        uint32_t pp[N];
_Pragma("unroll")
        for (int i = 0; i < N; i++) pp[i] = P::p(i);
        if (!gt(pp, r)) sub(r, pp);             // r >= p
        sub(pp, r);                              // pp = p - r = a^-1 * 2^k mod p
        Fp o;
_Pragma("unroll")
        for (int i = 0; i < N; i++) o.v[i] = pp[i];
        // o * 2^(2n-k): one Montgomery multiply by 2^j in Montgomery form (j = 2n-k <= n), built by square-and-double
        const int j = 64 * N - k;
        Fp t = one();
        for (int bit = 9; bit >= 0; bit--) { t = sqr(t); if ((j >> bit) & 1) t = dbl(t); }
        return mul(o, t);
    }
    // inverse by Fermat (a^(p-2)); inverse of 0 is 0
    SB_HD static Fp inv(const Fp& a) {
        uint32_t e[N];
        uint32_t bw = 2;   // e = p - 2 with borrow propagation (BLS12-381 Fr has p(0) == 1)
        for (int i = 0; i < N; i++) { uint32_t pi = P::p(i); e[i] = pi - bw; bw = pi < bw ? 1u : 0u; }
        return pow(a, e, N);
    }

    // multiply by a plain little-endian constant 1 => fromMontgomery (reference 3595)
    SB_HD static Fp from_mont(const Fp& a) { Fp o = zero(); o.v[0] = 1; return mul(a, o); }
};

}  // namespace sb
