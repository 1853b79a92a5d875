// verify.cuh — batched Groth16 verification (src/groth16_verify.js:26-87) on the device pairing of pairing.cuh, templated on
// the base field.  One proof per thread, the Fq12 accumulator in registers.  Per call:
//   k_verify_prepare  thread 0 / 1: the Miller-loop lines of gamma2 / delta2 (shared by every proof, read from global memory
//                     by all threads of a warp at once); thread 2: the target conj(e(alpha1, beta2)) = e(alpha1, beta2)^-1
//   k_verify_terms    one thread per (proof, public input): s_i * IC[i+1] by gfft.cuh's per-thread scalar multiplication
//   k_verify          one thread per proof: the reference's checks in its order (public inputs < r, else status 2; A, B, C on
//                     their curves, else 3), cpub = IC[0] + sum of the proof's terms, one multi-Miller loop over (-A, B),
//                     (cpub, gamma2), (C, delta2), one final exponentiation, and the comparison with the target (0, else 1).
#pragma once
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif
#include "pairing.cuh"
#include "gfft.cuh"

namespace sb {

static constexpr int VERIFY_THREADS = 64;

template <class P> struct FrOf;
template <> struct FrOf<BnFq> { typedef BnFr T; };
template <> struct FrOf<BlsFq> { typedef BlsFr T; };

// a plain little-endian public signal below r
template <class P> SB_HD bool below_r(const FrPlain& s) {
    typedef typename FrOf<P>::T R;
    bool lt = false, decided = false;
_Pragma("unroll")
    for (int i = 7; i >= 0; i--) {
        const uint32_t p = R::p(i);
        lt = (!decided && s.v[i] != p) ? s.v[i] < p : lt;
        decided = decided || s.v[i] != p;
    }
    return lt;
}

// Verification-key layout (Montgomery affine, all zero = infinity), in Fq elements:
// alpha1 at 0, beta2 at 2, gamma2 at 6, delta2 at 10, IC[i] at 14 + 2i.
template <class P> struct VkView {
    const Fp<P>* e;
    SB_HD Fp2<P> g2x(int o) const { Fp2<P> r; r.a = e[o]; r.b = e[o + 1]; return r; }
    SB_HD Fp2<P> g2y(int o) const { Fp2<P> r; r.a = e[o + 2]; r.b = e[o + 3]; return r; }
    SB_HD bool g2_inf(int o) const { return g2x(o).is_zero() && g2y(o).is_zero(); }
    SB_HD bool g1_inf(int o) const { return e[o].is_zero() && e[o + 1].is_zero(); }
};

// every vk point is on its curve (or infinity), coordinates below q
template <class P> bool vk_valid_host(const Fp<P>* vk, uint32_t n_public) {
    typedef Pairing<P> T;
    VkView<P> v{vk};
    bool ok = T::g1_valid(vk[0], vk[1]);
    for (int o = 2; o <= 10; o += 4) ok = ok && T::g2_valid(v.g2x(o), v.g2y(o));
    for (uint32_t i = 0; i <= n_public; i++) ok = ok && T::g1_valid(vk[14 + 2 * i], vk[15 + 2 * i]);
    return ok;
}

#ifdef __CUDACC__   // kernels; the helpers above are shared with host builds
template <class P> __global__ void __launch_bounds__(VERIFY_THREADS)
k_pair_eval(int op, const Fp<P>* __restrict__ in, Fp<P>* __restrict__ out, uint64_t n, int wi, int wo) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pair_eval_record<P>(op, in + i * wi, out + i * wo);
}

template <class P> __global__ void k_verify_prepare(const Fp<P>* __restrict__ vk, PairLine<P>* __restrict__ lines,
                                                    Fq12<P>* __restrict__ target) {
    typedef Pairing<P> T;
    const VkView<P> v{vk};
    const int t = threadIdx.x;
    if (t < 2) {
        const int o = t ? 10 : 6;
        if (!v.g2_inf(o)) T::prepare(v.g2x(o), v.g2y(o), lines + t * T::NLINES);
    } else if (t == 2) {
        const bool live = !v.g1_inf(0) && !v.g2_inf(2);
        const Fq12<P> f = T::miller(vk[0], vk[1], v.g2x(2), v.g2y(2), live, vk[0], vk[1], nullptr, false, vk[0], vk[1], nullptr, false);
        *target = T::conj(T::final_exp(f));
    }
}

template <class P> __global__ void __launch_bounds__(GFFT_THREADS)
k_verify_terms(const Fp<P>* __restrict__ vk, const FrPlain* __restrict__ pubs, uint32_t n_public, uint64_t n, XYZZ<Fp<P>>* __restrict__ terms) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = (uint32_t)(t % n_public);
    const FrPlain s = pubs[t];
    XYZZ<Fp<P>> r = XYZZ<Fp<P>>::inf();
    if (below_r<P>(s)) r = gfft_mul<Fp<P>>(gfft_get<Fp<P>>((const uint8_t*)(vk + 14), 0, i + 1), s);
    terms[t] = r;
}

template <class P> __global__ void __launch_bounds__(VERIFY_THREADS)
k_verify(const Fp<P>* __restrict__ vk, uint32_t n_public, const PairLine<P>* __restrict__ lines, const Fq12<P>* __restrict__ target,
         const FrPlain* __restrict__ pubs, const Fp<P>* __restrict__ proofs, const XYZZ<Fp<P>>* __restrict__ terms,
         uint32_t count, int32_t* __restrict__ status) {
    typedef Pairing<P> T;
    typedef Fp<P> F;
    typedef Fp2<P> F2;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    bool ok = true;
    for (uint32_t i = 0; i < n_public; i++) ok = ok && below_r<P>(pubs[(uint64_t)k * n_public + i]);
    if (!ok) { status[k] = 2; return; }
    const F* pr = proofs + (uint64_t)k * 8;
    const F ax = pr[0], ay = pr[1], cx = pr[6], cy = pr[7];
    F2 bx, by; bx.a = pr[2]; bx.b = pr[3]; by.a = pr[4]; by.b = pr[5];
    if (!T::g1_valid(ax, ay) || !T::g2_valid(bx, by) || !T::g1_valid(cx, cy)) { status[k] = 3; return; }
    XYZZ<F> acc = gfft_get<F>((const uint8_t*)(vk + 14), 0, 0);
    for (uint32_t i = 0; i < n_public; i++) acc.add(terms[(uint64_t)k * n_public + i]);
    F px = F::zero(), py = F::zero();
    if (!acc.is_inf()) {
        const F t = F::inv_binary(acc.zzz), u = F::mul(acc.zz, t);
        px = F::mul(acc.x, F::sqr(u)); py = F::mul(acc.y, t);
    }
    const VkView<P> v{vk};
    const bool live0 = !(ax.is_zero() && ay.is_zero()) && !(bx.is_zero() && by.is_zero());
    const bool live1 = !acc.is_inf() && !v.g2_inf(6);
    const bool live2 = !(cx.is_zero() && cy.is_zero()) && !v.g2_inf(10);
    const Fq12<P> f = T::miller(ax, F::neg(ay), bx, by, live0, px, py, lines, live1, cx, cy, lines + T::NLINES, live2);
    status[k] = T::eq(T::final_exp(f), *target) ? 0 : 1;
}

#endif  // __CUDACC__

}  // namespace sb
