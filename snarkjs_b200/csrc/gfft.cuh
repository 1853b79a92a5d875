// gfft.cuh — group FFT and group batchApplyKey (G.fft / G.ifft / G.lagrangeEvaluations / G.batchApplyKey, reference
// build/snarkjs.js:14671-15176 and 14268-14385), templated on the coordinate field.
//
// Every butterfly of a group FFT multiplies a curve point by a full-width Fr twiddle, so the kernels are built around one
// per-thread variable-base scalar multiplication (gfft_mul: signed 4-bit fixed window, an 8-point table, 252 doublings
// and at most 64 additions in XYZZ coordinates).  The transform is radix-2 decimation in time:
//   k_gfft_load   affine or Jacobian bytes -> XYZZ at the bit-reversed index (all-zero affine / Z = 0 Jacobian = infinity)
//   k_gfft_stage  one stage per launch: t = w^j b; a' = a + t; b' = a - t (stage 0 has no multiplication)
//   k_gfft_store  natural order out; the inverse reads X[(n-k) mod n] and multiplies by n^-1 here, so it needs no pass
//                 of its own; normalised with one inversion per point (affine, or Jacobian with Z = 1, infinity (0,1,0))
// Twiddles and apply-key scalars are plain (non-Montgomery) little-endian Fr values below r < 2^255.
#pragma once
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif
#include "ec.cuh"

namespace sb {

static constexpr int GFFT_THREADS = 128;

struct FrPlain { uint32_t v[8]; };

#ifdef __CUDACC__   // the rest is device code; FrPlain is shared with host builds of the verifiers

// k * p for a plain scalar k < 2^255.  Digits d_i in [-7, 8] with k = sum d_i 16^i: a nibble plus the incoming carry
// above 8 becomes d - 16 and carries one; the top nibble is at most 7, so no digit 64 is needed.
template <class F> __device__ __noinline__ XYZZ<F> gfft_mul(const XYZZ<F>& p, const FrPlain& k) {
    XYZZ<F> tab[8];
    tab[0] = p;
    tab[1] = XYZZ<F>::dbl(p);
    for (int i = 2; i < 8; i++) { tab[i] = tab[i - 1]; tab[i].add(p); }
    int8_t dg[64];
    int carry = 0;
    for (int i = 0; i < 64; i++) {
        const int d = (int)((k.v[i >> 3] >> (4 * (i & 7))) & 15u) + carry;
        carry = d > 8;
        dg[i] = (int8_t)(d - 16 * carry);
    }
    XYZZ<F> r = XYZZ<F>::inf();
    for (int i = 63; i >= 0; i--) {
        for (int j = 0; j < 4; j++) r = XYZZ<F>::dbl(r);
        const int d = dg[i];
        if (d) {
            XYZZ<F> q = tab[(d < 0 ? -d : d) - 1];
            if (d < 0) q.y = F::neg(q.y);
            r.add(q);
        }
    }
    return r;
}

template <class F> __device__ __forceinline__ XYZZ<F> gfft_get(const uint8_t* in, int in_jac, uint64_t i) {
    XYZZ<F> p = XYZZ<F>::inf();
    if (in_jac) {
        const F* s = (const F*)(in + i * 3 * sizeof(F));
        const F z = s[2];
        if (!z.is_zero()) { p.x = s[0]; p.y = s[1]; p.zz = F::sqr(z); p.zzz = F::mul(p.zz, z); }
    } else {
        const F* s = (const F*)(in + i * 2 * sizeof(F));
        const F x = s[0], y = s[1];
        if (!(x.is_zero() & y.is_zero())) { p.x = x; p.y = y; p.zz = F::one(); p.zzz = F::one(); }
    }
    return p;
}

// x = X/ZZ, y = Y/ZZZ with the single inversion t = 1/ZZZ: ZZ^3 = ZZZ^2 gives 1/ZZ = (ZZ t)^2.
template <class F> __device__ __forceinline__ void gfft_put(const XYZZ<F>& p, int out_jac, uint8_t* out, uint64_t i) {
    F x, y;
    if (p.is_inf()) { x = F::zero(); y = out_jac ? F::one() : F::zero(); }
    else {
        const F t = F::inv(p.zzz), u = F::mul(p.zz, t);
        x = F::mul(p.x, F::sqr(u)); y = F::mul(p.y, t);
    }
    if (out_jac) {
        F* o = (F*)(out + i * 3 * sizeof(F));
        o[0] = x; o[1] = y; o[2] = p.is_inf() ? F::zero() : F::one();
    } else {
        F* o = (F*)(out + i * 2 * sizeof(F));
        o[0] = x; o[1] = y;
    }
}

template <class F> __global__ void __launch_bounds__(GFFT_THREADS)
k_gfft_load(const uint8_t* __restrict__ in, int in_jac, uint64_t n, int L, XYZZ<F>* __restrict__ pts) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t j = L ? (__brevll(i) >> (64 - L)) : 0;
    pts[j] = gfft_get<F>(in, in_jac, i);
}

// stage s (0-based): butterflies of span 2^s, twiddle w_{2^(s+1)}^j = w_n^(j 2^(L-1-s)) from the table of w_n^j, j < n/2
template <class F> __global__ void __launch_bounds__(GFFT_THREADS)
k_gfft_stage(XYZZ<F>* __restrict__ pts, const FrPlain* __restrict__ tw, uint64_t n, int L, int s) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n / 2) return;
    const uint64_t half = 1ull << s, j = t & (half - 1);
    const uint64_t i0 = ((t >> s) << (s + 1)) + j, i1 = i0 + half;
    const XYZZ<F> a = pts[i0];
    XYZZ<F> b = pts[i1];
    if (s) b = gfft_mul<F>(b, tw[j << (L - 1 - s)]);
    XYZZ<F> u = a; u.add(b);
    b.y = F::neg(b.y);
    XYZZ<F> v = a; v.add(b);
    pts[i0] = u; pts[i1] = v;
}

template <class F> __global__ void __launch_bounds__(GFFT_THREADS)
k_gfft_store(const XYZZ<F>* __restrict__ pts, uint64_t n, const FrPlain* __restrict__ ninv, int out_jac, uint8_t* __restrict__ out) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    XYZZ<F> p = pts[ninv ? ((n - k) & (n - 1)) : k];
    if (ninv) p = gfft_mul<F>(p, *ninv);
    gfft_put<F>(p, out_jac, out, k);
}

// out[i] = in[i] * sc[i]
template <class F> __global__ void __launch_bounds__(GFFT_THREADS)
k_gapply(const uint8_t* __restrict__ in, int in_jac, const FrPlain* __restrict__ sc, uint64_t n, int out_jac, uint8_t* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    gfft_put<F>(gfft_mul<F>(gfft_get<F>(in, in_jac, i), sc[i]), out_jac, out, i);
}

inline unsigned gfft_blocks(uint64_t n) { return (unsigned)((n + GFFT_THREADS - 1) / GFFT_THREADS); }

// the whole transform of n = 2^L points on `stream`: d_pts = scratch of n XYZZ points; ninv = null for the forward one
template <class F> int gfft_run(const uint8_t* d_in, int in_jac, uint64_t n, int L, const FrPlain* d_tw, const FrPlain* d_ninv,
                                int out_jac, XYZZ<F>* d_pts, uint8_t* d_out, cudaStream_t stream, int* launches) {
    k_gfft_load<F><<<gfft_blocks(n), GFFT_THREADS, 0, stream>>>(d_in, in_jac, n, L, d_pts);
    for (int s = 0; s < L; s++) k_gfft_stage<F><<<gfft_blocks(n / 2), GFFT_THREADS, 0, stream>>>(d_pts, d_tw, n, L, s);
    k_gfft_store<F><<<gfft_blocks(n), GFFT_THREADS, 0, stream>>>(d_pts, n, d_ninv, out_jac, d_out);
    *launches = L + 2;
    return (int)cudaGetLastError();
}

#endif  // __CUDACC__

}  // namespace sb
