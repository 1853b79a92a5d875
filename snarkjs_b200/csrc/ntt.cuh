// ntt.cuh — radix-2 NTT/iNTT over Fr and the element-wise Fr kernels around it.
//
// Replaces ffjavascript engine_fft (_fft, reference build/snarkjs.js:14675-14918: JS bit-reverse
// 12640-12654 + per-chunk fftMix 8546-8666 + cross-chunk fftJoin 8089-8179 + fftFinal 8670-8772),
// engine_applykey (14268-14385 / 9315-9379), engine_batchconvert (12780-12830) and qap_joinABC
// (9174-9233).  Natural-order input, natural-order output, byte-identical results (every value is the
// canonical Montgomery residue).
//
// Formulation: Stockham autosort, log2(n) = sum of per-pass degrees.  After passes covering lgp bits,
//   Y[j*p + k] = sum_{m<p} x[j + m*(n/p)] * w_p^{mk}     (p = 2^lgp, j < n/p, k < p)
// so the bit-reversal permutation never exists as a separate step: it is absorbed into each pass's
// store addresses.  One pass of degree d (r = 2^d) does, per "index" = j'*p + k  (j' < n/(p r)):
//   u[a]   = Y[index + a*(n/r)] * w_{pr}^{a k}                      (a < r; twiddle = 2-level table product)
//   v      = DFT_r(u)                                               (d radix-2 DIF stages in shared memory)
//   Y'[((index-k) << d) + k + b*p] = v[b]
// A CTA owns a tile of C = 2^logc adjacent indices (C*32 B contiguous per row => coalesced loads and
// stores); the first pass (p = 1) stores transposed through an XOR-swizzled shared layout.
// Optional fusions: an element pre-multiplier c^i (coset shift = batchApplyKey with first = 1, optionally
// carrying the 1/n of a preceding unscaled inverse transform) on the first pass, and an output scale
// (1/n) on the last pass.
#pragma once
#include <cuda_runtime.h>
#include "fp.cuh"
#include "fr_entry.h"

namespace sb {

static constexpr int NTT_THREADS = 512;

template <class F> struct NttTables {
    // all device pointers
    const F* tw_lo = nullptr;  // w_n^e,           e < 2^h
    const F* tw_hi = nullptr;  // w_n^(e * 2^h),   e < 2^(L-h)
    int h = 0;
    const F* wr = nullptr;     // w_{2^DMAX}^j, j < 2^(DMAX-1)
};

template <class F> struct NttPre {   // element pre-multiplier c^i * scale by global input position i
    const F* lo = nullptr;     // c^e,                 e < 2^h
    const F* hi = nullptr;     // scale * c^(e * 2^h), e < 2^(L-h)
    int h = 0;
};

template <class F> __device__ __forceinline__ F lds_fe(const uint4* lo, const uint4* hi, uint32_t pos) {
    F x; uint4 a = lo[pos], b = hi[pos];
    x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
    return x;
}
template <class F> __device__ __forceinline__ void sts_fe(uint4* lo, uint4* hi, uint32_t pos, const F& x) {
    lo[pos] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
    hi[pos] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}
template <class F> __device__ __forceinline__ F ldg_fe(const F* p) {
    F x; const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
    return x;
}
template <class F> __device__ __forceinline__ void stg_fe(F* p, const F& x) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
    q[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}

// TMA 1-D bulk copies (cp.async.bulk, SASS UBLKCP) with an mbarrier transaction count: used to stage the in-tile twiddle
// table in shared memory once per CTA while the threads are busy with the global loads of the tile.
namespace tma {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// bytes: multiple of 16; dst / src 16-byte aligned.  Completion is signalled on `bar` (expect_tx issued here).
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
}  // namespace tma

static constexpr uint32_t NTT_WR_BYTES = (1u << (NTT_DMAX - 1)) * 32;   // the in-tile twiddle table w_{2^DMAX}^j, j < 2^(DMAX-1)
static constexpr size_t NTT_SMEM_EXTRA = NTT_WR_BYTES + 16;             // + the mbarrier

// One Stockham pass.  Fr has 8 limbs for both supported curves.
// several independent transforms of the same size per launch (blockIdx.y): Groth16 runs A, B and C together so that the
// grid fills whole waves (512 CTAs of one 2^20 pass are 1.15 waves at 3 CTAs/SM; 1536 are 3.46).  Up to 4 transforms
// anywhere in memory (stride = 0: in[y], out[y]), or any number of contiguous ones (stride = 2^L: in[0] + y * stride), the
// 3K transforms of a batch of K proofs.
template <class F> struct NttBatch { const F* in[4]; F* out[4]; uint64_t stride; };

// STRIDED selects the addressing at compile time, so the single-proof launches (stride 0) run the code they always ran.
template <class F, bool STRIDED>
__global__ void __launch_bounds__(NTT_THREADS)
k_ntt_pass(NttBatch<F> io, int L, int lgp, int deg, int logc,
           NttTables<F> tb, NttPre<F> pre, const F* __restrict__ post_scale) {
    const F* __restrict__ in = STRIDED ? io.in[0] + blockIdx.y * io.stride : io.in[blockIdx.y];
    F* __restrict__ out = STRIDED ? io.out[0] + blockIdx.y * io.stride : io.out[blockIdx.y];
    extern __shared__ uint4 ntt_smem[];
    const uint32_t r = 1u << deg, C = 1u << logc, tile = r << logc;
    uint4* slo = ntt_smem; uint4* shi = ntt_smem + tile;
    uint4* swr = ntt_smem + 2 * tile;                                      // staged copy of tb.wr (TMA bulk copy below)
    uint64_t* bar = reinterpret_cast<uint64_t*>(swr + NTT_WR_BYTES / 16);
    const uint32_t tid = threadIdx.x, T = blockDim.x;
    const bool use_wr = deg > 1;                                           // a radix-2 tile has no non-trivial in-tile twiddle
    if (use_wr && tid == 0) { tma::mbar_init(bar, 1); tma::bulk_g2s(swr, tb.wr, NTT_WR_BYTES, bar); }
    const uint64_t idx0 = (uint64_t)blockIdx.x << logc;
    const uint64_t stride = (1ull << L) >> deg;              // n / r
    const uint64_t pmask = (1ull << lgp) - 1;
    const int swz_shift = deg - logc;                        // swizzle: col ^= top logc bits of the row
    auto pos = [&](uint32_t a, uint32_t col) -> uint32_t { return (a << logc) + (col ^ ((a >> swz_shift) & (C - 1))); };

    // ---- load + twiddle
    for (uint32_t e = tid; e < tile; e += T) {
        uint32_t col = e & (C - 1), a = e >> logc;
        uint64_t index = idx0 + col;
        uint64_t src = index + (uint64_t)a * stride;
        F x = ldg_fe<F>(in + src);
        if (pre.lo) {
            F t = F::mul(ldg_fe<F>(pre.lo + (src & ((1ull << pre.h) - 1))), ldg_fe<F>(pre.hi + (src >> pre.h)));
            x = F::mul(x, t);
        }
        if (lgp) {
            uint64_t E = ((uint64_t)a * (index & pmask)) << (L - lgp - deg);
            if (E) {
                F t = F::mul(ldg_fe<F>(tb.tw_lo + (E & ((1ull << tb.h) - 1))), ldg_fe<F>(tb.tw_hi + (E >> tb.h)));
                x = F::mul(x, t);
            }
        }
        sts_fe<F>(slo, shi, pos(a, col), x);
    }
    __syncthreads();
    if (use_wr) tma::mbar_wait(bar, 0);                                    // the twiddle table has landed (it travelled during the loads above)
    // ---- deg radix-2 DIF stages
    const uint32_t nbf = tile >> 1;
    for (int rnd = 0; rnd < deg; rnd++) {
        const uint32_t bit = (r >> 1) >> rnd;
        for (uint32_t b = tid; b < nbf; b += T) {
            uint32_t col = b & (C - 1), i = b >> logc;
            uint32_t di = i & (bit - 1);
            uint32_t i0 = (i << 1) - di, i1 = i0 + bit;
            uint32_t p0 = pos(i0, col), p1 = pos(i1, col);
            F u0 = lds_fe<F>(slo, shi, p0), u1 = lds_fe<F>(slo, shi, p1);
            F s = F::add(u0, u1), d = F::sub(u0, u1);
            if (di) { const uint32_t wi = (di << rnd) << (NTT_DMAX - deg); d = F::mul(d, lds_fe<F>(swr, swr + 1, 2 * wi)); }
            sts_fe<F>(slo, shi, p0, s);
            sts_fe<F>(slo, shi, p1, d);
        }
        __syncthreads();
    }
    // ---- store (results sit at bit-reversed rows)
    F sc; if (post_scale) sc = ldg_fe<F>(post_scale);
    for (uint32_t e = tid; e < tile; e += T) {
        uint32_t col, b; uint64_t dst;
        if (lgp == 0) { b = e & (r - 1); col = e >> deg; dst = ((idx0 + col) << deg) + b; }
        else { col = e & (C - 1); b = e >> logc; uint64_t index = idx0 + col, k = index & pmask; dst = ((index - k) << deg) + k + ((uint64_t)b << lgp); }
        uint32_t rb = deg ? __brev(b) >> (32 - deg) : 0;                   // deg = 0: the one-element transform of n = 1
        F x = lds_fe<F>(slo, shi, pos(rb, col));
        if (post_scale) x = F::mul(x, sc);
        stg_fe<F>(out + dst, x);
    }
}

// out[i] = in[i] * lo[i & m] * hi[i >> h]     (batchApplyKey: first*inc^i split in two table levels)
template <class F>
__global__ void k_apply_key(const F* __restrict__ in, F* __restrict__ out, uint64_t n, NttPre<F> t) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    F k = F::mul(ldg_fe<F>(t.lo + (i & ((1ull << t.h) - 1))), ldg_fe<F>(t.hi + (i >> t.h)));
    stg_fe<F>(out + i, F::mul(ldg_fe<F>(in + i), k));
}
// frm_batchToMontgomery / frm_batchFromMontgomery
template <class F>
__global__ void k_convert(const F* __restrict__ in, F* __restrict__ out, uint64_t n, int to_mont) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x = ldg_fe<F>(in + i);
    stg_fe<F>(out + i, to_mont ? F::to_mont(x) : F::from_mont(x));
}
// qap_joinABC then frm_batchFromMontgomery (src/groth16_prove.js:320-374): out = fromMont(a*b - c)
template <class F>
__global__ void k_join_abc(const F* __restrict__ a, const F* __restrict__ b, const F* __restrict__ c, F* __restrict__ out, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x = F::sub(F::mul(ldg_fe<F>(a + i), ldg_fe<F>(b + i)), ldg_fe<F>(c + i));
    stg_fe<F>(out + i, F::from_mont(x));
}
// buildABC1 (src/groth16_prove.js:147-187) as a CSR sparse mat-vec: rows 0..n-1 -> A, n..2n-1 -> B;
// entry = (signal, coef*R^2); value = sum coef*R^2 (x) w[signal]  (Montgomery product with the plain
// witness gives a Montgomery result); C = A (x) B.  K proofs: witness k at witness + k*nw, its rows at A/B/C + k*n.
// BATCH = false is the single proof (K = 1): no proof index to divide out.
template <class F, bool BATCH>
__global__ void k_qap_rows(const uint64_t* __restrict__ row_ptr, const uint32_t* __restrict__ sig, const F* __restrict__ coef,
                           const F* __restrict__ witness, uint64_t nw, F* __restrict__ A, F* __restrict__ B, F* __restrict__ Cc,
                           uint64_t n, uint32_t K) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n * K) return;
    const uint64_t kp = BATCH ? i / n : 0, row = i - kp * n;
    const F* __restrict__ wk = witness + kp * nw;
    F acc[2];
#pragma unroll 1
    for (int m = 0; m < 2; m++) {
        F s = F::zero();
        uint64_t lo = row_ptr[m * n + row], hi = row_ptr[m * n + row + 1];
        for (uint64_t e = lo; e < hi; e++) s = F::add(s, F::mul(ldg_fe<F>(coef + e), ldg_fe<F>(wk + sig[e])));
        acc[m] = s;
    }
    stg_fe<F>(A + i, acc[0]); stg_fe<F>(B + i, acc[1]);
    stg_fe<F>(Cc + i, F::mul(acc[0], acc[1]));
}

// ------------------------------------------------------------------------------------------------
// host-side pass planning
// ------------------------------------------------------------------------------------------------
struct NttPlan { int npass; int deg[8]; int logc[8]; };

extern int g_ntt_tile_log;   // log2 of the largest tile (elements); 12 = 128 KiB smem (1 CTA/SM), 11 = 64 KiB (3 CTAs/SM)
inline NttPlan ntt_plan(int L) {
    NttPlan pl{};
    // n = 1 still takes one (degree-0) pass: it applies the pre-multiplier and the post-scale
    if (L <= NTT_DMAX) { pl.npass = 1; pl.deg[0] = L; pl.logc[0] = 0; return pl; }
    int np = (L + NTT_DMAX - 1) / NTT_DMAX;
    int base = L / np, rem = L % np;
    pl.npass = np;
    for (int i = 0; i < np; i++) {
        pl.deg[i] = base + (i < rem ? 1 : 0);
        int lc = g_ntt_tile_log - pl.deg[i]; if (lc > 3) lc = 3; if (lc < 0) lc = 0;
        if (lc > L - pl.deg[i]) lc = L - pl.deg[i];
        pl.logc[i] = lc;
    }
    return pl;
}

// Runs all passes over `count` transforms; a[i] holds input i, b[i] is its scratch; returns 0 if the results end
// in a[], 1 if in b[].  pre/post optional.  stride = 0: count <= 4 separate arrays; stride = 2^L: a[0] and b[0] hold
// `count` contiguous transforms each (count <= 65535, the grid's y limit).
template <class F>
int ntt_run_batch(F* const* a, F* const* b, int count, int L, const NttTables<F>& tb, const NttPre<F>* pre, const F* post_scale,
                  cudaStream_t stream, int* launches, uint64_t stride = 0) {
    NttPlan pl = ntt_plan(L);
    int lgp = 0, side = 0;
    for (int i = 0; i < pl.npass; i++) {
        int deg = pl.deg[i], logc = pl.logc[i];
        uint32_t tile = 1u << (deg + logc);
        size_t smem = (size_t)tile * 32 + NTT_SMEM_EXTRA;
        dim3 grid((unsigned)((1ull << L) >> (deg + logc)), (unsigned)count);
        unsigned threads = tile / 2 < (unsigned)NTT_THREADS ? (tile / 2 < 32 ? 32 : tile / 2) : NTT_THREADS;
        NttBatch<F> io;
        for (int k = 0; k < 4; k++) { int kk = (k < count && !stride) ? k : 0; io.in[k] = side ? b[kk] : a[kk]; io.out[k] = side ? a[kk] : b[kk]; }
        io.stride = stride;
        NttPre<F> p0; if (i == 0 && pre) p0 = *pre;
        if (stride) k_ntt_pass<F, true><<<grid, threads, smem, stream>>>(io, L, lgp, deg, logc, tb, p0, (i == pl.npass - 1) ? post_scale : nullptr);
        else k_ntt_pass<F, false><<<grid, threads, smem, stream>>>(io, L, lgp, deg, logc, tb, p0, (i == pl.npass - 1) ? post_scale : nullptr);
        if (launches) (*launches)++;
        lgp += deg; side ^= 1;
    }
    return side;
}

// Runs all passes; `a` holds the input, result ends in the returned pointer (a or b).  pre/post optional.
template <class F>
F* ntt_run(F* a, F* b, int L, const NttTables<F>& tb, const NttPre<F>* pre, const F* post_scale, cudaStream_t stream, int* launches) {
    F* aa[1] = {a}; F* bb[1] = {b};
    return ntt_run_batch<F>(aa, bb, 1, L, tb, pre, post_scale, stream, launches) ? b : a;
}
template <class F> inline cudaError_t ntt_configure() {
    cudaError_t e = cudaFuncSetAttribute(k_ntt_pass<F, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(128 * 1024 + NTT_SMEM_EXTRA));
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_ntt_pass<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(128 * 1024 + NTT_SMEM_EXTRA));
}

}  // namespace sb
