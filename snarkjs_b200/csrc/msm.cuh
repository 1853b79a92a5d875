// msm.cuh — Pippenger multi-scalar multiplication on one GPU (templated on the coordinate field).
//
// Replaces ffjavascript engine_multiexp (_multiExp/_multiExpChunk, reference build/snarkjs.js:14517-14669)
// and wasmcurves build_multiexp (g?m_multiexpAffine_chunk 5542-5695, _getChunk 5471-5540,
// _reduceTable 5819-5907).  The reference runs one task per (point-chunk, window), each re-copying its
// chunk; here all windows are processed in one pass over the scalars:
//
//   k_digits      scalars -> signed c-bit digits; one (key = window*B + |d|-1, val = index | sign<<31)
//                 entry per non-zero digit   (B = 2^(c-1) buckets per window)
//   radix sort    entries by key (cub::DeviceRadixSort, library plumbing)
//   k_accumulate  balanced segmented bucket accumulation: every thread owns SEG consecutive sorted
//                 entries regardless of bucket sizes (robust to witness-like skew: many 0/1 scalars),
//                 gathers affine bases with 128-bit loads, XYZZ mixed adds; a run that starts inside
//                 the segment is written straight to its bucket, the thread's first run goes to a
//                 "head" partial that the next (32x smaller) level folds in.
//   k_fold        same segmented walk over the head partials (full XYZZ adds) until one thread is left
//   k_reduce      per window sum_b (b+1)*bucket[b] by chunked running sums + small scalar multiply,
//                 then a shared-memory tree to one point per window
//   host          Horner over the W window sums (W*c doublings on 1 point: latency-bound, CPU is faster)
#pragma once
#include <cuda_runtime.h>
#include "ec.cuh"
#include "msm_geom.h"

namespace sb {

static constexpr int MSM_SEG = 32;          // sorted entries per thread in k_accumulate / k_fold
static constexpr int MSM_ACC_THREADS = 128;
static constexpr int MSM_RED_CHUNK = 16;    // buckets per thread in k_reduce
static constexpr uint32_t MSM_INVALID_KEY = 0xffffffffu;
static constexpr int MSM_COUNTS_SEG = 8;      // counts[8]: sorted entries per k_accumulate thread (counts[0] = valid entries, [1..7] = fold level sizes)

// sb_set_tuning(13, c): window bits (3..22) that msm_choose and msm_geometry_precomp return instead of their own choice
// (test hook; 0 = the heuristics below)
extern int g_msm_force_c;

// Window-size choice.  Cost model: W_eff*n mixed adds (10 modmul) + one pass over the buckets (~60 modmul each);
// buckets = 2^(c-1) per window, shared by all windows in the precomputed-table mode.  `fr_bits` is the bit length of
// the scalar field (254 / 255): field-element scalars leave the windows above it empty, and the top *occupied* window
// only has top_bits = fr_bits + 1 - (W_eff-1)*c significant bits, i.e. it funnels all n terms into 2^top_bits buckets.
// Candidates whose top window is more than 32x denser than the others are skipped (giant buckets are handled
// correctly by the fold cascade, but cost latency-bound milliseconds).  W itself always covers 8*scalar_bytes + 1 bits,
// so arbitrary scalars (the reference accepts any value < 2^(8*sScalar)) stay correct.
__host__ inline MsmGeom msm_choose(uint64_t n, uint32_t scalar_bytes, int fr_bits, bool precomp) {
    int eff = (int)(8 * scalar_bytes) < fr_bits ? (int)(8 * scalar_bytes) : fr_bits;
    int best_c = 3; double best = 1e300;
    for (int c = 3; c <= 22; c++) {
        int weff = (eff + 1 + c - 1) / c, top = eff + 1 - (weff - 1) * c;
        if (weff > 1 && top < c - 5) continue;
        double buckets = (precomp ? 1.0 : (double)weff) * (double)(1u << (c - 1));
        double cost = (double)weff * (double)n * 10.0 + buckets * 60.0;
        if (cost < best) { best = cost; best_c = c; }
    }
    if (g_msm_force_c) best_c = g_msm_force_c;
    MsmGeom g; g.c = best_c; g.W = (int)((8 * scalar_bytes + 1 + best_c - 1) / best_c); g.B = 1u << (best_c - 1);
    return g;
}
// Precomputed-window mode (tables cover 32-byte scalars): all windows share one bucket set, so the bucket pass is
// cheap and what matters is the number of windows: take the largest c (fewest windows) that keeps the top window's
// density within 32x of the others and leaves on average >= ~W entries per bucket (2^(c-1) <= n).  Sparse buckets
// (a few dozen entries) also keep the per-thread head partials short-run, i.e. on the parallel k_fold_short path.
__host__ inline MsmGeom msm_geometry_precomp(uint64_t n_set, uint32_t scalar_bytes, int fr_bits = 254) {
    int l2 = 0; while ((1ull << (l2 + 1)) <= n_set) l2++;
    int cmax = l2; if (cmax > 22) cmax = 22; if (cmax < 8) cmax = 8;   // 2^(c-1) <= n/2: the bucket pass (1.3 ns/bucket) stays below ~1/3 of the accumulation (0.16 ns/entry)
    int c = 8;
    for (int cc = cmax; cc >= 8; cc--) {
        int weff = (fr_bits + 1 + cc - 1) / cc, top = fr_bits + 1 - (weff - 1) * cc;
        if (weff > 1 && top < cc - 5) continue;
        c = cc; break;
    }
    if (g_msm_force_c) c = g_msm_force_c;
    MsmGeom g; g.c = c; g.W = (int)((8 * scalar_bytes + 1 + c - 1) / c); g.B = 1u << (c - 1);
    g.precomp = 1; g.stride = n_set; g.first = 0;
    return g;
}
__host__ inline MsmGeom msm_geometry(uint64_t n, uint32_t scalar_bytes, int fr_bits = 254) {
    return msm_choose(n, scalar_bytes, fr_bits, false);
}

template <class F> __device__ __forceinline__ void load_affine(const Affine<F>* __restrict__ bases, uint32_t idx, F& x, F& y) {
    constexpr int NV = sizeof(F) / 16;
    const uint4* p = reinterpret_cast<const uint4*>(bases + idx);
    uint4* dx = reinterpret_cast<uint4*>(&x);
    uint4* dy = reinterpret_cast<uint4*>(&y);
#pragma unroll
    for (int k = 0; k < NV; k++) dx[k] = __ldg(p + k);
#pragma unroll
    for (int k = 0; k < NV; k++) dy[k] = __ldg(p + NV + k);
}
template <class T> __device__ __forceinline__ void store_vec(T* dst, const T& v) {
    constexpr int NV = sizeof(T) / 16;
    const uint4* s = reinterpret_cast<const uint4*>(&v);
    uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int k = 0; k < NV; k++) d[k] = s[k];
}
template <class T> __device__ __forceinline__ T load_vec(const T* src) {
    constexpr int NV = sizeof(T) / 16;
    T v; const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(&v);
#pragma unroll
    for (int k = 0; k < NV; k++) d[k] = s[k];
    return v;
}

// field inversion on the device: binary (Kaliski) for Fp, norm + binary for Fp2
template <class P> __device__ __forceinline__ Fp<P> PairInvF(const Fp<P>& a) { return Fp<P>::inv_binary(a); }
template <class P> __device__ __forceinline__ Fp2<P> PairInvF(const Fp2<P>& a) { return Fp2<P>::inv(a); }

// ------------------------------------------------------------------------------------------------
// level 0: affine bases gathered through the sorted (key, val) list
// ------------------------------------------------------------------------------------------------
template <class F, int MINB>
__global__ void __launch_bounds__(MSM_ACC_THREADS, MINB)
k_accumulate(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
             const uint64_t* __restrict__ counts, XYZZ<F>* __restrict__ buckets,
             XYZZ<F>* __restrict__ heads, uint32_t* __restrict__ head_keys) {
    const uint64_t M = counts[0];
    const uint32_t seg = (uint32_t)counts[MSM_COUNTS_SEG];          // entries per thread, fitted to whole waves by k_count_valid
    uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint64_t lo = t * seg;
    if (lo >= M) return;
    uint64_t hi = lo + seg < M ? lo + seg : M;
    const F one = F::one();
    XYZZ<F> acc = XYZZ<F>::inf();
    uint32_t cur = keys[lo];
    bool first = true;
    for (uint64_t e = lo; e < hi; e++) {
        uint32_t k = keys[e], v = vals ? vals[e] : (uint32_t)e;
        if (k != cur) {
            if (first) { store_vec(heads + t, acc); head_keys[t] = cur; first = false; }
            else store_vec(buckets + cur, acc);
            acc = XYZZ<F>::inf(); cur = k;
        }
        F px, py;
        load_affine<F>(bases, v & 0x7fffffffu, px, py);
        if (!(px.is_zero() & py.is_zero())) {          // base at infinity contributes nothing (reference 6068-6086)
            py = F::cneg(py, (v >> 31) != 0);
            acc.add_affine(px, py, one);
        }
    }
    if (first) { store_vec(heads + t, acc); head_keys[t] = cur; }
    else store_vec(buckets + cur, acc);
}

// ------------------------------------------------------------------------------------------------
// level 1 fast path: one thread per head partial.  Heads are sorted by key; a run of equal keys of length
// <= MSM_SHORT_RUN is summed by its first thread and added to the bucket (for uniform scalars practically every
// run has length 1, so this is one fully parallel read-modify-write per head).  Heads consumed here are marked
// INVALID in keys_out; longer runs (skewed scalars: giant buckets) keep their key and go to the k_fold cascade.
// ------------------------------------------------------------------------------------------------
static constexpr int MSM_SHORT_RUN = 8;
template <class F, int MINB>
__global__ void __launch_bounds__(MSM_ACC_THREADS, MINB)
k_fold_short(const XYZZ<F>* __restrict__ heads, const uint32_t* __restrict__ keys_in, uint32_t* __restrict__ keys_out,
             const uint64_t* __restrict__ counts, XYZZ<F>* __restrict__ buckets) {
    const uint64_t M = counts[1];
    uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= M) return;
    const uint32_t k = keys_in[t];
    // locate the start of my run (looking back at most MSM_SHORT_RUN entries)
    uint64_t start = t; int back = 0;
    while (start > 0 && back < MSM_SHORT_RUN && keys_in[start - 1] == k) { start--; back++; }
    bool is_short = back < MSM_SHORT_RUN;
    uint64_t len = 0;
    if (is_short) {
        len = 1;
        while (start + len < M && len <= (uint64_t)MSM_SHORT_RUN && keys_in[start + len] == k) len++;
        is_short = len <= (uint64_t)MSM_SHORT_RUN;
    }
    keys_out[t] = is_short ? MSM_INVALID_KEY : k;
    if (!is_short || start != t) return;
    XYZZ<F> acc = load_vec(buckets + k);
    for (uint64_t e = 0; e < len; e++) { XYZZ<F> p = load_vec(heads + t + e); acc.add_i(p); }
    store_vec(buckets + k, acc);
}

// ------------------------------------------------------------------------------------------------
// level >= 1 cascade: fold the remaining head partials (sorted by key, INVALID = already consumed).
// `last` = single-thread final level.
// ------------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(MSM_ACC_THREADS)
k_fold(const XYZZ<F>* __restrict__ in, const uint32_t* __restrict__ in_keys, const uint64_t* __restrict__ counts, int level,
       XYZZ<F>* __restrict__ buckets, XYZZ<F>* __restrict__ heads, uint32_t* __restrict__ head_keys) {
    const uint64_t M = counts[level];
    const bool last = M <= MSM_SEG;
    uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint64_t lo = t * MSM_SEG;
    if (lo >= M) return;
    uint64_t hi = lo + MSM_SEG < M ? lo + MSM_SEG : M;
    XYZZ<F> acc = XYZZ<F>::inf();
    uint32_t cur = in_keys[lo];
    bool first = !last;
    auto flush = [&]() __attribute__((always_inline)) {
        if (first) { store_vec(heads + t, acc); head_keys[t] = cur; first = false; }
        else if (cur != MSM_INVALID_KEY) { XYZZ<F> b = load_vec(buckets + cur); b.add_i(acc); store_vec(buckets + cur, b); }
    };
    for (uint64_t e = lo; e < hi; e++) {
        uint32_t k = in_keys[e];
        if (k != cur) { flush(); acc = XYZZ<F>::inf(); cur = k; }
        if (k != MSM_INVALID_KEY) { XYZZ<F> p = load_vec(in + e); acc.add_i(p); }
    }
    flush();
}

// ------------------------------------------------------------------------------------------------
// bucket reduction.  Thread (w, j) owns buckets [j*L, (j+1)*L) of window w:
//   run = sum bucket[b],  sum = sum (b - j*L + 1) * bucket[b]   (running sums, reference _reduceTable
//   computes the same weighted sum by recursive halving), partial = sum + (j*L) * run.
// Then a shared-memory tree adds the partials of one CTA; CTAs of a window write to partials[w][cta].
// ------------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(128)
k_reduce(const XYZZ<F>* __restrict__ buckets, MsmGeom g, XYZZ<F>* __restrict__ partials, uint32_t ctas_per_window) {
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* sm = reinterpret_cast<XYZZ<F>*>(smem_raw);
    const uint32_t w = blockIdx.x / ctas_per_window, cta = blockIdx.x % ctas_per_window;
    const uint32_t L = g.B < (uint32_t)MSM_RED_CHUNK ? g.B : MSM_RED_CHUNK;
    const uint32_t chunks = g.B / L;
    const uint32_t j = cta * blockDim.x + threadIdx.x;
    XYZZ<F> part = XYZZ<F>::inf();
    if (j < chunks) {
        const XYZZ<F>* bk = buckets + (uint64_t)w * g.B + (uint64_t)j * L;
        XYZZ<F> run = XYZZ<F>::inf(), sum = XYZZ<F>::inf();
        for (int b = (int)L - 1; b >= 0; b--) {
            XYZZ<F> p = load_vec(bk + b);
            run.add_i(p);
            sum.add_i(run);
        }
        // part = sum + (j*L) * run   (double-and-add, MSB first)
        uint32_t k = j * L;
        if (k) {
            int top = 31 - __clz(k);
            part = run;
            for (int bit = top - 1; bit >= 0; bit--) {
                part = XYZZ<F>::dbl(part);
                if ((k >> bit) & 1) part.add_i(run);
            }
        }
        part.add_i(sum);
    }
    store_vec(sm + threadIdx.x, part);
    __syncthreads();
    for (uint32_t s = blockDim.x >> 1; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            XYZZ<F> a = load_vec(sm + threadIdx.x), b = load_vec(sm + threadIdx.x + s);
            a.add_i(b);
            store_vec(sm + threadIdx.x, a);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) store_vec(partials + (uint64_t)w * ctas_per_window + cta, load_vec(sm));
}

// one warp per window: lanes stride over the per-CTA partials of k_reduce, then a shared-memory tree
template <class F>
__global__ void __launch_bounds__(32)
k_window_sum(const XYZZ<F>* __restrict__ partials, uint32_t per_window, XYZZ<F>* __restrict__ out) {
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* sm = reinterpret_cast<XYZZ<F>*>(smem_raw);
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t i = threadIdx.x; i < per_window; i += 32) { XYZZ<F> p = load_vec(partials + (uint64_t)blockIdx.x * per_window + i); acc.add_i(p); }
    store_vec(sm + threadIdx.x, acc);
    __syncwarp();
    for (uint32_t s = 16; s > 0; s >>= 1) {
        if (threadIdx.x < s) { XYZZ<F> a = load_vec(sm + threadIdx.x), b = load_vec(sm + threadIdx.x + s); a.add_i(b); store_vec(sm + threadIdx.x, a); }
        __syncwarp();
    }
    if (threadIdx.x == 0) store_vec(out + blockIdx.x, load_vec(sm));
}

// ------------------------------------------------------------------------------------------------
// Bucket reduction, second design (default): axis sums + warp-shuffle weighted sums.
//
// The window sum  sum_b (b+1) * bucket[b]  is  T + sum_b b * bucket[b]  with T = sum of all buckets.  Write the bucket
// index as b = hi * 2^m + lo (a matrix of H rows by 2^m columns); with the row sums R_hi and the column sums C_lo
//     sum_b b * bucket[b] = 2^m * sum_hi hi * R_hi + sum_lo lo * C_lo,        T = sum_lo C_lo.
// Every bucket is added once into a row sum and once into a column sum (2 additions per bucket, the same count as the
// running-sum recursion of the reference's _reduceTable 5819-5907 or of k_reduce above), but the additions form plain
// trees: no per-thread scalar multiply and 4x the threads of k_reduce at the first level.
//   k_axis_sum   out[o][i] = sum_{s<S} in[o][s][i]  (S <= 8 per level; rows and columns of one level in one launch:
//                the row job views its rows as [S][len/S] so that both jobs read coalesced 128 B .. 4 KiB runs)
//   k_ws_chunks  one warp per 32 entries of R / C: lane l holds v_l; a shuffle suffix scan gives the suffix sums, their
//                shuffle-tree sum is sum_l l*v_l (weighted) and the first suffix sum is the plain total
//   k_ws_final   one CTA per window: the same warp routine over the chunk totals, then the power-of-two weights
//                (2^m, 2^5) by doublings of single points.
// ------------------------------------------------------------------------------------------------

struct AxisJob { const void* in; void* out; uint64_t total; uint32_t S; uint32_t log_inner; };

template <class F, int MINB>
__global__ void __launch_bounds__(128, MINB)
k_axis_sum(AxisJob j0, AxisJob j1) {
    const AxisJob j = blockIdx.y ? j1 : j0;
    const uint64_t gid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (gid >= j.total) return;
    const uint64_t o = gid >> j.log_inner, i = gid & ((1ull << j.log_inner) - 1);
    const XYZZ<F>* p = (const XYZZ<F>*)j.in + ((o * j.S) << j.log_inner) + i;
    XYZZ<F> acc = load_vec(p);
#pragma unroll 1
    for (uint32_t s = 1; s < j.S; s++) { XYZZ<F> v = load_vec(p + ((uint64_t)s << j.log_inner)); acc.add_i(v); }
    store_vec((XYZZ<F>*)j.out + gid, acc);
}

template <class F> __device__ __forceinline__ XYZZ<F> shfl_down_pt(const XYZZ<F>& v, int d) {
    constexpr int NW32 = sizeof(XYZZ<F>) / 4;
    union U { XYZZ<F> p; uint32_t w[NW32]; __device__ U() {} };
    U a, r; a.p = v;
#pragma unroll
    for (int k = 0; k < NW32; k++) r.w[k] = __shfl_down_sync(0xffffffffu, a.w[k], d);
    return r.p;
}
// lane l holds v_l.  Lane 0 receives T = sum_l v_l and W = sum_l l * v_l (all 32 lanes must call).
template <class F> __device__ __forceinline__ void warp_weighted_sum(XYZZ<F> v, XYZZ<F>& T, XYZZ<F>& W) {
    const int lane = threadIdx.x & 31;
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) { XYZZ<F> o = shfl_down_pt<F>(v, d); if (lane + d < 32) v.add_i(o); }   // suffix sums
    T = v;
    XYZZ<F> x = lane ? v : XYZZ<F>::inf();
#pragma unroll 1
    for (int d = 16; d >= 1; d >>= 1) { XYZZ<F> o = shfl_down_pt<F>(x, d); if (lane < d) x.add_i(o); }
    W = x;
}
template <class F> __device__ __forceinline__ XYZZ<F> warp_sum(XYZZ<F> x) {
    const int lane = threadIdx.x & 31;
#pragma unroll 1
    for (int d = 16; d >= 1; d >>= 1) { XYZZ<F> o = shfl_down_pt<F>(x, d); if (lane < d) x.add_i(o); }
    return x;
}

// vecR: [NW][lenR] (may be null / lenR = 0), vecC: [NW][lenC].  tw: [NW][nR + nC][2] = (T, W) of every 32-entry chunk.
template <class F>
__global__ void __launch_bounds__(128)
k_ws_chunks(const XYZZ<F>* __restrict__ vecR, uint32_t lenR, const XYZZ<F>* __restrict__ vecC, uint32_t lenC, uint32_t NW, XYZZ<F>* __restrict__ tw) {
    const uint32_t nR = (lenR + 31) / 32, nC = (lenC + 31) / 32, per = nR + nC;
    const uint32_t wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (wid >= NW * per) return;
    const uint32_t w = wid / per, jj = wid % per;
    const bool isR = jj < nR;
    const uint32_t j = isR ? jj : jj - nR, len = isR ? lenR : lenC, idx = j * 32 + lane;
    const XYZZ<F>* vec = (isR ? vecR : vecC) + (uint64_t)w * len;
    XYZZ<F> v = XYZZ<F>::inf();
    if (idx < len) v = load_vec(vec + idx);
    XYZZ<F> T, W;
    warp_weighted_sum<F>(v, T, W);
    if (lane == 0) { store_vec(tw + 2 * (uint64_t)wid, T); store_vec(tw + 2 * (uint64_t)wid + 1, W); }
}

// window sum = 2^(m+5) * a0 + 2^m * a1 + 2^5 * a2 + a3 + a4 with (chunk index j)
//   a0 = sum_j j * T^R_j,  a1 = sum_j W^R_j,  a2 = sum_j j * T^C_j,  a3 = sum_j W^C_j,  a4 = sum_j T^C_j (= all buckets).
// One CTA of four warps per window writes the five parts out[5 w + k]; the power-of-two weights (m + 10 doublings of single
// points: pure latency here) are applied by the host (msm_group.inl combine).
template <class F>
__global__ void __launch_bounds__(128)
k_ws_final(const XYZZ<F>* __restrict__ tw, uint32_t nR, uint32_t nC, XYZZ<F>* __restrict__ out) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, per = nR + nC;
    const XYZZ<F>* base = tw + 2 * (uint64_t)blockIdx.x * per;
    const bool r_side = warp < 2;
    const uint32_t cnt = r_side ? nR : nC, off = r_side ? 0 : nR;
    XYZZ<F> v = XYZZ<F>::inf();
    if (lane < cnt) v = load_vec(base + 2 * (uint64_t)(off + lane) + (warp & 1));   // even warps: T entries, odd warps: W entries
    XYZZ<F>* o = out + 5 * (uint64_t)blockIdx.x;
    if ((warp & 1) == 0) {
        XYZZ<F> tot, res;
        warp_weighted_sum<F>(v, tot, res);
        if (lane == 0) { store_vec(o + (r_side ? 0 : 2), res); if (!r_side) store_vec(o + 4, tot); }
    } else {
        XYZZ<F> res = warp_sum<F>(v);
        if (lane == 0) store_vec(o + (r_side ? 1 : 3), res);
    }
}

// One warp per output: out[o][i] = sum_{s<S} in[o][s][i], S <= 128: lane l adds s = l, l + 32, ... and a shuffle tree joins
// the lanes.  Used for everything the first axis-sum level leaves (2^16 partials per chain at 2^19 buckets): the work is
// negligible there and the latency (<= 3 + 5 dependent additions) is what counts.
template <class F>
__global__ void __launch_bounds__(128)
k_axis_tree(AxisJob j0, AxisJob j1) {
    const AxisJob j = blockIdx.y ? j1 : j0;
    const uint64_t wid = blockIdx.x * (uint64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint32_t lane = threadIdx.x & 31;
    if (wid >= j.total) return;
    const uint64_t o = wid >> j.log_inner, i = wid & ((1ull << j.log_inner) - 1);
    const XYZZ<F>* p = (const XYZZ<F>*)j.in + ((o * j.S) << j.log_inner) + i;
    XYZZ<F> acc = XYZZ<F>::inf();
#pragma unroll 1
    for (uint32_t s = lane; s < j.S; s += 32) { XYZZ<F> v = load_vec(p + ((uint64_t)s << j.log_inner)); acc.add_i(v); }
    acc = warp_sum<F>(acc);
    if (lane == 0) store_vec((XYZZ<F>*)j.out + wid, acc);
}

// sb_set_tuning(1, 1): reduce the buckets with k_reduce / k_window_sum even where ws_plan accepts the geometry
extern int g_msm_force_reduce;

// Host plan of the axis-sum levels for one geometry.  Buckets of a window form H = 2^er rows... of 2^m columns
// (m = WS_COL_BITS when the window has more than 2^m buckets, else there is no split and C = the buckets themselves).
static constexpr int WS_COL_BITS = 10;
struct WsPlan {
    bool ok = false;                 // false: geometry outside the design (more than 2^20 buckets per window) -> k_reduce
    int m = 0, er = 0, ec = 0;       // column bits, bits the row chain reduces (= m), bits the column chain reduces
    int levels = 0; int br[8] = {0}, bc[8] = {0};
    uint32_t lenR = 0, lenC = 0, nR = 0, nC = 0;
    size_t rowA = 0, rowB = 0, colA = 0, colB = 0, tw = 0;   // scratch sizes in XYZZ elements
    size_t elems() const { return rowA + rowB + colA + colB + tw + 8; }
};
__host__ inline WsPlan ws_plan(const MsmGeom& g) {
    WsPlan p; const int cbits = g.c - 1; const size_t NW = g.windows();
    if (cbits > 2 * WS_COL_BITS || cbits < 0) return p;
    p.ok = true;
    if (cbits > WS_COL_BITS) { p.m = WS_COL_BITS; p.er = p.m; p.ec = cbits - p.m; p.lenR = 1u << p.ec; p.lenC = 1u << p.m; }
    else { p.lenR = 0; p.lenC = g.B; }
    // level 0: S = 8 (k_axis_sum, carries the work); level 1: everything left, <= 7 bits (k_axis_tree, one warp per output)
    int rr = p.er, rc = p.ec;
    for (int l = 0; l < 2 && (rr > 0 || rc > 0); l++) {
        p.levels++;
        p.br[l] = l == 0 ? (rr < 3 ? rr : 3) : rr; p.bc[l] = l == 0 ? (rc < 3 ? rc : 3) : rc; rr -= p.br[l]; rc -= p.bc[l];
        const size_t orow = p.br[l] ? (NW * g.B) >> (p.er - rr) : 0, ocol = p.bc[l] ? (NW * g.B) >> (p.ec - rc) : 0;
        if (l & 1) { p.rowB = orow; p.colB = ocol; } else { p.rowA = orow; p.colA = ocol; }
    }
    p.nR = (p.lenR + 31) / 32; p.nC = (p.lenC + 31) / 32;
    p.tw = 2 * NW * (p.nR + p.nC);
    return p;
}
// Points per window that msm_buckets writes as window sums, the layout msm_group.inl's combine reads: the five weighted
// parts of k_ws_final, or one point (k_reduce / k_window_sum) when ws_plan rejects the geometry or sb_set_tuning(1, 1)
// forces the running-sum reduction.  A batch's proof k starts at point k * windows_per_proof() * msm_wsum_parts(g).
__host__ inline uint32_t msm_wsum_parts(const MsmGeom& g) { return (ws_plan(g).ok && !g_msm_force_reduce) ? 5u : 1u; }
// scratch (in XYZZ elements) of the reduction: k_reduce partials, or the axis-sum ping-pong buffers + chunk pairs
__host__ inline size_t msm_reduce_scratch_elems(const MsmGeom& g) {
    const uint32_t NW = g.windows();
    const uint32_t L = g.B < (uint32_t)MSM_RED_CHUNK ? g.B : MSM_RED_CHUNK;
    const uint32_t ctas_per_window = (g.B / L + 127) / 128;
    const size_t legacy = (size_t)2 * NW * ctas_per_window;
    const WsPlan p = ws_plan(g);
    return (p.ok && p.elems() > legacy) ? p.elems() : legacy;
}

// ------------------------------------------------------------------------------------------------
// Precomputed window multiples for a registered base set: table[w*n + i] = 2^(c*w) * P_i (affine), w < W.
// One thread per point: c doublings per window in XYZZ, one inversion per table entry.  One-time cost per key.
// ------------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(128) k_precompute(const Affine<F>* __restrict__ bases, uint64_t n, int c, int W, Affine<F>* __restrict__ table) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine<F> a = load_vec(bases + i);
    store_vec(table + i, a);
    if (a.is_inf()) {
        for (int w = 1; w < W; w++) store_vec(table + (uint64_t)w * n + i, a);
        return;
    }
    XYZZ<F> p; p.x = a.x; p.y = a.y; p.zz = F::one(); p.zzz = F::one();
    for (int w = 1; w < W; w++) {
        for (int j = 0; j < c; j++) p = XYZZ<F>::dbl(p);
        Affine<F> o;
        if (p.is_inf()) { o.x = F::zero(); o.y = F::zero(); }
        else { F t = PairInvF(F::mul(p.zz, p.zzz)); o.x = F::mul(p.x, F::mul(t, p.zzz)); o.y = F::mul(p.y, F::mul(t, p.zz)); p.x = o.x; p.y = o.y; p.zz = F::one(); p.zzz = F::one(); }
        store_vec(table + (uint64_t)w * n + i, o);
    }
}

// ------------------------------------------------------------------------------------------------
// Synthetic bases for benchmarks and tests, written as affine Montgomery points.  The definition is the CPU
// oracle's incremental generator (chunks of 4096 points: P_{c,0} = k0(c)*G, P_{c,j+1} = P_{c,j} + kd*G), which costs the
// host two additions per point; here every point is computed independently as (k0(c) + j*kd)*G — the same group
// element, hence the same affine bytes — so the B200 arm and the CPU reference arm of bench.py build identical keys.
// One thread per point: 77-bit double-and-add in XYZZ, then one field inversion.
__host__ __device__ inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
static constexpr uint64_t GEN_CHUNK = 4096;
template <class F>
__global__ void __launch_bounds__(128) k_gen_points(Affine<F> g, uint64_t seed, uint64_t n, Affine<F>* __restrict__ out) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t c = i / GEN_CHUNK, j = i % GEN_CHUNK;
    const uint64_t k0 = (seed ^ 0x9E3779B97F4A7C15ull) + c * 0xD1B54A32D192ED03ull, kd = seed * 2654435761ull + 12345ull;
    // s = k0 + j*kd  (< 2^77) as (hi, lo)
    uint64_t lo = j * kd, hi = __umul64hi(j, kd);
    lo += k0; hi += lo < k0 ? 1 : 0;
    const F one = F::one();
    XYZZ<F> r = XYZZ<F>::inf();
    for (int bit = 79; bit >= 0; bit--) {
        r = XYZZ<F>::dbl(r);
        const uint64_t wd = bit >= 64 ? hi : lo;
        if ((wd >> (bit & 63)) & 1) r.add_affine(g.x, g.y, one);
    }
    Affine<F> a;
    if (r.is_inf()) { a.x = F::zero(); a.y = F::zero(); }
    else { F t = PairInvF(F::mul(r.zz, r.zzz)); a.x = F::mul(r.x, F::mul(t, r.zzz)); a.y = F::mul(r.y, F::mul(t, r.zz)); }
    store_vec(out + i, a);
}

// ------------------------------------------------------------------------------------------------
// Device scratch (grow-only) and the two halves of the pipeline.
// ------------------------------------------------------------------------------------------------
struct MsmScratch {
    void* p = nullptr; size_t cap = 0;
    void* get(size_t bytes) {
        if (bytes > cap) { if (p) cudaFree(p); p = nullptr; cap = 0; if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr; cap = bytes; }
        return p;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};


struct MsmLaunchStats {
    int launches = 0;
    // optional profiling: event pairs recorded around kernel groups (tag = PROF_* below; accumulation uses cur_tag)
    cudaEvent_t* ev = nullptr; int nev = 0; int used = 0; int tag[128] = {0}; int cur_tag = 0;
};
enum { PROF_ACC_G1 = 1, PROF_ACC_G2 = 2, PROF_SORT = 3, PROF_FOLD = 4, PROF_REDUCE = 5, PROF_QAP = 6, PROF_NTT = 7, PROF_JOIN = 8,
       PROF_FOLD_G2 = 9, PROF_REDUCE_G2 = 10 };
// one event pair around a group of launches on `st`; a no-op unless profiling is armed (api.cu prof_begin)
struct ProfScope {
    MsmLaunchStats* s; cudaStream_t st; int idx = -1;
    ProfScope(MsmLaunchStats* s_, int tag, cudaStream_t st_) : s(s_), st(st_) {
        if (s && s->ev && s->used + 2 <= s->nev && s->used / 2 < 128) { idx = s->used; s->used += 2; s->tag[idx / 2] = tag; cudaEventRecord(s->ev[idx], st); }
    }
    void end() { if (idx >= 0) { cudaEventRecord(s->ev[idx + 1], st); idx = -1; } }
    void end(cudaStream_t other) { st = other; end(); }
};

// Sorted digit entries of one scalar vector; shared by every MSM that uses the same scalars
// (Groth16: A, B1, B2 and C all multiply the witness, src/groth16_prove.js:84-97).
struct MsmSorted {
    const uint32_t* keys = nullptr; const uint32_t* vals = nullptr; const uint64_t* counts = nullptr;
    uint64_t n = 0, total = 0; MsmGeom g{};
    // Sorted entries per k_accumulate thread.  The target is MSM_SEG, or more when the buckets are dense (hundreds of entries
    // per bucket, e.g. the 9n-point fflonk commitments: a thread's first run becomes a head partial, and with several heads
    // per bucket the runs of equal head keys outgrow k_fold_short's parallel path).  The actual value is chosen on the
    // device (k_count_valid, counts[MSM_COUNTS_SEG]) once the number of valid entries M is known: every thread does the same
    // work, so the kernel time is waves x seg, and seg = ceil(M / (k * resident threads)) makes the grid exactly k full waves
    // of the SMs instead of k - 1 waves and a fraction (applied for k <= 3: shards of a multi-GPU proof, small MSMs; with
    // more waves the effect vanishes).  seg_lo = the smallest value the device may pick (grid and
    // head-buffer sizing on the host).
    uint32_t seg_lo = MSM_SEG;
};

// msm_sort.cu: digits + radix sort + valid count.  d_scalars is a device pointer.
int msm_sort_entries(const uint8_t* d_scalars, uint32_t sbytes, uint64_t n, MsmGeom g, MsmScratch& scratch,
                     cudaStream_t stream, MsmSorted* out, MsmLaunchStats* stats);

// Bucket accumulation + reduction for one base set.  Writes g.W window sums to d_wsum (device).  Asynchronous.
// If tail_stream differs from stream, the throughput-bound accumulation runs on `stream` and the latency-bound tail
// (fold, bucket reduction, window sum) on `tail_stream` after `ev_acc` (recorded here): with a higher-priority tail
// stream the tail of one MSM slips into the SM slots freed by the next MSM's accumulation instead of queueing behind it.
template <class F>
int msm_buckets(const Affine<F>* d_bases, const MsmSorted& s, MsmScratch& scratch, cudaStream_t stream,
                XYZZ<F>* d_wsum, MsmLaunchStats* stats, cudaStream_t tail_stream = nullptr, cudaEvent_t ev_acc = nullptr) {
    const MsmGeom g = s.g;
    const uint32_t NW = g.windows();
    const uint64_t nbuckets = (uint64_t)NW * g.B;
    const uint64_t heads0 = (s.total + s.seg_lo - 1) / s.seg_lo;   // upper bound; the device knows the exact count (counts[1])
    const uint64_t heads1 = (heads0 + MSM_SEG - 1) / MSM_SEG;
    const uint32_t L = g.B < (uint32_t)MSM_RED_CHUNK ? g.B : MSM_RED_CHUNK;
    const uint32_t chunks = g.B / L;
    const uint32_t red_threads = 128;
    const uint32_t ctas_per_window = (chunks + red_threads - 1) / red_threads;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t o_buckets = 0;
    size_t o_headsA = o_buckets + al(nbuckets * sizeof(XYZZ<F>)), o_hkA = o_headsA + al(heads0 * sizeof(XYZZ<F>));
    size_t o_headsB = o_hkA + al(heads0 * 4), o_hkB = o_headsB + al(heads1 * sizeof(XYZZ<F>));
    size_t o_hkM = o_hkB + al(heads1 * 4);                     // level-1 keys after the short-run fast path
    size_t o_part = o_hkM + al(heads0 * 4);
    size_t bytes = o_part + al(msm_reduce_scratch_elems(g) * sizeof(XYZZ<F>));
    uint8_t* base = (uint8_t*)scratch.get(bytes);
    if (!base) return (int)cudaErrorMemoryAllocation;
    XYZZ<F>* buckets = (XYZZ<F>*)(base + o_buckets);
    XYZZ<F>* headsA = (XYZZ<F>*)(base + o_headsA); uint32_t* hkA = (uint32_t*)(base + o_hkA);
    XYZZ<F>* headsB = (XYZZ<F>*)(base + o_headsB); uint32_t* hkB = (uint32_t*)(base + o_hkB);
    XYZZ<F>* partials = (XYZZ<F>*)(base + o_part);
    uint32_t* hkM = (uint32_t*)(base + o_hkM);
    int launches = 0;
    const bool g2 = stats && stats->cur_tag == PROF_ACC_G2;     // the tail's profiling tags name the MSM's group
    // minBlocksPerSM of the two wide tail kernels (k_fold_short, k_axis_sum), per coordinate field as for k_accumulate
    // below.  ptxas, sm_90a, registers of k_fold_short / k_axis_sum: BN254 G1 124 / 124, BLS12-381 G1 190 / 190, BN254 G2
    // 248 / 242, all without spills; BLS12-381 G2 255 / 255 with 132 / 52 B of spill stores, which no launch bound can
    // remove (255 is the per-thread cap).  H100 at 400 W: a 2^20 BLS12-381 G2 MSM 26.5 ms, 26.6 with the
    // out-of-line additions of XYZZ::add.
    constexpr int TAIL_MINB = sizeof(F) > 32 ? 2 : 4;
    cudaMemsetAsync(buckets, 0, nbuckets * sizeof(XYZZ<F>), stream);
    if (heads0) {
        ProfScope prof(stats, stats ? stats->cur_tag : 0, stream);
        {
            const unsigned grid = (unsigned)((heads0 + MSM_ACC_THREADS - 1) / MSM_ACC_THREADS);
            // minBlocksPerSM per coordinate field, measured on an H100 at 400 W:
            // - extension field (G2): 2.  2^20 G2 accumulation 7.6 ms, vs 8.3 at 3 and 9.2 at 4.
            // - 12-limb base field (BLS12-381 G1): 2.  At 4 the 128-register cap spills ~50 words of the mixed addition (ptxas,
            //   sm_90a: 184 B spill stores / 132 B loads); 3 (167 registers) and 2 (182) do not spill.  Nine accumulations of a
            //   2^18 PLONK BLS12-381 proof: 15.5 ms at 2, 16.7 at 4, 19.1 at 3.
            // - 8-limb base field (BN254 G1): 4 (116 registers, no spills).  2^20 Groth16: 2, 3 and 4 within 1 %.
            constexpr int MINB = sizeof(F) > 32 ? 2 : 4;
            k_accumulate<F, MINB><<<grid, MSM_ACC_THREADS, 0, stream>>>(d_bases, s.keys, s.vals, s.counts, buckets, headsA, hkA);
            launches++;
        }
        prof.end();
        if (tail_stream && tail_stream != stream && ev_acc) {
            cudaEventRecord(ev_acc, stream); cudaStreamWaitEvent(tail_stream, ev_acc, 0); stream = tail_stream;
        }
        ProfScope pfold(stats, g2 ? PROF_FOLD_G2 : PROF_FOLD, stream);
        k_fold_short<F, TAIL_MINB><<<(unsigned)((heads0 + MSM_ACC_THREADS - 1) / MSM_ACC_THREADS), MSM_ACC_THREADS, 0, stream>>>(
            headsA, hkA, hkM, s.counts, buckets); launches++;
        // fold cascade: level l consumes counts[l] heads (upper bound m on the host, exact count on the device)
        uint64_t m = heads0; int level = 1;
        XYZZ<F>* hin = headsA; uint32_t* kin = hkM; XYZZ<F>* hout = headsB; uint32_t* kout = hkB;
        while (true) {
            uint64_t threads = (m + MSM_SEG - 1) / MSM_SEG;
            k_fold<F><<<(unsigned)((threads + MSM_ACC_THREADS - 1) / MSM_ACC_THREADS), MSM_ACC_THREADS, 0, stream>>>(
                hin, kin, s.counts, level, buckets, hout, kout); launches++;
            if (m <= (uint64_t)MSM_SEG) break;
            m = threads; level++;
            XYZZ<F>* th = hin; hin = hout; hout = th; uint32_t* tk = kin; kin = kout; kout = tk;
            if (level >= 8) return (int)cudaErrorUnknown;
        }
        pfold.end();
    }
    if (!heads0 && tail_stream && tail_stream != stream && ev_acc) { cudaEventRecord(ev_acc, stream); cudaStreamWaitEvent(tail_stream, ev_acc, 0); stream = tail_stream; }
    ProfScope pred(stats, g2 ? PROF_REDUCE_G2 : PROF_REDUCE, stream);
    const WsPlan wp = ws_plan(g);
    if (msm_wsum_parts(g) == 5) {
        // axis sums (rows and columns of one level per launch), then the warp-shuffle weighted sums
        XYZZ<F>* rowb[2] = {partials, partials + wp.rowA};
        XYZZ<F>* colb[2] = {partials + wp.rowA + wp.rowB, partials + wp.rowA + wp.rowB + wp.colA};
        XYZZ<F>* tw = partials + wp.rowA + wp.rowB + wp.colA + wp.colB;
        const XYZZ<F>* rin = buckets; const XYZZ<F>* cin = buckets;
        int rr = wp.er, rc = wp.ec;
        for (int l = 0; l < wp.levels; l++) {
            AxisJob jr{nullptr, nullptr, 0, 1, 0}, jc{nullptr, nullptr, 0, 1, 0};
            if (wp.br[l]) { rr -= wp.br[l]; jr = AxisJob{rin, rowb[l & 1], (uint64_t)nbuckets >> (wp.er - rr), 1u << wp.br[l], (uint32_t)rr}; rin = rowb[l & 1]; }
            if (wp.bc[l]) { rc -= wp.bc[l]; jc = AxisJob{cin, colb[l & 1], (uint64_t)nbuckets >> (wp.ec - rc), 1u << wp.bc[l], (uint32_t)wp.m}; cin = colb[l & 1]; }
            const uint64_t mx = jr.total > jc.total ? jr.total : jc.total;
            if (l == 0) k_axis_sum<F, TAIL_MINB><<<dim3((unsigned)((mx + 127) / 128), 2), 128, 0, stream>>>(jr, jc);
            else k_axis_tree<F><<<dim3((unsigned)((mx + 3) / 4), 2), 128, 0, stream>>>(jr, jc);
            launches++;
        }
        const uint32_t per = wp.nR + wp.nC;
        k_ws_chunks<F><<<(NW * per + 3) / 4, 128, 0, stream>>>(wp.lenR ? rin : nullptr, wp.lenR, cin, wp.lenC, NW, tw); launches++;
        k_ws_final<F><<<NW, 128, 0, stream>>>(tw, wp.nR, wp.nC, d_wsum); launches++;
    } else {
        k_reduce<F><<<NW * ctas_per_window, red_threads, red_threads * sizeof(XYZZ<F>), stream>>>(buckets, g, partials, ctas_per_window); launches++;
        k_window_sum<F><<<NW, 32, 32 * sizeof(XYZZ<F>), stream>>>(partials, ctas_per_window, d_wsum); launches++;
    }
    pred.end();
    if (stats) stats->launches += launches;
    return (int)cudaGetLastError();
}

}  // namespace sb
