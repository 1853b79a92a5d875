// fr_kernels.cu — instantiates ntt.cuh for BN254 Fr and BLS12-381 Fr.
#include "ntt.cuh"
#include "fr_entry.h"
namespace sb {
int g_ntt_tile_log = 11;   // measured: 2^20 NTT 0.277 ms (tile 2^11, 3 CTAs/SM) vs 0.299 ms (2^12)
typedef Fp<BnFr> FrBn;
typedef Fp<BlsFr> FrBls;
#define FR_DISPATCH(curve, ...) \
    if (curve == 0) { typedef FrBn F; __VA_ARGS__; } else if (curve == 1) { typedef FrBls F; __VA_ARGS__; } else return -1;

int fr_configure(int curve) {
    FR_DISPATCH(curve, return (int)ntt_configure<F>())
}
int fr_ntt(int curve, void* a, void* b, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
           cudaStream_t stream, void** result, int* launches) {
    FR_DISPATCH(curve, {
        NttTables<F> t; t.tw_lo = (const F*)tb->tw_lo; t.tw_hi = (const F*)tb->tw_hi; t.h = tb->h; t.wr = (const F*)tb->wr;
        NttPre<F> p; if (pre) { p.lo = (const F*)pre->lo; p.hi = (const F*)pre->hi; p.h = pre->h; }
        *result = ntt_run<F>((F*)a, (F*)b, L, t, pre ? &p : nullptr, (const F*)post_scale, stream, launches);
        return (int)cudaGetLastError();
    })
}
int fr_ntt_batch(int curve, void* const* a, void* const* b, int count, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
                 cudaStream_t stream, int* side, int* launches) {
    if (count < 1 || count > 4) return -1;
    FR_DISPATCH(curve, {
        NttTables<F> t; t.tw_lo = (const F*)tb->tw_lo; t.tw_hi = (const F*)tb->tw_hi; t.h = tb->h; t.wr = (const F*)tb->wr;
        NttPre<F> p; if (pre) { p.lo = (const F*)pre->lo; p.hi = (const F*)pre->hi; p.h = pre->h; }
        *side = ntt_run_batch<F>((F* const*)a, (F* const*)b, count, L, t, pre ? &p : nullptr, (const F*)post_scale, stream, launches);
        return (int)cudaGetLastError();
    })
}
int fr_ntt_strided(int curve, void* a, void* b, int count, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
                   cudaStream_t stream, int* side, int* launches) {
    if (count < 1 || count > 65535 || L < 0) return -1;
    FR_DISPATCH(curve, {
        NttTables<F> t; t.tw_lo = (const F*)tb->tw_lo; t.tw_hi = (const F*)tb->tw_hi; t.h = tb->h; t.wr = (const F*)tb->wr;
        NttPre<F> p; if (pre) { p.lo = (const F*)pre->lo; p.hi = (const F*)pre->hi; p.h = pre->h; }
        F* aa[1] = {(F*)a}; F* bb[1] = {(F*)b};
        *side = ntt_run_batch<F>(aa, bb, count, L, t, pre ? &p : nullptr, (const F*)post_scale, stream, launches, 1ull << L);
        return (int)cudaGetLastError();
    })
}
int fr_ntt_passes(int L) { return ntt_plan(L).npass; }
int fr_apply_key(int curve, const void* in, void* out, uint64_t n, const FrPre* t, cudaStream_t stream) {
    FR_DISPATCH(curve, {
        NttPre<F> p; p.lo = (const F*)t->lo; p.hi = (const F*)t->hi; p.h = t->h;
        if (n) k_apply_key<F><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const F*)in, (F*)out, n, p);
        return (int)cudaGetLastError();
    })
}
int fr_convert(int curve, const void* in, void* out, uint64_t n, int to_mont, cudaStream_t stream) {
    FR_DISPATCH(curve, {
        if (n) k_convert<F><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const F*)in, (F*)out, n, to_mont);
        return (int)cudaGetLastError();
    })
}
int fr_join_abc(int curve, const void* a, const void* b, const void* c, void* out, uint64_t n, cudaStream_t stream) {
    FR_DISPATCH(curve, {
        if (n) k_join_abc<F><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const F*)a, (const F*)b, (const F*)c, (F*)out, n);
        return (int)cudaGetLastError();
    })
}
int fr_qap_rows(int curve, const uint64_t* row_ptr, const uint32_t* sig, const void* coef, const void* witness, uint64_t n_witness,
                void* A, void* B, void* C, uint64_t n, uint32_t K, cudaStream_t stream) {
    FR_DISPATCH(curve, {
        const unsigned grid = (unsigned)((n * K + 127) / 128);
        if (n && K == 1) k_qap_rows<F, false><<<grid, 128, 0, stream>>>(row_ptr, sig, (const F*)coef, (const F*)witness, n_witness, (F*)A, (F*)B, (F*)C, n, 1);
        else if (n && K) k_qap_rows<F, true><<<grid, 128, 0, stream>>>(row_ptr, sig, (const F*)coef, (const F*)witness, n_witness, (F*)A, (F*)B, (F*)C, n, K);
        return (int)cudaGetLastError();
    })
}
}
