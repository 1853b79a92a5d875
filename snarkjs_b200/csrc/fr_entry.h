// fr_entry.h — untyped entry points for the Fr kernels (NTT passes, apply-key, conversions, QAP), one
// translation unit (fr_kernels.cu) instantiates them for BN254 Fr and BLS12-381 Fr (both 8 limbs).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
namespace sb {
static constexpr int NTT_DMAX = 10;          // largest per-pass degree (tile 2^(deg+logc) <= 4096 elements = 128 KiB)
struct FrNttTables { const void* tw_lo; const void* tw_hi; int h; const void* wr; };
struct FrPre { const void* lo; const void* hi; int h; };
// all pointers are device pointers to 32-byte Fr elements
int fr_configure(int curve);
// runs log2(n) = L; input in a, scratch b; *result = a or b.  pre/post may be null.
int fr_ntt(int curve, void* a, void* b, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
           cudaStream_t stream, void** result, int* launches);
// batched variant: count (<= 4) transforms of size 2^L; a[i] input, b[i] scratch; *side = 0 results in a[], 1 in b[]
int fr_ntt_batch(int curve, void* const* a, void* const* b, int count, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
                 cudaStream_t stream, int* side, int* launches);
// count (<= 65535) contiguous transforms of size 2^L: a = count * 2^L inputs back to back, b = as much scratch; *side as above
int fr_ntt_strided(int curve, void* a, void* b, int count, int L, const FrNttTables* tb, const FrPre* pre, const void* post_scale,
                   cudaStream_t stream, int* side, int* launches);
// number of passes fr_ntt / fr_ntt_batch run for size 2^L (the result lands in the scratch buffers iff it is odd)
int fr_ntt_passes(int L);
int fr_apply_key(int curve, const void* in, void* out, uint64_t n, const FrPre* t, cudaStream_t stream);
int fr_convert(int curve, const void* in, void* out, uint64_t n, int to_mont, cudaStream_t stream);
int fr_join_abc(int curve, const void* a, const void* b, const void* c, void* out, uint64_t n, cudaStream_t stream);
// K proofs: witness k (n_witness elements) at witness + k * n_witness; its A/B/C rows at A/B/C + k * n
int fr_qap_rows(int curve, const uint64_t* row_ptr, const uint32_t* sig, const void* coef, const void* witness, uint64_t n_witness,
                void* A, void* B, void* C, uint64_t n, uint32_t K, cudaStream_t stream);
}
