// gfft_entry.h — untyped per-(curve, group) entry points of the group FFT and group batchApplyKey (gfft.cuh); each
// pair lives in its own translation unit (gfft_group.inl) so the four instantiations compile in parallel.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
namespace sb {
// All pointers are device pointers.  Points are affine (2 coordinates) or Jacobian (3) Montgomery bytes; tw = n/2 plain Fr
// twiddles w_n^j; ninv = plain n^-1 for the inverse transform, null for the forward one; pts = scratch of n XYZZ points.
#define SB_DECL_GFFT(NAME) \
    int NAME##_gfft(const void* in, int in_jac, uint64_t n, int L, const void* tw, const void* ninv, int out_jac, void* pts, \
                    void* out, cudaStream_t stream, int* launches); \
    /* out[i] = in[i] * sc[i], sc = n plain Fr scalars */ \
    int NAME##_gapply(const void* in, int in_jac, const void* sc, uint64_t n, int out_jac, void* out, cudaStream_t stream);
SB_DECL_GFFT(bn254_g1)
SB_DECL_GFFT(bn254_g2)
SB_DECL_GFFT(bls12381_g1)
SB_DECL_GFFT(bls12381_g2)
}
