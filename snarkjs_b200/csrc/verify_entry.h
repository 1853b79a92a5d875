// verify_entry.h — untyped per-curve entry points of the device pairing and the batched Groth16 verifier (verify.cuh); each
// curve lives in its own translation unit (verify_curve.inl) so the two instantiations compile in parallel.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
namespace sb {
// All pointers but the vk of NAME_vk_valid are device pointers.  vk: alpha1 || beta2 || gamma2 || delta2 || IC[0..n_public],
// affine Montgomery.  lines: verify_bytes(0); target: verify_bytes(1); terms: count * n_public * verify_bytes(2).
#define SB_DECL_VERIFY(NAME) \
    int NAME##_pair_eval(int op, const void* in, void* out, uint64_t n, cudaStream_t stream); \
    bool NAME##_vk_valid(const uint8_t* vk, uint32_t n_public); \
    uint64_t NAME##_verify_bytes(int what); \
    int NAME##_verify_prepare(const void* vk, void* lines, void* target, cudaStream_t stream); \
    int NAME##_verify_run(const void* vk, uint32_t n_public, const void* lines, const void* target, const void* pubs, \
                          const void* proofs, uint32_t count, void* terms, int32_t* status, cudaStream_t stream, int* launches);
SB_DECL_VERIFY(bn254)
SB_DECL_VERIFY(bls12381)
}
