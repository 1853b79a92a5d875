// verify_entry.h — untyped per-curve entry points of the device pairing and the batched Groth16 verifier (verify.cuh); each
// curve lives in its own translation unit (verify_curve.inl) so the two instantiations compile in parallel.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
namespace sb {
// All pointers but the vk of NAME_vk_valid are device pointers.  vk: alpha1 || beta2 || gamma2 || delta2 || IC[0..n_public],
// affine Montgomery.  lines: verify_bytes(0); target: verify_bytes(1); terms: count * n_public * verify_bytes(2).
// The PLONK (proto 0) / fflonk (proto 1, BN254 only) verifier of verify_plonk.cuh: pv_bytes(proto, 0) key, 1 lines, 2 terms
// per proof, 3 proof, 4 scalars per proof; pv_key builds the key on the host (false: a key point is not valid); key, lines, scalars
// (sc) and terms are device buffers of those sizes.
#define SB_DECL_VERIFY(NAME) \
    int NAME##_pair_eval(int op, const void* in, void* out, uint64_t n, cudaStream_t stream); \
    bool NAME##_vk_valid(const uint8_t* vk, uint32_t n_public); \
    uint64_t NAME##_verify_bytes(int what); \
    int NAME##_verify_prepare(const void* vk, void* lines, void* target, cudaStream_t stream); \
    int NAME##_verify_run(const void* vk, uint32_t n_public, const void* lines, const void* target, const void* pubs, \
                          const void* proofs, uint32_t count, void* terms, int32_t* status, cudaStream_t stream, int* launches); \
    uint64_t NAME##_pv_bytes(int proto, int what); \
    bool NAME##_pv_key(int proto, const uint8_t* vk, uint32_t n_public, uint32_t power, const uint8_t* gen1, const uint8_t* gen2, \
                       const uint8_t* wpow, void* out); \
    int NAME##_pv_prepare(const void* key, void* lines, cudaStream_t stream); \
    int NAME##_pv_run(int proto, const void* key, const void* lines, const void* pubs, const void* proofs, uint32_t count, void* sc, \
                      void* terms, int32_t* status, cudaStream_t stream, int* launches);
SB_DECL_VERIFY(bn254)
SB_DECL_VERIFY(bls12381)
}
