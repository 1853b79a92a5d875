#pragma once
#include <cstdint>
namespace sb {
struct MsmGeom {
    int c;            // window bits
    int W;            // windows
    uint32_t B;       // buckets per window = 2^(c-1)
    // precomputed-window mode (registered bases): the table holds 2^(c*w) * P_i at [w*stride + i], every window
    // shares ONE bucket set (key = |digit|-1, value = table index), so there is a single bucket reduction and no
    // Horner recombination.  first = index of this call's point 0 inside the registered set.
    int precomp = 0;
    uint64_t stride = 0, first = 0;
    // proofs (scalar vectors of n scalars each, over the same bases) sorted and reduced together: proof k owns the bucket
    // sets [k * windows_per_proof(), (k+1) * windows_per_proof())
    uint32_t K = 1;
    uint32_t windows_per_proof() const { return precomp ? 1u : (uint32_t)W; }
    uint32_t windows() const { return K * windows_per_proof(); }
    // points the bucket reduction returns per MSM: every window sum comes back as 5 parts with power-of-two weights
    // (msm.cuh k_ws_final); the host applies the weights (a few doublings of single points, microseconds on a CPU core)
    uint32_t wsum_points() const { return 5u * windows(); }
};

// Largest batch K of n-scalar vectors that one sort can take with window bits c and W windows per scalar: every bucket key
// (k * windows_per_proof + w) * B + |d| - 1 stays below the INVALID key 2^32 - 1 (so K * windows_per_proof * B <= 2^32 - 2),
// and the K * n * W sorted entries stay below 2^32.  0 when not even one vector fits.
inline uint64_t msm_batch_limit(uint64_t n, int c, int W, int precomp) {
    if (c < 1 || c > 32 || W < 1) return 0;
    const uint64_t B = 1ull << (c - 1), wpp = precomp ? 1u : (uint64_t)W;
    const uint64_t lim = 0xfffffffeull / (wpp * B);
    const uint64_t per = n * (uint64_t)W;
    const uint64_t lim_e = per ? 0xffffffffull / per : lim;
    return lim < lim_e ? lim : lim_e;
}
}
