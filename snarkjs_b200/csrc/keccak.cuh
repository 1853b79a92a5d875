// keccak.cuh — Keccak-256 as src/Keccak256Transcript.js:21 uses it (@noble/hashes keccak_256: Keccak-f[1600], rate 136,
// domain byte 0x01).  The permutation is __host__ __device__: the provers' host transcript (plonk_flow.h) and the device
// verifiers' transcripts (verify_plonk.cuh) run this one copy.  The permutation's loops are fully unrolled, so its lane
// indices are constants; the sponge's byte() indexes the state by the runtime byte position, so on the device the state
// of a Keccak256 lives in local memory (the stack frame of k_pv_scalars, DESIGN §9d).
#pragma once
#include <cstddef>
#include <cstdint>
#include "fp.cuh"

namespace sb {

SB_CONSTEXPR_HD constexpr uint64_t keccak_rc(int i) {
    constexpr uint64_t v[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull, 0x000000000000808Bull,
        0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008Aull, 0x0000000000000088ull, 0x0000000080008009ull,
        0x000000008000000Aull, 0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull, 0x8000000000008003ull, 0x8000000000008002ull,
        0x8000000000000080ull, 0x000000000000800Aull, 0x800000008000000Aull, 0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull,
        0x8000000080008008ull};
    return v[i];
}
SB_CONSTEXPR_HD constexpr int keccak_rot(int i) {   // [x + 5y]
    constexpr int v[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
    return v[i];
}

SB_HD void keccak_f1600(uint64_t* a) {
    auto rol = [](uint64_t x, int n) { return n ? (x << n) | (x >> (64 - n)) : x; };
#pragma unroll 1
    for (int round = 0; round < 24; round++) {
        uint64_t c[5], d[5], b[25];
#pragma unroll
        for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
#pragma unroll
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rol(c[(x + 1) % 5], 1);
#pragma unroll
        for (int i = 0; i < 25; i++) a[i] ^= d[i % 5];
#pragma unroll
        for (int x = 0; x < 5; x++)
#pragma unroll
            for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rol(a[x + 5 * y], keccak_rot(x + 5 * y));
#pragma unroll
        for (int x = 0; x < 5; x++)
#pragma unroll
            for (int y = 0; y < 5; y++) a[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
        a[0] ^= keccak_rc(round);
    }
}

// Keccak-256 absorbing one byte at a time, so a transcript needs no buffer of its own.
struct Keccak256 {
    static constexpr int RATE = 136;
    uint64_t a[25];
    int pos;
    SB_HD void reset() {
#pragma unroll
        for (int i = 0; i < 25; i++) a[i] = 0;
        pos = 0;
    }
    SB_HD void byte(uint8_t v) {
        a[pos >> 3] ^= (uint64_t)v << (8 * (pos & 7));
        if (++pos == RATE) { keccak_f1600(a); pos = 0; }
    }
    // the digest, little-endian lanes as bytes; the sponge must be reset before reuse
    SB_HD void finish(uint8_t out[32]) {
        a[pos >> 3] ^= (uint64_t)0x01 << (8 * (pos & 7));
        a[RATE / 8 - 1] ^= 0x80ull << 56;
        keccak_f1600(a);
#pragma unroll
        for (int i = 0; i < 32; i++) out[i] = (uint8_t)(a[i >> 3] >> (8 * (i & 7)));
    }
};

}  // namespace sb
