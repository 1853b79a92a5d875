// Sharded commitments for the host PLONK / fflonk flows (tests/host/host_plonk.cpp, host_fflonk.cpp): a stand-in for the
// CPU oracle library that forwards the NTT, group and root calls to the real oracle, and computes every G1 MSM the way
// sb_plonk_prove_multi / sb_fflonk_prove_multi compute a commitment: the P PTau points split into n_shards contiguous
// ranges by the library's own sb_shard_range, each shard's part of [0, len) multiplied on its own (an empty part adds
// nothing), the partials summed.  The host flows load it in place of the oracle, so their commit_plain sums the oracle's
// MSMs over the same slices as the device path.  Driven by tests/test_host_plonk_sharded.py.  Test infrastructure only.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <vector>

typedef int (*fft_t)(int, const uint8_t*, uint64_t, int, uint8_t*);
typedef int (*msm_t)(int, int, const uint8_t*, const uint8_t*, int, uint64_t, int, uint8_t*);
typedef int (*gop_t)(int, int, int, const uint8_t*, const uint8_t*, uint8_t*);
typedef int (*root_t)(int, int, uint8_t*);
typedef void (*range_t)(uint64_t, int, int, uint64_t*, uint64_t*);

static fft_t r_fft; static msm_t r_msm; static gop_t r_gop; static root_t r_root; static range_t r_range;
static uint64_t g_points = 0; static int g_shards = 1;
static uint64_t g_msms = 0, g_parts = 0, g_empty = 0;   // sharded MSMs, shard parts multiplied, shard parts left empty

extern "C" {
// oracle_so: the real oracle; points: P, the PTau set the commitments index; shard_range: sb_shard_range of libsnarkb200
int hs_configure(const char* oracle_so, uint64_t points, int n_shards, void* shard_range) {
    void* so = dlopen(oracle_so, RTLD_NOW);
    if (!so || n_shards < 1 || !shard_range) return -1;
    r_fft = (fft_t)dlsym(so, "or_fr_fft"); r_msm = (msm_t)dlsym(so, "or_multiexp_affine");
    r_gop = (gop_t)dlsym(so, "or_group_op"); r_root = (root_t)dlsym(so, "or_fr_root");
    r_range = (range_t)shard_range;
    g_points = points; g_shards = n_shards; g_msms = g_parts = g_empty = 0;
    return r_fft && r_msm && r_gop && r_root ? 0 : -1;
}
void hs_stats(uint64_t* out) { out[0] = g_msms; out[1] = g_parts; out[2] = g_empty; }

int or_fr_fft(int curve, const uint8_t* in, uint64_t n, int inverse, uint8_t* out) { return r_fft(curve, in, n, inverse, out); }
int or_group_op(int curve, int group, int op, const uint8_t* a, const uint8_t* b, uint8_t* out) { return r_gop(curve, group, op, a, b, out); }
int or_fr_root(int curve, int what, uint8_t* out) { return r_root(curve, what, out); }

int or_multiexp_affine(int curve, int group, const uint8_t* bases, const uint8_t* scalars, int sb, uint64_t n, int conc, uint8_t* out) {
    if (group != 1) return r_msm(curve, group, bases, scalars, sb, n, conc, out);
    const size_t aff = curve == 0 ? 64 : 96, jac = curve == 0 ? 96 : 144;
    std::vector<uint8_t> acc(jac), part(jac), sum(jac);
    int rc = r_msm(curve, group, bases, scalars, sb, 0, conc, acc.data());     // the empty sum
    g_msms++;
    for (int i = 0; i < g_shards && !rc; i++) {
        uint64_t lo = 0, cnt = 0;
        r_range(g_points, i, g_shards, &lo, &cnt);
        const uint64_t m = n > lo ? (cnt < n - lo ? cnt : n - lo) : 0;
        if (!m) { g_empty++; continue; }
        g_parts++;
        rc = r_msm(curve, group, bases + lo * aff, scalars + lo * sb, sb, m, conc, part.data());
        if (!rc) rc = r_gop(curve, group, 0, acc.data(), part.data(), sum.data());
        acc.swap(sum);
    }
    memcpy(out, acc.data(), jac);
    return rc;
}
}
