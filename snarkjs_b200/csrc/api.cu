// api.cu — the C ABI of libsnarkb200.so (include/snarkb200.h): context, device buffers, table caches, the
// drop-in bulk operations, and the fused Groth16 prover.  Host-side orchestration only; kernels live in
// msm*.cu / fr_kernels.cu.  There is no CPU fallback: without a CUDA device sb_create fails.
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <map>
#include <algorithm>
#include <mutex>
#include <atomic>
#include <future>
#include <thread>
#include <functional>
#include <condition_variable>
#include <deque>
#include <memory>
#include <dlfcn.h>
#include <nccl.h>      // types and prototypes only: the library is dlopen'ed on first use (no link-time dependency)
#include <fcntl.h>
#include <unistd.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include "../../include/snarkb200.h"
#include "ec.cuh"
#include "msm.cuh"
#include "msm_entry.h"
#include "fr_entry.h"
#include "gfft_entry.h"
#include "field_entry.h"
#include "zkey.h"

using namespace sb;
namespace sb { double calibrate(int what, cudaStream_t stream); extern int g_ntt_tile_log; }

namespace {

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    void* get(size_t bytes) {
        if (bytes > cap) { if (p) cudaFree(p); p = nullptr; cap = 0; if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) return nullptr; cap = bytes; }
        return p;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// group vtable (one per curve x group)
struct GroupOps {
    int (*buckets)(const void*, const MsmSorted&, MsmScratch&, cudaStream_t, void*, MsmLaunchStats*, cudaStream_t, cudaEvent_t);
    void (*combine)(const uint8_t*, const MsmGeom&, uint8_t*);
    void (*add)(uint8_t*, const uint8_t*);
    void (*to_jacobian)(const uint8_t*, uint8_t*);
    void (*to_affine)(const uint8_t*, uint8_t*);
    void (*from_affine)(const uint8_t*, uint8_t*);
    void (*times)(const uint8_t*, const uint8_t*, int, uint8_t*);
    int (*gen_points)(const uint8_t*, uint64_t, uint64_t, void*, cudaStream_t);
    int (*precompute)(const void*, uint64_t, int, int, void*, cudaStream_t);
    int (*gfft)(const void*, int, uint64_t, int, const void*, const void*, int, void*, void*, cudaStream_t, int*);
    int (*gapply)(const void*, int, const void*, uint64_t, int, void*, cudaStream_t);
    uint32_t xyzz_bytes;
    uint32_t aff_bytes;
};
#define SB_GROUP_OPS(NAME, AFF) GroupOps{NAME##_buckets, NAME##_combine, NAME##_add, NAME##_to_jacobian, NAME##_to_affine, NAME##_from_affine, NAME##_times, NAME##_gen_points, NAME##_precompute, NAME##_gfft, NAME##_gapply, NAME##_xyzz_bytes(), AFF}

struct NttTab { DevBuf lo, hi; int h = 0; };
struct PreTab { DevBuf lo, hi; int h = 0; std::string key; };

struct BaseSet { int group = 0; uint64_t n = 0; void* d = nullptr; void* table = nullptr; MsmGeom gp{}; };

struct Groth16Key {
    uint32_t nVars = 0, nPublic = 0, domainSize = 0; int power = 0;
    std::vector<uint8_t> alpha1, beta1, beta2, gamma2, delta1, delta2;
    void *dA = nullptr, *dB1 = nullptr, *dB2 = nullptr, *dC = nullptr, *dH = nullptr;   // bases (C padded to nVars)
    void *tA = nullptr, *tB1 = nullptr, *tB2 = nullptr, *tC = nullptr, *tH = nullptr;   // precomputed window tables
    MsmGeom gpW{}, gpH{};                                                                // their geometry (precomp != 0 when built)
    // sharded load (multi-GPU): only the point ranges [wlo, wlo+wcnt) of A/B1/B2/C and [hlo, hlo+hcnt) of H are resident
    int shard = 0, n_shards = 1; uint64_t wlo = 0, wcnt = 0, hlo = 0, hcnt = 0;
    // a whole key made by sb_groth16_load_replicas call replica_id (0: any other load), on context `replica` of n_replicas
    uint64_t replica_id = 0; int replica = 0, n_replicas = 0;
    uint64_t* d_rowptr = nullptr; uint32_t* d_sig = nullptr; void* d_coef = nullptr; uint64_t nCoef = 0;
    // device work buffers
    bool witness_resident = false;   // set by the first upload: sb_groth16_prove_resident refuses to run before it
    void *dW = nullptr, *dWsum = nullptr;
    size_t wsum_bytes = 0;           // size of dWsum (groth16_wsum_room grows it)
    // sb_groth16_prove_batch's K witnesses, and the transforms of K proofs with their scratch (3Kn elements each: loaded
    // for one proof, grown by the batch to its largest sub-batch)
    DevBuf batchW, batchX, batchY;
};

}  // namespace

namespace { struct PlonkKeyDev; void plonk_free_key(PlonkKeyDev*); }     // api_plonk.inl
namespace { struct FflonkKeyDev; void fflonk_free_key(FflonkKeyDev*); }  // api_fflonk.inl

static constexpr size_t STAGE_BYTES = 8u << 20;

struct sb_ctx {
    // Every entry point that takes a context locks it for the duration of the call: overlapping calls on one context
    // (the reference awaits several bulk calls at once, build/snarkjs.js:14653, 14929-14932; the N-API shim runs them
    // as AsyncWorkers on libuv threads) are serialised here instead of racing on the staging buffers and streams.
    // Recursive because some entries are thin wrappers over others (prove_wtns -> prove, load_file -> load).
    std::recursive_mutex mu;
    int curve = 0, device = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    uint32_t n8q = 32;
    GroupOps g1, g2;
    MsmScratch sort_scratch, bucket_scratch;
    MsmScratch sort_scratch2, bscr[5];           // per-MSM scratch for the overlapped Groth16 pipeline
    cudaStream_t aux[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // side streams (tails, NTT chain), the main stream's priority
    cudaEvent_t pev[16];                         // pipeline events
    uint8_t* pinned = nullptr;                   // pinned staging of a Groth16 proof's window sums and counters: 256 KiB,
    size_t pinned_bytes = 0;                     // grown by groth16_wsum_room when a geometry needs more
    uint8_t* stage[2] = {nullptr, nullptr};      // 2 x 8 MiB pinned staging for large pageable host buffers
    cudaEvent_t stage_ev[2];
    MsmLaunchStats stats;
    uint64_t launches = 0;
    DevBuf io[4];
    std::map<int, NttTab> ntt_fwd, ntt_inv;
    DevBuf wr_fwd, wr_inv;
    std::map<int, DevBuf> ninv;           // n^-1 per L
    std::vector<PreTab*> pre_cache;
    std::vector<BaseSet> bases;
    std::vector<Groth16Key*> keys;
    std::vector<PlonkKeyDev*> plonk_keys;
    std::vector<FflonkKeyDev*> fflonk_keys;
    cudaEvent_t ev[8];
    float last_ms[8] = {0};
    int fr_s = 0, fr_bits = 254;
    std::vector<std::vector<uint8_t>> roots;   // w[0..s] Montgomery bytes
    std::vector<uint8_t> nqr, shift;
    std::vector<uint8_t> gen1, gen2;            // affine generators, Montgomery
    cudaEvent_t prof_ev[256];
    double stat[18] = {0};                       // see sb_last_stat
    // multi-GPU (sb_comm_init_rank): one NCCL rank per context
    ncclComm_t comm = nullptr; int rank = 0, world = 1;
    void* d_xchg = nullptr; uint8_t* h_xchg = nullptr;   // partial exchange: world x partial bytes (device / pinned)
};

namespace {

// the message of the last failed call is kept per calling thread, so that two threads sharing a context each read
// their own error text from sb_last_error
thread_local const sb_ctx* t_err_ctx = nullptr;
thread_local std::string t_err;
int fail(sb_ctx* c, int code, const std::string& msg) { if (c) { c->err = msg; t_err_ctx = c; t_err = msg; } return code; }
#define SB_LOCK(c) std::unique_lock<std::recursive_mutex> _sb_lk; if (c) _sb_lk = std::unique_lock<std::recursive_mutex>((c)->mu)
int cuda_fail(sb_ctx* c, cudaError_t e, const char* where) {
    return fail(c, e == cudaErrorMemoryAllocation ? SB_ERR_NOMEM : SB_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
}
#define CU(c, call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return cuda_fail(c, _e, #call); } while (0)

// Host <-> device copies of caller buffers.  Callers hand us pageable memory (Node Buffers, numpy arrays): the driver's
// own pageable path runs at 5-10 GB/s, so large transfers are staged through two pinned 8 MiB buffers (CPU memcpy of
// chunk k+1 overlaps the DMA of chunk k).  Pinned caller memory (bench.py's witness) and small transfers go direct.
int g_stage_enabled = 1;   // sb_set_tuning(8, 0) falls back to the driver's pageable path
bool host_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}
cudaError_t h2d(sb_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!bytes) return cudaSuccess;
    if (!g_stage_enabled || bytes < (1u << 20) || !c->stage[0] || !c->stage[1] || host_is_pinned(src))
        return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream);
    size_t off = 0; int k = 0; cudaError_t e = cudaSuccess;
    while (off < bytes && e == cudaSuccess) {
        const int b = k & 1; const size_t n = std::min(STAGE_BYTES, bytes - off);
        if (k >= 2) e = cudaEventSynchronize(c->stage_ev[b]);
        if (e != cudaSuccess) break;
        memcpy(c->stage[b], (const uint8_t*)src + off, n);
        e = cudaMemcpyAsync((uint8_t*)dst + off, c->stage[b], n, cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess) e = cudaEventRecord(c->stage_ev[b], c->stream);
        off += n; k++;
    }
    // the staging buffers may be reused by the next call: make sure their DMAs are done
    if (e == cudaSuccess) e = cudaEventSynchronize(c->stage_ev[0]);
    if (e == cudaSuccess && k > 1) e = cudaEventSynchronize(c->stage_ev[1]);
    return e;
}
// synchronous on return (the data is in dst)
cudaError_t d2h(sb_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!bytes) return cudaSuccess;
    if (!g_stage_enabled || bytes < (1u << 20) || !c->stage[0] || !c->stage[1] || host_is_pinned(dst)) {
        cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream);
        return e == cudaSuccess ? cudaStreamSynchronize(c->stream) : e;
    }
    size_t off = 0, prev_off = 0, prev_n = 0; int k = 0; cudaError_t e = cudaSuccess;
    while (off < bytes && e == cudaSuccess) {
        const int b = k & 1; const size_t n = std::min(STAGE_BYTES, bytes - off);
        e = cudaMemcpyAsync(c->stage[b], (const uint8_t*)src + off, n, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaEventRecord(c->stage_ev[b], c->stream);
        if (e == cudaSuccess && k >= 1) { e = cudaEventSynchronize(c->stage_ev[b ^ 1]); if (e == cudaSuccess) memcpy((uint8_t*)dst + prev_off, c->stage[b ^ 1], prev_n); }
        prev_off = off; prev_n = n; off += n; k++;
    }
    if (e == cudaSuccess && k >= 1) { const int b = (k - 1) & 1; e = cudaEventSynchronize(c->stage_ev[b]); if (e == cudaSuccess) memcpy((uint8_t*)dst + prev_off, c->stage[b], prev_n); }
    return e;
}

// ------------------------------------------------------------------------------------------------------------
// host Fr helpers, templated on the scalar-field tag
// ------------------------------------------------------------------------------------------------------------
template <class P> struct HostFr {
    typedef Fp<P> F;
    static F from_u32(uint32_t x) { F a = F::zero(); a.v[0] = x; return F::to_mont(a); }
    static void roots(int& s, std::vector<F>& w, F& nqr, F& shift) {
        // reference 12866-12889: nqr = first non-residue from 2, s = 2-adicity, w[s] = nqr^((r-1)/2^s), w[i] = w[i+1]^2
        const int N = P::N;
        uint32_t pm1[N]; for (int i = 0; i < N; i++) pm1[i] = P::p(i); pm1[0] -= 1;
        uint32_t half[N]; for (int i = 0; i < N; i++) half[i] = (pm1[i] >> 1) | (i + 1 < N ? pm1[i + 1] << 31 : 0);
        F negone = F::neg(F::one());
        nqr = from_u32(2);
        while (!(F::pow(nqr, half, N) == negone)) nqr = F::add(nqr, F::one());
        shift = F::sqr(nqr);
        uint32_t t[N]; memcpy(t, pm1, sizeof t); s = 0;
        while (!(t[0] & 1)) { for (int i = 0; i < N; i++) t[i] = (t[i] >> 1) | (i + 1 < N ? t[i + 1] << 31 : 0); s++; }
        w.assign(s + 1, F::zero());
        w[s] = F::pow(nqr, t, N);
        for (int i = s - 1; i >= 0; i--) w[i] = F::sqr(w[i + 1]);
    }
    // lo[e] = base^e (e < 2^h), hi[e] = scale * (base^(2^h))^e (e < nhi)
    static void pow_tables(const F& base, const F& scale, int h, uint64_t nhi, std::vector<F>& lo, std::vector<F>& hi) {
        lo.resize((size_t)1 << h); hi.resize(nhi ? nhi : 1);
        F t = F::one();
        for (size_t e = 0; e < lo.size(); e++) { lo[e] = t; t = F::mul(t, base); }
        F step = t;   // base^(2^h)
        t = scale;
        for (size_t e = 0; e < hi.size(); e++) { hi[e] = t; t = F::mul(t, step); }
    }
};

template <class P> int init_roots(sb_ctx* c) {
    typedef Fp<P> F;
    std::vector<F> w; F nqr, shift; int s;
    HostFr<P>::roots(s, w, nqr, shift);
    c->fr_s = s;
    c->roots.resize(s + 1);
    for (int i = 0; i <= s; i++) c->roots[i].assign((uint8_t*)&w[i], (uint8_t*)&w[i] + 32);
    c->nqr.assign((uint8_t*)&nqr, (uint8_t*)&nqr + 32);
    c->shift.assign((uint8_t*)&shift, (uint8_t*)&shift + 32);
    // in-tile roots w_{2^DMAX}^j and inverse
    F wd = w[NTT_DMAX], wdi = F::inv(wd);
    std::vector<F> lo, hi;
    HostFr<P>::pow_tables(wd, F::one(), NTT_DMAX - 1, 1, lo, hi);
    if (!c->wr_fwd.get(lo.size() * 32)) return SB_ERR_NOMEM;
    cudaMemcpy(c->wr_fwd.p, lo.data(), lo.size() * 32, cudaMemcpyHostToDevice);
    HostFr<P>::pow_tables(wdi, F::one(), NTT_DMAX - 1, 1, lo, hi);
    if (!c->wr_inv.get(lo.size() * 32)) return SB_ERR_NOMEM;
    cudaMemcpy(c->wr_inv.p, lo.data(), lo.size() * 32, cudaMemcpyHostToDevice);
    return 0;
}

template <class P> int build_ntt_tab(sb_ctx* c, int L, bool inverse, NttTab& tab) {
    typedef Fp<P> F;
    F w; memcpy(&w, c->roots[L].data(), 32);
    if (inverse) w = F::inv(w);
    int h = (L + 1) / 2;
    std::vector<F> lo, hi;
    HostFr<P>::pow_tables(w, F::one(), h, (uint64_t)1 << (L - h), lo, hi);
    tab.h = h;
    if (!tab.lo.get(lo.size() * 32) || !tab.hi.get(hi.size() * 32)) return SB_ERR_NOMEM;
    cudaMemcpy(tab.lo.p, lo.data(), lo.size() * 32, cudaMemcpyHostToDevice);
    cudaMemcpy(tab.hi.p, hi.data(), hi.size() * 32, cudaMemcpyHostToDevice);
    return 0;
}

int get_ntt_tab(sb_ctx* c, int L, bool inverse, FrNttTables* out) {
    auto& m = inverse ? c->ntt_inv : c->ntt_fwd;
    auto it = m.find(L);
    if (it == m.end()) {
        NttTab& t = m[L];
        int rc = c->curve == SB_BN254 ? build_ntt_tab<BnFr>(c, L, inverse, t) : build_ntt_tab<BlsFr>(c, L, inverse, t);
        if (rc) { m.erase(L); return fail(c, rc, "ntt table allocation failed"); }
        it = m.find(L);
    }
    out->tw_lo = it->second.lo.p; out->tw_hi = it->second.hi.p; out->h = it->second.h;
    out->wr = inverse ? c->wr_inv.p : c->wr_fwd.p;
    return 0;
}

template <class P> void ninv_bytes(int L, uint8_t* out) {
    typedef Fp<P> F;
    F two = F::add(F::one(), F::one()), n = F::one();
    for (int i = 0; i < L; i++) n = F::mul(n, two);
    F r = F::inv(n); memcpy(out, &r, 32);
}
const void* get_ninv(sb_ctx* c, int L) {
    auto it = c->ninv.find(L);
    if (it == c->ninv.end()) {
        uint8_t b[32];
        if (c->curve == SB_BN254) ninv_bytes<BnFr>(L, b); else ninv_bytes<BlsFr>(L, b);
        DevBuf& d = c->ninv[L];
        if (!d.get(32)) return nullptr;
        cudaMemcpy(d.p, b, 32, cudaMemcpyHostToDevice);
        it = c->ninv.find(L);
    }
    return it->second.p;
}

// plain (non-Montgomery) n^-1 for n = 2^L: the group iFFT scalar
template <class P> void ninv_plain_bytes(int L, uint8_t* out) {
    Fp<P> a; ninv_bytes<P>(L, (uint8_t*)&a); a = Fp<P>::from_mont(a); memcpy(out, &a, 32);
}

// apply-key tables for (n, first, inc): lo[e] = inc^e, hi[e] = first * inc^(e 2^h)
template <class P> int build_pre(sb_ctx* c, uint64_t n, const uint8_t* first, const uint8_t* inc, PreTab& t) {
    typedef Fp<P> F;
    int bits = 0; while (((uint64_t)1 << bits) < n) bits++;
    int h = (bits + 1) / 2;
    F f, i; memcpy(&f, first, 32); memcpy(&i, inc, 32);
    std::vector<F> lo, hi;
    HostFr<P>::pow_tables(i, f, h, (n + ((uint64_t)1 << h) - 1) >> h, lo, hi);
    t.h = h;
    if (!t.lo.get(lo.size() * 32) || !t.hi.get(hi.size() * 32)) return SB_ERR_NOMEM;
    cudaMemcpy(t.lo.p, lo.data(), lo.size() * 32, cudaMemcpyHostToDevice);
    cudaMemcpy(t.hi.p, hi.data(), hi.size() * 32, cudaMemcpyHostToDevice);
    return 0;
}
int get_pre(sb_ctx* c, uint64_t n, const uint8_t* first, const uint8_t* inc, FrPre* out) {
    std::string key((const char*)&n, 8); key.append((const char*)first, 32); key.append((const char*)inc, 32);
    for (PreTab* t : c->pre_cache) if (t->key == key) { out->lo = t->lo.p; out->hi = t->hi.p; out->h = t->h; return 0; }
    PreTab* t = new PreTab(); t->key = key;
    int rc = c->curve == SB_BN254 ? build_pre<BnFr>(c, n, first, inc, *t) : build_pre<BlsFr>(c, n, first, inc, *t);
    if (rc) { delete t; return fail(c, rc, "apply-key table allocation failed"); }
    if (c->pre_cache.size() >= 16) { delete c->pre_cache.front(); c->pre_cache.erase(c->pre_cache.begin()); }
    c->pre_cache.push_back(t);
    out->lo = t->lo.p; out->hi = t->hi.p; out->h = t->h;
    return 0;
}

// affine generators as plain big-endian hex (build/snarkjs.js:9468-9472, 9419-9422 region; 10821-10833 for BLS12-381)
template <class P> void hex_to_mont(const char* hex, uint8_t* out) {
    typedef Fp<P> F; F a = F::zero();
    int len = (int)strlen(hex);
    for (int i = 0; i < len; i++) {
        char ch = hex[len - 1 - i];
        uint32_t d = (ch >= '0' && ch <= '9') ? ch - '0' : (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : ch - 'A' + 10;
        a.v[i / 8] |= d << (4 * (i % 8));
    }
    a = F::to_mont(a); memcpy(out, &a, sizeof a);
}
void init_generators(sb_ctx* c) {
    if (c->curve == SB_BN254) {
        c->gen1.resize(64); c->gen2.resize(128);
        hex_to_mont<BnFq>("1", c->gen1.data()); hex_to_mont<BnFq>("2", c->gen1.data() + 32);
        hex_to_mont<BnFq>("1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed", c->gen2.data());
        hex_to_mont<BnFq>("198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2", c->gen2.data() + 32);
        hex_to_mont<BnFq>("12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa", c->gen2.data() + 64);
        hex_to_mont<BnFq>("090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b", c->gen2.data() + 96);
    } else {
        c->gen1.resize(96); c->gen2.resize(192);
        hex_to_mont<BlsFq>("17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb", c->gen1.data());
        hex_to_mont<BlsFq>("08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1", c->gen1.data() + 48);
        hex_to_mont<BlsFq>("024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8", c->gen2.data());
        hex_to_mont<BlsFq>("13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e", c->gen2.data() + 48);
        hex_to_mont<BlsFq>("0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801", c->gen2.data() + 96);
        hex_to_mont<BlsFq>("0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be", c->gen2.data() + 144);
    }
}

// profiling helpers: accumulate-kernel event pairs
void prof_begin(sb_ctx* c) { c->stats.ev = c->prof_ev; c->stats.nev = 256; c->stats.used = 0; for (double& d : c->stat) d = 0; }
void prof_end(sb_ctx* c) {
    for (int i = 0; i + 1 < c->stats.used; i += 2) {
        float ms = 0; if (cudaEventElapsedTime(&ms, c->prof_ev[i], c->prof_ev[i + 1]) != cudaSuccess) { cudaGetLastError(); continue; }
        const int g = c->stats.tag[i / 2];
        if (g == PROF_ACC_G1) { c->stat[0] += ms; c->stat[2] += 1; c->stat[9] += ms; }
        else if (g == PROF_ACC_G2) { c->stat[1] += ms; c->stat[3] += 1; c->stat[10] += ms; }
        else if (g == PROF_SORT) c->stat[8] += ms;
        else if (g >= PROF_FOLD && g <= PROF_JOIN) c->stat[11 + (g - PROF_FOLD)] += ms;
        else if (g == PROF_FOLD_G2) { c->stat[11] += ms; c->stat[16] += ms; }
        else if (g == PROF_REDUCE_G2) { c->stat[12] += ms; c->stat[17] += ms; }
    }
    c->stats.ev = nullptr; c->stats.used = 0;
}

// Process-wide switches of sb_set_tuning (key 1 is g_msm_force_reduce, msm.cuh).
int g_serial_prove = 0;     // key 2: run every stream of a Groth16 prove call serialised on one stream (per-kernel-class timing)
int g_no_tables = 0;        // key 3: ignore the precomputed window tables
int g_msm_chunk_log = 0;    // key 6: log2 of the points per MSM chunk, 0 = 23 (a test hook)
int g_batch_cap = 0;        // key 14: most proofs (MSM rows) per sub-batch of the batch entries, 0 = as many as memory takes

// Precomputed window tables (msm.cuh k_precompute).  Built for sets of >= 2^12 points whose table index fits the
// 31-bit entry value; g_no_tables disables them (plain windowed Pippenger on the raw bases).
bool want_precomp(sb_ctx* c, uint64_t n) {
    if (g_no_tables || n < (1ull << 12)) return false;
    MsmGeom g = msm_geometry_precomp(n, 32, c->fr_bits);
    return (uint64_t)g.W * n < (1ull << 31);
}
int build_table(sb_ctx* c, const GroupOps& G, const void* d_bases, uint64_t n, void** table, MsmGeom* gp) {
    MsmGeom g = msm_geometry_precomp(n, 32, c->fr_bits);
    cudaError_t e = cudaMalloc(table, (size_t)g.W * n * G.aff_bytes);
    if (e != cudaSuccess) { *table = nullptr; return cuda_fail(c, e, "precompute table allocation"); }
    int rc = G.precompute(d_bases, n, g.c, g.W, *table, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "k_precompute");
    e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return cuda_fail(c, e, "k_precompute");
    *gp = g;
    return 0;
}

void tick(sb_ctx* c, int i) { cudaEventRecord(c->ev[i], c->stream); }
float elapsed(sb_ctx* c, int a, int b) { float ms = 0; cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]); return ms; }

// ------------------------------------------------------------------------------------------------------------
// MSMs over device-resident bases/scalars: sort once, one bucket pipeline, host recombination.
// ------------------------------------------------------------------------------------------------------------
// rows MSMs of n scalars each over one base set (row q's scalars at d_sc + q * n * sb, on the device), sorted and reduced
// together: one sort with MsmGeom::K = rows, one bucket pipeline, one download of the window sums, and each row recombined
// on its own into out (rows x XYZZ, accumulated into).  g is the set's geometry (table mode: the table's, with first and W
// set); rows must not exceed msm_batch_limit, and n one MSM chunk.
int msm_rows_dev(sb_ctx* c, const GroupOps& G, const void* d_bases, const MsmGeom& g, const uint8_t* d_sc, uint32_t sb, uint64_t n,
                 uint32_t rows, uint8_t* out) {
    const size_t wrow = (size_t)msm_wsum_parts(g) * g.windows_per_proof() * G.xyzz_bytes;   // window-sum bytes of one row
    MsmGeom gK = g; gK.K = rows;
    void* d_wsum = c->io[3].get(rows * wrow);
    if (!d_wsum) return fail(c, SB_ERR_NOMEM, "out of device memory");
    MsmSorted srt;
    int rc = msm_sort_entries(d_sc, sb, n, gK, c->sort_scratch, c->stream, &srt, &c->stats);
    if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_sort_entries");
    c->stats.cur_tag = (&G == &c->g1) ? SB_G1 : SB_G2;
    rc = G.buckets(d_bases, srt, c->bucket_scratch, c->stream, d_wsum, &c->stats, nullptr, nullptr);
    if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_buckets");
    std::vector<uint8_t> ws(rows * wrow);
    uint64_t entries = 0;
    CU(c, cudaMemcpyAsync(ws.data(), d_wsum, ws.size(), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(&entries, srt.counts, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    c->stat[(&G == &c->g1) ? 4 : 5] += (double)entries;
    for (uint32_t q = 0; q < rows; q++) G.combine(ws.data() + q * wrow, g, out + (size_t)q * G.xyzz_bytes);
    return 0;
}

// One MSM of any length, chunk by chunk: acc (host XYZZ bytes) += result
int msm_dev_accumulate(sb_ctx* c, const GroupOps& G, const void* d_bases, const uint8_t* d_scalars, uint32_t sbytes, uint64_t n,
                       uint8_t* acc_xyzz, const MsmGeom* gp = nullptr, uint64_t first = 0) {
    const uint64_t MAXC = 1ull << (g_msm_chunk_log > 0 ? g_msm_chunk_log : 23);   // points per MSM chunk
    for (uint64_t off = 0; off < n; off += MAXC) {
        uint64_t cn = std::min(MAXC, n - off);
        MsmGeom g = msm_geometry(cn, sbytes, c->fr_bits);
        if (gp) {   // registered set with precomputed window multiples: d_bases is the table
            g = *gp; g.first = first + off; g.W = (int)((8 * sbytes + 1 + g.c - 1) / g.c);
        }
        int rc = msm_rows_dev(c, G, gp ? d_bases : (const void*)((const uint8_t*)d_bases + off * G.aff_bytes), g, d_scalars + off * sbytes,
                              sbytes, cn, 1, acc_xyzz);
        if (rc) return rc;
    }
    return 0;
}

int msm_host_inputs(sb_ctx* c, int group, const uint8_t* bases, const void* d_bases_opt, const uint8_t* scalars, uint32_t sbytes,
                    uint64_t n, uint8_t* out_jac, uint8_t* out_partial, const MsmGeom* gp = nullptr, uint64_t first = 0) {
    if (!c) return SB_ERR_ARG;
    const GroupOps& G = group == SB_G1 ? c->g1 : c->g2;
    std::vector<uint8_t> acc(G.xyzz_bytes, 0);
    if (n) {
        if (sbytes == 0 || sbytes > 64) return fail(c, SB_ERR_ARG, "Scalar size does not match");
        cudaSetDevice(c->device);
        tick(c, 0);
        const void* d_bases = d_bases_opt;
        if (!d_bases) {
            void* p = c->io[0].get(n * G.aff_bytes);
            if (!p) return fail(c, SB_ERR_NOMEM, "out of device memory");
            CU(c, h2d(c, p, bases, n * G.aff_bytes));
            d_bases = p;
        }
        uint8_t* d_sc = (uint8_t*)c->io[1].get(n * sbytes);
        if (!d_sc) return fail(c, SB_ERR_NOMEM, "out of device memory");
        CU(c, h2d(c, d_sc, scalars, n * sbytes));
        tick(c, 1);
        prof_begin(c);
        int rc = msm_dev_accumulate(c, G, d_bases, d_sc, sbytes, n, acc.data(), gp, first);
        if (rc) return rc;
        tick(c, 2);
        cudaEventSynchronize(c->ev[2]);
        prof_end(c);
        c->last_ms[0] = elapsed(c, 0, 2); c->last_ms[1] = elapsed(c, 0, 1); c->last_ms[2] = elapsed(c, 1, 2);
    }
    if (out_partial) memcpy(out_partial, acc.data(), acc.size());
    if (out_jac) G.to_jacobian(acc.data(), out_jac);
    return 0;
}

void free_key(Groth16Key* k) {
    for (void* p : {k->tA, k->tB1, k->tB2, k->tC, k->tH, k->dA, k->dB1, k->dB2, k->dC, k->dH, (void*)k->d_rowptr, (void*)k->d_sig, k->d_coef, k->dW, k->dWsum})
        if (p) cudaFree(p);
    k->batchW.release(); k->batchX.release(); k->batchY.release();
    delete k;
}

template <class PR> static void fr_from_mont_bytes(const uint8_t* in, uint8_t* out) { Fp<PR> a; memcpy(&a, in, 32); a = Fp<PR>::from_mont(a); memcpy(out, &a, 32); }
template <class PR> static void fr_neg_mul_bytes(const uint8_t* r, const uint8_t* s, uint8_t* out) { Fp<PR> a, b; memcpy(&a, r, 32); memcpy(&b, s, 32); a = Fp<PR>::neg(Fp<PR>::mul(a, b)); memcpy(out, &a, 32); }

}  // namespace

// ================================================================================================================
extern "C" {

const char* sb_version(void) { return "snarkb200 0.2 (sm_90a)"; }
int sb_comm_destroy(sb_ctx* c);

int sb_create(int curve, int device_id, sb_ctx** out) {
    if (!out || (curve != SB_BN254 && curve != SB_BLS12_381)) return SB_ERR_ARG;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return SB_ERR_NODEVICE;
    if (device_id < 0 || device_id >= ndev) return SB_ERR_ARG;
    if (cudaSetDevice(device_id) != cudaSuccess) return SB_ERR_CUDA;
    sb_ctx* c = new sb_ctx();
    c->curve = curve; c->device = device_id;
    c->n8q = curve == SB_BN254 ? 32 : 48;
    c->fr_bits = curve == SB_BN254 ? 254 : 255;
    if (curve == SB_BN254) { c->g1 = SB_GROUP_OPS(bn254_g1, 64); c->g2 = SB_GROUP_OPS(bn254_g2, 128); }
    else { c->g1 = SB_GROUP_OPS(bls12381_g1, 96); c->g2 = SB_GROUP_OPS(bls12381_g2, 192); }
    if (cudaStreamCreate(&c->stream) != cudaSuccess) { delete c; return SB_ERR_CUDA; }
    for (auto& e : c->ev) cudaEventCreate(&e);
    for (auto& e : c->prof_ev) cudaEventCreate(&e);
    for (auto& e : c->pev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    // The side streams take the main stream's priority: a higher one lets every latency-bound tail CTA take the SM slot
    // of a retiring accumulation CTA ahead of the accumulation's next block, which stretches the accumulation by the
    // tail's full length (2^20 Groth16 proof, H100 at 700 W: 41.2 proofs/s with high-priority side streams, 42.0-42.3
    // without; DESIGN §7).  At equal priority the tails fill the slots the accumulation leaves in its last wave.
    for (auto& st : c->aux) cudaStreamCreate(&st);
    if (cudaHostAlloc((void**)&c->pinned, 256 * 1024, cudaHostAllocDefault) != cudaSuccess) c->pinned = nullptr;
    else c->pinned_bytes = 256 * 1024;
    for (int i = 0; i < 2; i++) { if (cudaHostAlloc((void**)&c->stage[i], STAGE_BYTES, cudaHostAllocDefault) != cudaSuccess) c->stage[i] = nullptr; cudaEventCreateWithFlags(&c->stage_ev[i], cudaEventDisableTiming); }
    init_generators(c);
    int rc = curve == SB_BN254 ? init_roots<BnFr>(c) : init_roots<BlsFr>(c);
    if (rc == 0 && fr_configure(curve) != 0) rc = SB_ERR_CUDA;
    if (rc) { sb_destroy(c); return rc; }
    *out = c;
    return SB_OK;
}

void sb_destroy(sb_ctx* c) {
    if (!c) return;
    sb_comm_destroy(c);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (auto* k : c->keys) if (k) free_key(k);
    for (auto* k : c->plonk_keys) if (k) plonk_free_key(k);
    for (auto* k : c->fflonk_keys) if (k) fflonk_free_key(k);
    for (auto& b : c->bases) { if (b.d) cudaFree(b.d); if (b.table) cudaFree(b.table); }
    for (auto* t : c->pre_cache) { t->lo.release(); t->hi.release(); delete t; }
    for (auto& kv : c->ntt_fwd) { kv.second.lo.release(); kv.second.hi.release(); }
    for (auto& kv : c->ntt_inv) { kv.second.lo.release(); kv.second.hi.release(); }
    for (auto& kv : c->ninv) kv.second.release();
    c->wr_fwd.release(); c->wr_inv.release();
    for (auto& b : c->io) b.release();
    c->sort_scratch.release(); c->bucket_scratch.release();
    for (auto& e : c->ev) cudaEventDestroy(e);
    for (auto& e : c->prof_ev) cudaEventDestroy(e);
    for (auto& e : c->pev) cudaEventDestroy(e);
    for (auto& st : c->aux) { if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); } }
    if (c->pinned) cudaFreeHost(c->pinned);
    for (int i = 0; i < 2; i++) { if (c->stage[i]) cudaFreeHost(c->stage[i]); cudaEventDestroy(c->stage_ev[i]); }
    c->sort_scratch2.release(); for (auto& b : c->bscr) b.release();
    cudaStreamDestroy(c->stream);
    delete c;
}

const char* sb_last_error(sb_ctx* c) {
    if (!c) return "null context";
    if (t_err_ctx == c) return t_err.c_str();
    SB_LOCK(c); t_err_ctx = c; t_err = c->err; return t_err.c_str();
}
uint64_t sb_launch_count(sb_ctx* c) { SB_LOCK(c); return c ? c->launches + (uint64_t)c->stats.launches : 0; }
float sb_last_ms(sb_ctx* c, int which) { SB_LOCK(c); return (c && which >= 0 && which < 8) ? c->last_ms[which] : 0.f; }
int sb_sync(sb_ctx* c) { SB_LOCK(c); if (!c) return SB_ERR_ARG; cudaSetDevice(c->device); CU(c, cudaStreamSynchronize(c->stream)); return 0; }

int sb_msm_g1_affine(sb_ctx* c, const uint8_t* bases, const uint8_t* scalars, uint32_t sb, uint64_t n, uint8_t* out) { SB_LOCK(c);
    return msm_host_inputs(c, SB_G1, bases, nullptr, scalars, sb, n, out, nullptr);
}
int sb_msm_g2_affine(sb_ctx* c, const uint8_t* bases, const uint8_t* scalars, uint32_t sb, uint64_t n, uint8_t* out) { SB_LOCK(c);
    return msm_host_inputs(c, SB_G2, bases, nullptr, scalars, sb, n, out, nullptr);
}

int sb_bases_register(sb_ctx* c, int group, const uint8_t* bases, uint64_t n, uint64_t* handle) { SB_LOCK(c);
    if (!c || !handle || (group != SB_G1 && group != SB_G2)) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    const GroupOps& G = group == SB_G1 ? c->g1 : c->g2;
    BaseSet b; b.group = group; b.n = n;
    CU(c, cudaMalloc(&b.d, n ? n * G.aff_bytes : 16));
    CU(c, cudaMemcpy(b.d, bases, n * G.aff_bytes, cudaMemcpyHostToDevice));
    if (want_precomp(c, n)) { int rc = build_table(c, G, b.d, n, &b.table, &b.gp); if (rc) { cudaFree(b.d); return rc; } }
    c->bases.push_back(b);
    *handle = c->bases.size();
    return 0;
}
int sb_bases_release(sb_ctx* c, uint64_t h) { SB_LOCK(c);
    if (!c || h == 0 || h > c->bases.size() || !c->bases[h - 1].d) return fail(c, SB_ERR_ARG, "invalid bases handle");
    cudaSetDevice(c->device);
    cudaFree(c->bases[h - 1].d); c->bases[h - 1].d = nullptr; c->bases[h - 1].n = 0;
    if (c->bases[h - 1].table) { cudaFree(c->bases[h - 1].table); c->bases[h - 1].table = nullptr; }
    return 0;
}
static int msm_registered_impl(sb_ctx* c, uint64_t h, uint64_t first, const uint8_t* scalars, uint32_t sb, uint64_t n, uint8_t* out, uint8_t* partial) {
    if (!c || h == 0 || h > c->bases.size() || !c->bases[h - 1].d) return fail(c, SB_ERR_ARG, "invalid bases handle");
    const BaseSet& b = c->bases[h - 1];
    if (first + n > b.n) return fail(c, SB_ERR_ARG, "registered base range out of bounds");
    const GroupOps& G = b.group == SB_G1 ? c->g1 : c->g2;
    if (b.table && sb >= 1 && sb <= 32)
        return msm_host_inputs(c, b.group, nullptr, b.table, scalars, sb, n, out, partial, &b.gp, first);
    return msm_host_inputs(c, b.group, nullptr, (const uint8_t*)b.d + first * G.aff_bytes, scalars, sb, n, out, partial);
}
int sb_msm_registered(sb_ctx* c, uint64_t h, uint64_t first, const uint8_t* scalars, uint32_t sb, uint64_t n, uint8_t* out) { SB_LOCK(c);
    return msm_registered_impl(c, h, first, scalars, sb, n, out, nullptr);
}
int sb_msm_registered_partial(sb_ctx* c, uint64_t h, uint64_t first, const uint8_t* scalars, uint32_t sb, uint64_t n, uint8_t* partial) { SB_LOCK(c);
    return msm_registered_impl(c, h, first, scalars, sb, n, nullptr, partial);
}
// A fixed set of host threads draining one FIFO of tasks: the host work of a Groth16 batch (fixed parts, recombination,
// assembly) never runs on more threads than the machine has cores, however many sub-batches are in flight.  The destructor
// runs whatever is still queued before it joins, so tasks may reference locals declared before the pool.
class HostPool {
public:
    explicit HostPool(unsigned n) { for (unsigned i = 0; i < std::max(1u, n); i++) th_.emplace_back([this]() { run(); }); }
    ~HostPool() {
        { std::lock_guard<std::mutex> l(mu_); stop_ = true; }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    void submit(std::function<void()> f) {
        { std::lock_guard<std::mutex> l(mu_); q_.push_back(std::move(f)); pending_++; }
        cv_.notify_one();
    }
    void wait() { std::unique_lock<std::mutex> l(mu_); idle_.wait(l, [this]() { return pending_ == 0; }); }
private:
    void run() {
        for (;;) {
            std::function<void()> f;
            { std::unique_lock<std::mutex> l(mu_);
              cv_.wait(l, [this]() { return stop_ || !q_.empty(); });
              if (q_.empty()) return;
              f = std::move(q_.front()); q_.pop_front(); }
            f();
            { std::lock_guard<std::mutex> l(mu_); if (--pending_ == 0) idle_.notify_all(); }
        }
    }
    std::mutex mu_; std::condition_variable cv_, idle_;
    std::deque<std::function<void()>> q_; size_t pending_ = 0; bool stop_ = false;
    std::vector<std::thread> th_;
};

// Device bytes of one MSM over `entries` sorted (digit, point) entries into `buckets` buckets of `xb`-byte points: keys and
// values double-buffered and about as much again for the radix sort's temporary storage (20 B per entry), the buckets, the
// accumulation's head partials (<= one per 16 entries) with their keys, and the reduction's scratch (< 1/4 of the buckets).
static size_t msm_batch_bytes(uint64_t entries, uint64_t buckets, size_t xb) {
    return (size_t)(buckets + buckets / 4 + entries / 16 + 64) * xb + entries / 2;
}
static size_t sort_batch_bytes(uint64_t entries) { return (size_t)entries * 20; }

// Proofs (or MSM rows) per sub-batch: what the 32-bit bucket keys allow, what fits in 85 % of the free device memory plus
// what the context's grow-only buffers already hold (they are reallocated, not added), and the sb_set_tuning(14) cap.
static uint32_t batch_size(sb_ctx* c, uint32_t count, uint64_t key_limit, size_t per_item, size_t held) {
    uint64_t kb = std::min<uint64_t>(count, key_limit);
    if (g_batch_cap > 0) kb = std::min<uint64_t>(kb, (uint64_t)g_batch_cap);
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
    held += c->sort_scratch.cap + c->sort_scratch2.cap + c->bucket_scratch.cap;
    for (const MsmScratch& b : c->bscr) held += b.cap;
    const size_t budget = (size_t)((double)(free_b + held) * 0.85);
    kb = std::min<uint64_t>(kb, budget / std::max<size_t>(per_item, 1));
    return (uint32_t)std::max<uint64_t>(kb, 1);
}

// count MSMs over the same registered bases: the rows are sorted and reduced together in sub-batches (MsmGeom::K), each row
// recombined on its own.  Rows longer than an MSM chunk (2^23 points) go one by one through sb_msm_registered's path.
int sb_msm_registered_batch(sb_ctx* c, uint64_t h, uint64_t first, const uint8_t* scalars, uint32_t sb, uint64_t n, uint32_t count, uint8_t* out) { SB_LOCK(c);
    if (!c || h == 0 || h > c->bases.size() || !c->bases[h - 1].d) return fail(c, SB_ERR_ARG, "invalid bases handle");
    const BaseSet& b = c->bases[h - 1];
    if (first + n > b.n) return fail(c, SB_ERR_ARG, "registered base range out of bounds");
    if (count == 0) return SB_OK;
    if (!out || (n && !scalars)) return fail(c, SB_ERR_ARG, "null argument");
    const GroupOps& G = b.group == SB_G1 ? c->g1 : c->g2;
    const size_t jb = (size_t)3 * (G.aff_bytes / 2);   // normalised Jacobian output point
    std::vector<uint8_t> acc(G.xyzz_bytes, 0);
    if (n == 0) { for (uint32_t i = 0; i < count; i++) G.to_jacobian(acc.data(), out + i * jb); return SB_OK; }
    if (sb == 0 || sb > 64) return fail(c, SB_ERR_ARG, "Scalar size does not match");
    cudaSetDevice(c->device);
    const uint64_t MAXC = 1ull << (g_msm_chunk_log > 0 ? g_msm_chunk_log : 23);
    if (n > MAXC) {
        tick(c, 4);
        for (uint32_t i = 0; i < count; i++) { int rc = msm_registered_impl(c, h, first, scalars + (size_t)i * n * sb, sb, n, out + i * jb, nullptr); if (rc) return rc; }
        tick(c, 5); cudaEventSynchronize(c->ev[5]); c->last_ms[0] = elapsed(c, 4, 5);
        return SB_OK;
    }
    const bool table = b.table && sb <= 32;
    MsmGeom g = msm_geometry(n, sb, c->fr_bits);
    if (table) { g = b.gp; g.first = first; g.W = (int)((8 * sb + 1 + g.c - 1) / g.c); }
    const void* d_bases = table ? b.table : (const void*)((const uint8_t*)b.d + first * G.aff_bytes);
    const uint64_t e = n * (uint64_t)g.W;
    const size_t per_row = (size_t)n * sb + sort_batch_bytes(e) + msm_batch_bytes(e, (uint64_t)g.windows_per_proof() * g.B, G.xyzz_bytes);
    const uint32_t KB = batch_size(c, count, msm_batch_limit(n, g.c, g.W, g.precomp), per_row, c->io[1].cap + c->io[3].cap);
    std::vector<uint8_t> sums((size_t)KB * G.xyzz_bytes);
    tick(c, 0);
    prof_begin(c);
    for (uint32_t r0 = 0; r0 < count; r0 += KB) {
        const uint32_t kb = std::min(KB, count - r0);
        std::fill(sums.begin(), sums.end(), 0);
        uint8_t* d_sc = (uint8_t*)c->io[1].get((size_t)kb * n * sb);
        if (!d_sc) return fail(c, SB_ERR_NOMEM, "out of device memory");
        CU(c, h2d(c, d_sc, scalars + (size_t)r0 * n * sb, (size_t)kb * n * sb));
        int rc = msm_rows_dev(c, G, d_bases, g, d_sc, sb, n, kb, sums.data());
        if (rc) return rc;
        for (uint32_t q = 0; q < kb; q++) G.to_jacobian(sums.data() + (size_t)q * G.xyzz_bytes, out + (size_t)(r0 + q) * jb);
    }
    tick(c, 1);
    CU(c, cudaEventSynchronize(c->ev[1]));
    prof_end(c);
    c->last_ms[0] = elapsed(c, 0, 1);
    return SB_OK;
}
uint32_t sb_msm_partial_bytes(sb_ctx* c, int group) { return c ? (group == SB_G1 ? c->g1.xyzz_bytes : c->g2.xyzz_bytes) : 0; }
int sb_msm_sum_partials(sb_ctx* c, int group, const uint8_t* partials, int count, uint8_t* out) { SB_LOCK(c);
    if (!c || (group != SB_G1 && group != SB_G2) || count < 0) return SB_ERR_ARG;
    const GroupOps& G = group == SB_G1 ? c->g1 : c->g2;
    std::vector<uint8_t> acc(G.xyzz_bytes, 0);
    for (int i = 0; i < count; i++) G.add(acc.data(), partials + (size_t)i * G.xyzz_bytes);
    G.to_jacobian(acc.data(), out);
    return 0;
}

int sb_msm_dev(sb_ctx* c, int group, const void* bases_dev, const void* scalars_dev, uint32_t sb, uint64_t n, uint8_t* out) { SB_LOCK(c);
    if (!c || (group != SB_G1 && group != SB_G2)) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    const GroupOps& G = group == SB_G1 ? c->g1 : c->g2;
    std::vector<uint8_t> acc(G.xyzz_bytes, 0);
    tick(c, 0);
    prof_begin(c);
    if (n) { int rc = msm_dev_accumulate(c, G, bases_dev, (const uint8_t*)scalars_dev, sb, n, acc.data()); if (rc) return rc; }
    tick(c, 1); cudaEventSynchronize(c->ev[1]); c->last_ms[0] = elapsed(c, 0, 1);
    prof_end(c);
    G.to_jacobian(acc.data(), out);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- Fr ops
static int ntt_dev(sb_ctx* c, void* a, void* b, uint64_t n, int inverse, const FrPre* pre, bool scale, void** result) {
    if (n == 0 || (n & (n - 1))) return fail(c, SB_ERR_ARG, "fft must be multiple of 2");
    int L = 0; while (((uint64_t)1 << L) < n) L++;
    if (L > c->fr_s) return fail(c, SB_ERR_ARG, "fft size exceeds the 2-adicity of Fr (fftExt path not supported)");
    if (L == 0) { *result = a; return 0; }
    FrNttTables tb;
    int rc = get_ntt_tab(c, L, inverse != 0, &tb); if (rc) return rc;
    const void* post = nullptr;
    if (inverse && scale) { post = get_ninv(c, L); if (!post) return fail(c, SB_ERR_NOMEM, "out of device memory"); }
    int launches = 0;
    ProfScope pn(&c->stats, PROF_NTT, c->stream);
    rc = fr_ntt(c->curve, a, b, L, &tb, pre, post, c->stream, result, &launches);
    pn.end();
    c->launches += launches;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_ntt");
    return 0;
}

int sb_ntt_fr(sb_ctx* c, const uint8_t* in, uint64_t n, int inverse, uint8_t* out) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (n == 0 || (n & (n - 1))) return fail(c, SB_ERR_ARG, "fft must be multiple of 2");
    cudaSetDevice(c->device);
    void* a = c->io[0].get(n * 32); void* b = c->io[1].get(n * 32);
    if (!a || !b) return fail(c, SB_ERR_NOMEM, "out of device memory");
    tick(c, 0);
    CU(c, h2d(c, a, in, n * 32));
    tick(c, 1);
    void* res = nullptr;
    int rc = ntt_dev(c, a, b, n, inverse, nullptr, true, &res); if (rc) return rc;
    tick(c, 2);
    CU(c, d2h(c, out, res, n * 32));
    tick(c, 3);
    CU(c, cudaStreamSynchronize(c->stream));
    c->last_ms[0] = elapsed(c, 0, 3); c->last_ms[1] = elapsed(c, 0, 1); c->last_ms[2] = elapsed(c, 1, 2); c->last_ms[3] = elapsed(c, 2, 3);
    return 0;
}
int sb_ntt_fr_dev(sb_ctx* c, void* data, void* scratch, uint64_t n, int inverse, void** result) { SB_LOCK(c);
    if (!c || !result) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    tick(c, 0);
    int rc = ntt_dev(c, data, scratch, n, inverse, nullptr, true, result); if (rc) return rc;
    tick(c, 1);
    CU(c, cudaStreamSynchronize(c->stream));
    c->last_ms[0] = elapsed(c, 0, 1);
    return 0;
}

int sb_fr_batch_apply_key(sb_ctx* c, const uint8_t* in, uint64_t n, const uint8_t first[32], const uint8_t inc[32], uint8_t* out) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (n == 0) return 0;
    cudaSetDevice(c->device);
    FrPre pre; int rc = get_pre(c, n, first, inc, &pre); if (rc) return rc;
    void* a = c->io[0].get(n * 32); void* b = c->io[1].get(n * 32);
    if (!a || !b) return fail(c, SB_ERR_NOMEM, "out of device memory");
    CU(c, h2d(c, a, in, n * 32));
    rc = fr_apply_key(c->curve, a, b, n, &pre, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_apply_key");
    CU(c, d2h(c, out, b, n * 32));
    return 0;
}
static int convert_impl(sb_ctx* c, const uint8_t* in, uint64_t n, uint8_t* out, int to_mont) {
    if (!c) return SB_ERR_ARG;
    if (n == 0) return 0;
    cudaSetDevice(c->device);
    void* a = c->io[0].get(n * 32); void* b = c->io[1].get(n * 32);
    if (!a || !b) return fail(c, SB_ERR_NOMEM, "out of device memory");
    CU(c, h2d(c, a, in, n * 32));
    int rc = fr_convert(c->curve, a, b, n, to_mont, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_convert");
    CU(c, d2h(c, out, b, n * 32));
    return 0;
}
int sb_fr_batch_to_montgomery(sb_ctx* c, const uint8_t* in, uint64_t n, uint8_t* out) { SB_LOCK(c); return convert_impl(c, in, n, out, 1); }
int sb_fr_batch_from_montgomery(sb_ctx* c, const uint8_t* in, uint64_t n, uint8_t* out) { SB_LOCK(c); return convert_impl(c, in, n, out, 0); }

int sb_qap_join_abc(sb_ctx* c, const uint8_t* a, const uint8_t* b, const uint8_t* cc, uint64_t n, uint8_t* out) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (n == 0) return 0;
    cudaSetDevice(c->device);
    void* da = c->io[0].get(n * 32); void* db = c->io[1].get(n * 32); void* dc = c->io[2].get(n * 32); void* dout = c->io[3].get(n * 32);
    if (!da || !db || !dc || !dout) return fail(c, SB_ERR_NOMEM, "out of device memory");
    CU(c, h2d(c, da, a, n * 32));
    CU(c, h2d(c, db, b, n * 32));
    CU(c, h2d(c, dc, cc, n * 32));
    int rc = fr_join_abc(c->curve, da, db, dc, dout, n, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_join_abc");
    CU(c, d2h(c, out, dout, n * 32));
    return 0;
}

// ---------------------------------------------------------------------------------------------------- group FFT
// plain Fr values first * inc^i, i < n, into d_out (d_tmp: n more elements): the apply-key kernel over Montgomery ones,
// then out of Montgomery form (first, inc Montgomery)
static int fr_powers_plain(sb_ctx* c, uint64_t n, const uint8_t* first, const uint8_t* inc, void* d_tmp, void* d_out) {
    FrPre pre; int rc = get_pre(c, n, first, inc, &pre); if (rc) return rc;
    uint8_t* o = (uint8_t*)d_out;
    CU(c, cudaMemcpyAsync(o, c->roots[0].data(), 32, cudaMemcpyHostToDevice, c->stream));        // w[0] = Montgomery one
    for (uint64_t k = 1; k < n; k *= 2) CU(c, cudaMemcpyAsync(o + k * 32, o, std::min(k, n - k) * 32, cudaMemcpyDeviceToDevice, c->stream));
    rc = fr_apply_key(c->curve, d_out, d_tmp, n, &pre, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_apply_key");
    rc = fr_convert(c->curve, d_tmp, d_out, n, 0, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_convert");
    return 0;
}
static void* io_get(sb_ctx* c, int i, uint64_t bytes, int* rc) {
    void* p = c->io[i].get(bytes);
    if (!p) *rc = fail(c, SB_ERR_NOMEM, "out of device memory (" + std::to_string(bytes) + " bytes)");
    return p;
}
static int group_ops(sb_ctx* c, int group, const GroupOps** G) {
    if (!c || (group != SB_G1 && group != SB_G2)) return c ? fail(c, SB_ERR_ARG, "invalid group") : SB_ERR_ARG;
    *G = group == SB_G1 ? &c->g1 : &c->g2;
    return 0;
}

int sb_group_fft(sb_ctx* c, int group, const uint8_t* in, int in_jac, uint64_t n, int inverse, int out_jac, uint8_t* out) { SB_LOCK(c);
    const GroupOps* G; int rc = group_ops(c, group, &G); if (rc) return rc;
    if (n == 0 || (n & (n - 1))) return fail(c, SB_ERR_ARG, "fft must be multiple of 2");
    int L = 0; while (((uint64_t)1 << L) < n) L++;
    if (L > c->fr_s) return fail(c, SB_ERR_ARG, "fft size exceeds the 2-adicity of Fr (fftExt path not supported)");
    cudaSetDevice(c->device);
    const uint64_t n8 = G->aff_bytes / 2, sin = (in_jac ? 3 : 2) * n8, sout = (out_jac ? 3 : 2) * n8, ntw = std::max<uint64_t>(n / 2, 1);
    uint8_t* d_io = (uint8_t*)io_get(c, 0, n * std::max(sin, sout), &rc);
    void* d_pts = d_io ? io_get(c, 1, n * G->xyzz_bytes, &rc) : nullptr;
    uint8_t* d_tw = d_pts ? (uint8_t*)io_get(c, 2, (ntw + 1) * 32, &rc) : nullptr;
    void* d_tmp = d_tw ? io_get(c, 3, ntw * 32, &rc) : nullptr;
    if (!d_tmp) return rc;
    tick(c, 0);
    CU(c, h2d(c, d_io, in, n * sin));
    tick(c, 1);
    if (L > 1) { rc = fr_powers_plain(c, n / 2, c->roots[0].data(), c->roots[L].data(), d_tmp, d_tw); if (rc) return rc; }
    uint8_t* d_ninv = nullptr;
    if (inverse) {
        uint8_t b[32];
        if (c->curve == SB_BN254) ninv_plain_bytes<BnFr>(L, b); else ninv_plain_bytes<BlsFr>(L, b);
        d_ninv = d_tw + ntw * 32;
        CU(c, cudaMemcpyAsync(d_ninv, b, 32, cudaMemcpyHostToDevice, c->stream));
    }
    int launches = 0;
    rc = G->gfft(d_io, in_jac, n, L, d_tw, d_ninv, out_jac, d_pts, d_io, c->stream, &launches);
    c->launches += launches;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "group fft");
    tick(c, 2);
    CU(c, d2h(c, out, d_io, n * sout));
    tick(c, 3);
    CU(c, cudaStreamSynchronize(c->stream));
    c->last_ms[0] = elapsed(c, 0, 3); c->last_ms[1] = elapsed(c, 0, 1); c->last_ms[2] = elapsed(c, 1, 2); c->last_ms[3] = elapsed(c, 2, 3);
    return 0;
}

int sb_group_batch_apply_key(sb_ctx* c, int group, const uint8_t* in, int in_jac, uint64_t n, const uint8_t first[32],
                             const uint8_t inc[32], int out_jac, uint8_t* out) { SB_LOCK(c);
    const GroupOps* G; int rc = group_ops(c, group, &G); if (rc) return rc;
    c->last_ms[0] = 0;
    if (n == 0) return 0;
    cudaSetDevice(c->device);
    const uint64_t n8 = G->aff_bytes / 2, sin = (in_jac ? 3 : 2) * n8, sout = (out_jac ? 3 : 2) * n8;
    void* d_in = io_get(c, 0, n * sin, &rc);
    void* d_out = d_in ? io_get(c, 1, n * sout, &rc) : nullptr;
    void* d_sc = d_out ? io_get(c, 2, n * 32, &rc) : nullptr;
    void* d_tmp = d_sc ? io_get(c, 3, n * 32, &rc) : nullptr;
    if (!d_tmp) return rc;
    tick(c, 0);
    CU(c, h2d(c, d_in, in, n * sin));
    tick(c, 1);
    rc = fr_powers_plain(c, n, first, inc, d_tmp, d_sc); if (rc) return rc;
    rc = G->gapply(d_in, in_jac, d_sc, n, out_jac, d_out, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "group batchApplyKey");
    tick(c, 2);
    CU(c, d2h(c, out, d_out, n * sout));
    tick(c, 3);
    CU(c, cudaStreamSynchronize(c->stream));
    c->last_ms[0] = elapsed(c, 0, 3); c->last_ms[1] = elapsed(c, 0, 1); c->last_ms[2] = elapsed(c, 1, 2); c->last_ms[3] = elapsed(c, 2, 3);
    return 0;
}

int sb_fr_root(sb_ctx* c, int what, uint8_t out[32]) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (what == -1) memcpy(out, c->shift.data(), 32);
    else if (what == -2) memcpy(out, c->nqr.data(), 32);
    else if (what >= 0 && what <= c->fr_s) memcpy(out, c->roots[what].data(), 32);
    else return fail(c, SB_ERR_ARG, "root index out of range");
    return c->fr_s;
}

int sb_set_tuning(int key, int value) {
    switch (key) {
    case 1: if (value != 0 && value != 1) return SB_ERR_ARG; g_msm_force_reduce = value; return 0;   // bucket reduction
    case 2: g_serial_prove = value; return 0;                                                           // serialised prove call
    case 3: g_no_tables = value; return 0;                                                              // no window tables
    case 6: if (value < 0 || value > 23) return SB_ERR_ARG; g_msm_chunk_log = value; return 0;         // MSM chunk size
    case 7: if (value < 10 || value > 12) return SB_ERR_ARG; g_ntt_tile_log = value; return 0;         // NTT tile size
    case 8: g_stage_enabled = value; return 0;                                                          // pinned staging of pageable buffers
    case 13: if (value != 0 && (value < 3 || value > 22)) return SB_ERR_ARG; g_msm_force_c = value; return 0;   // MSM window bits
    case 14: if (value < 0) return SB_ERR_ARG; g_batch_cap = value; return 0;                                    // proofs per sub-batch
    default: return SB_ERR_ARG;
    }
}
double sb_last_stat(sb_ctx* c, int which) { SB_LOCK(c); return (c && which >= 0 && which < 18) ? c->stat[which] : 0.0; }
double sb_calibrate(sb_ctx* c, int what) { SB_LOCK(c); if (!c) return -1; cudaSetDevice(c->device); return calibrate(what, c->stream); }
int sb_gen_points(sb_ctx* c, int group, uint64_t seed, uint64_t n, uint8_t* out) { SB_LOCK(c);
    if (!c || (group != SB_G1 && group != SB_G2)) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    const GroupOps& G = group == SB_G1 ? c->g1 : c->g2;
    void* d = c->io[0].get(n * G.aff_bytes);
    if (!d) return fail(c, SB_ERR_NOMEM, "out of device memory");
    int rc = G.gen_points(group == SB_G1 ? c->gen1.data() : c->gen2.data(), seed, n, d, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "gen_points");
    CU(c, d2h(c, out, d, n * G.aff_bytes));
    return 0;
}
int sb_field_eval(sb_ctx* c, int field, int op, const uint8_t* in, uint64_t n, uint8_t* out) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    int wi, wo;
    if (field_eval_shape(field, op, &wi, &wo)) return fail(c, SB_ERR_ARG, "sb_field_eval: op " + std::to_string(op) + " is not defined on field " + std::to_string(field));
    if (n == 0) return 0;
    cudaSetDevice(c->device);
    void* d_in = c->io[0].get(n * wi * 4); void* d_out = c->io[1].get(n * wo * 4);
    if (!d_in || !d_out) return fail(c, SB_ERR_NOMEM, "out of device memory");
    CU(c, h2d(c, d_in, in, n * wi * 4));
    int rc = field_eval(field, op, d_in, d_out, n, c->stream); c->launches++;
    if (rc) return cuda_fail(c, (cudaError_t)rc, "field_eval");
    CU(c, d2h(c, out, d_out, n * wo * 4));
    return 0;
}
// The NTT launches the provers make, on host data.  One device region holds the post-scale, then each input and scratch area
// (per transform in layout 0, one for all in layout 1) with a guard of NTT_EVAL_GUARD sentinel elements after every part, so
// that a launch reading another slot's data corrupts a neighbour instead of landing on the right bytes by chance, and a write
// outside the areas is reported.
static constexpr uint64_t NTT_EVAL_GUARD = 61;
int sb_ntt_eval(sb_ctx* c, int L, int count, int layout, int inverse, const uint8_t* pre_first, const uint8_t* pre_inc,
                const uint8_t* post_scale, const uint8_t* in, uint8_t* out) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (L < 0 || L > c->fr_s) return fail(c, SB_ERR_ARG, "sb_ntt_eval: L must be in 0..Fr.s");
    if (layout != 0 && layout != 1) return fail(c, SB_ERR_ARG, "sb_ntt_eval: layout must be 0 (by pointer) or 1 (strided)");
    if (count < 1 || count > (layout ? 65535 : 4)) return fail(c, SB_ERR_ARG, "sb_ntt_eval: count must be in 1..4 (layout 0) or 1..65535 (layout 1)");
    if (!in || !out || !pre_first != !pre_inc) return fail(c, SB_ERR_ARG, "sb_ntt_eval: null argument");
    cudaSetDevice(c->device);
    const uint64_t n = 1ull << L, G = NTT_EVAL_GUARD;
    const uint64_t span = layout ? (uint64_t)count * n : n;   // elements of one input or scratch area
    const int areas = layout ? 1 : count;
    const uint64_t total = 1 + G + 2 * (uint64_t)areas * (span + G);
    uint8_t* d = (uint8_t*)c->io[0].get(total * 32);
    if (!d) return fail(c, SB_ERR_NOMEM, "out of device memory");
    auto area = [&](int k, int scratch) { return d + (1 + G + (2 * (uint64_t)k + scratch) * (span + G)) * 32; };
    CU(c, cudaMemsetAsync(d, 0xA5, total * 32, c->stream));
    for (int k = 0; k < areas; k++) CU(c, h2d(c, area(k, 0), in + (uint64_t)k * span * 32, span * 32));
    if (post_scale) CU(c, cudaMemcpyAsync(d, post_scale, 32, cudaMemcpyHostToDevice, c->stream));
    FrNttTables tb;
    int rc = get_ntt_tab(c, L, inverse != 0, &tb); if (rc) return rc;
    FrPre pre;
    if (pre_first) { rc = get_pre(c, n, pre_first, pre_inc, &pre); if (rc) return rc; }
    int side = 0, launches = 0;
    if (layout == 0) {
        void* a[4]; void* b[4];
        for (int k = 0; k < 4; k++) { a[k] = area(k < count ? k : 0, 0); b[k] = area(k < count ? k : 0, 1); }
        rc = fr_ntt_batch(c->curve, a, b, count, L, &tb, pre_first ? &pre : nullptr, post_scale ? d : nullptr, c->stream, &side, &launches);
    } else {
        rc = fr_ntt_strided(c->curve, area(0, 0), area(0, 1), count, L, &tb, pre_first ? &pre : nullptr, post_scale ? d : nullptr, c->stream, &side, &launches);
    }
    c->launches += launches;
    if (rc) return cuda_fail(c, (cudaError_t)rc, layout ? "fr_ntt_strided" : "fr_ntt_batch");
    std::vector<uint8_t> h(total * 32);
    CU(c, d2h(c, h.data(), d, total * 32));
    for (int k = 0; k <= 2 * areas; k++) {   // the guard after the post-scale slot and after every area
        const uint8_t* g = h.data() + (k ? (1 + G + (uint64_t)k * (span + G) - G) : 1) * 32;
        for (uint64_t i = 0; i < G * 32; i++)
            if (g[i] != 0xA5) return fail(c, SB_ERR_CUDA, "sb_ntt_eval: a launch wrote outside its transforms");
    }
    for (int k = 0; k < areas; k++) memcpy(out + (uint64_t)k * span * 32, h.data() + (area(k, side) - d), span * 32);
    return 0;
}
int sb_generator(sb_ctx* c, int group, uint8_t* out) { SB_LOCK(c);
    if (!c || (group != SB_G1 && group != SB_G2)) return SB_ERR_ARG;
    const std::vector<uint8_t>& g = group == SB_G1 ? c->gen1 : c->gen2;
    memcpy(out, g.data(), g.size()); return 0;
}

void* sb_dev_alloc(sb_ctx* c, uint64_t bytes) { SB_LOCK(c); if (!c) return nullptr; cudaSetDevice(c->device); void* p = nullptr; if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) return nullptr; return p; }
int sb_dev_free(sb_ctx* c, void* p) { SB_LOCK(c); if (!c) return SB_ERR_ARG; cudaSetDevice(c->device); CU(c, cudaFree(p)); return 0; }
int sb_dev_upload(sb_ctx* c, void* dst, const uint8_t* src, uint64_t bytes) { SB_LOCK(c); if (!c) return SB_ERR_ARG; cudaSetDevice(c->device); CU(c, h2d(c, dst, src, bytes)); CU(c, cudaStreamSynchronize(c->stream)); return 0; }
int sb_dev_download(sb_ctx* c, uint8_t* dst, const void* src, uint64_t bytes) { SB_LOCK(c); if (!c) return SB_ERR_ARG; cudaSetDevice(c->device); CU(c, d2h(c, dst, src, bytes)); return 0; }

// ---------------------------------------------------------------------------------------------------- Groth16
static int groth16_load_impl(sb_ctx* c, const uint8_t* zkey, uint64_t zlen, int shard, int n_shards, uint64_t* handle) {
    if (!c || !zkey || !handle || n_shards < 1 || shard < 0 || shard >= n_shards) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    Groth16Zkey z; std::string err;
    if (groth16_parse_zkey(zkey, zlen, z, err)) return fail(c, SB_ERR_FORMAT, err);
    if (z.n8q != c->n8q || !modulus_matches(z.q, z.n8q, c->curve, false) || !modulus_matches(z.r, z.n8r, c->curve, true))
        return fail(c, SB_ERR_FORMAT, "zkey curve does not match the context curve");
    if (z.power > c->fr_s) return fail(c, SB_ERR_FORMAT, "Circuit too big for this curve");
    Groth16Key* k = new Groth16Key();
    k->nVars = z.nVars; k->nPublic = z.nPublic; k->domainSize = z.domainSize; k->power = z.power; k->nCoef = z.sig.size();
    const uint32_t sG1 = 2 * c->n8q, sG2 = 4 * c->n8q;
    k->alpha1.assign(z.alpha1, z.alpha1 + sG1); k->beta1.assign(z.beta1, z.beta1 + sG1); k->beta2.assign(z.beta2, z.beta2 + sG2);
    k->gamma2.assign(z.gamma2, z.gamma2 + sG2); k->delta1.assign(z.delta1, z.delta1 + sG1); k->delta2.assign(z.delta2, z.delta2 + sG2);
    const uint64_t n = z.domainSize, nv = z.nVars;
    k->shard = shard; k->n_shards = n_shards;
    sb_shard_range(nv, shard, n_shards, &k->wlo, &k->wcnt);
    sb_shard_range(n, shard, n_shards, &k->hlo, &k->hcnt);
    const uint64_t wlo = k->wlo, wcnt = k->wcnt, hlo = k->hlo, hcnt = k->hcnt;
    cudaError_t e = cudaSuccess;
    auto alloc = [&](void** d, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(d, bytes ? bytes : 16); };
    auto up = [&](void** d, const void* src, size_t bytes) { alloc(d, bytes); if (e == cudaSuccess) e = h2d(c, *d, src, bytes); };
    up(&k->dA, z.A.p + wlo * sG1, wcnt * sG1);
    up(&k->dB1, z.B1.p + wlo * sG1, wcnt * sG1);
    up(&k->dB2, z.B2.p + wlo * sG2, wcnt * sG2);
    // C bases are indexed by signal - (nPublic+1): pad so that one sorted digit list of the witness serves A, B1, B2 and C
    alloc(&k->dC, wcnt * sG1);
    if (e == cudaSuccess && wcnt) e = cudaMemsetAsync(k->dC, 0, wcnt * sG1, c->stream);
    const uint64_t np1 = (uint64_t)k->nPublic + 1, g0 = std::max(wlo, np1), g1 = wlo + wcnt;
    if (e == cudaSuccess && g1 > g0) e = h2d(c, (uint8_t*)k->dC + (g0 - wlo) * sG1, z.C.p + (g0 - np1) * sG1, (g1 - g0) * sG1);
    up(&k->dH, z.H.p + hlo * sG1, hcnt * sG1);
    up((void**)&k->d_rowptr, z.rowptr.data(), z.rowptr.size() * 8);
    up((void**)&k->d_sig, z.sig.data(), z.sig.size() * 4);
    up(&k->d_coef, z.coef.data(), z.coef.size());
    alloc(&k->dW, (nv + 64) * 32);   // + room for the padded slices of the distributed witness all-gather
    if (e == cudaSuccess && (!k->batchX.get(3 * n * 32) || !k->batchY.get(3 * n * 32))) e = cudaErrorMemoryAllocation;
    alloc(&k->dWsum, 8 * 80 * 4 * 96);
    if (e == cudaSuccess) k->wsum_bytes = 8 * 80 * 4 * 96;
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);   // the CSR vectors and the caller's bytes go away on return
    if (e != cudaSuccess) { free_key(k); return cuda_fail(c, e, "sb_groth16_load upload"); }
    if (want_precomp(c, wcnt) && want_precomp(c, hcnt)) {
        int rc2 = build_table(c, c->g1, k->dA, wcnt, &k->tA, &k->gpW);
        if (!rc2) rc2 = build_table(c, c->g1, k->dB1, wcnt, &k->tB1, &k->gpW);
        if (!rc2) rc2 = build_table(c, c->g2, k->dB2, wcnt, &k->tB2, &k->gpW);
        if (!rc2) rc2 = build_table(c, c->g1, k->dC, wcnt, &k->tC, &k->gpW);
        if (!rc2) rc2 = build_table(c, c->g1, k->dH, hcnt, &k->tH, &k->gpH);
        if (rc2) { free_key(k); return rc2; }
    }
    c->keys.push_back(k);
    *handle = c->keys.size();
    return 0;
}

int sb_groth16_load(sb_ctx* c, const uint8_t* z, uint64_t zlen, uint64_t* handle) { SB_LOCK(c);
    return groth16_load_impl(c, z, zlen, 0, 1, handle);
}
int sb_groth16_load_sharded(sb_ctx* c, const uint8_t* z, uint64_t zlen, int shard, int n_shards, uint64_t* handle) { SB_LOCK(c);
    return groth16_load_impl(c, z, zlen, shard, n_shards, handle);
}

static Groth16Key* get_key(sb_ctx* c, uint64_t h) { return (c && h >= 1 && h <= c->keys.size()) ? c->keys[h - 1] : nullptr; }

int sb_groth16_info(sb_ctx* c, uint64_t h, uint32_t* nv, uint32_t* np, uint32_t* ds) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (nv) *nv = k->nVars; if (np) *np = k->nPublic; if (ds) *ds = k->domainSize;
    return 0;
}
int sb_groth16_release(sb_ctx* c, uint64_t h) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    cudaSetDevice(c->device); free_key(k); c->keys[h - 1] = nullptr; return 0;
}
uint32_t sb_groth16_partials_bytes(sb_ctx* c) { return c ? 4 * c->g1.xyzz_bytes + c->g2.xyzz_bytes : 0; }

// ---------------------------------------------------------------------------------------------------- NCCL
// libnccl is opened on first use, so libsnarkb200.so loads (and every single-GPU entry works) on hosts without NCCL.
// If the process already has a libnccl.so.2 (torch bundles one) that copy is reused.
struct NcclApi {
    void* so = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi* nccl_api(std::string* why) {
    static std::mutex mu; static NcclApi api; static bool tried = false; static std::string err;
    std::lock_guard<std::mutex> lk(mu);
    if (!tried) {
        tried = true;
        const char* env = getenv("SB_NCCL_LIB");
        void* so = env ? dlopen(env, RTLD_NOW | RTLD_LOCAL) : nullptr;
        if (!so) so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!so) so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!so) so = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
        if (!so) err = std::string("cannot load libnccl.so.2: ") + dlerror();
        else {
            api.so = so;
            bool ok = true;
            auto sym = [&](const char* n) { void* p = dlsym(so, n); if (!p) { ok = false; err = std::string("libnccl: missing symbol ") + n; } return p; };
            api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
            api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
            api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
            api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
            api.Send = (decltype(api.Send))sym("ncclSend");
            api.Recv = (decltype(api.Recv))sym("ncclRecv");
            api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
            api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
            api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
            if (!ok) api.so = nullptr;
        }
    }
    if (!api.so) { if (why) *why = err; return nullptr; }
    return &api;
}
#define NC(c, api, call) do { ncclResult_t _r = (call); if (_r != ncclSuccess) return fail(c, SB_ERR_CUDA, std::string(#call) + ": " + (api)->GetErrorString(_r)); } while (0)

int sb_comm_unique_id(uint8_t out[128]) {
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    if (!out) return SB_ERR_ARG;
    NcclApi* nc = nccl_api(nullptr); if (!nc) return SB_ERR_CUDA;
    ncclUniqueId id; if (nc->GetUniqueId(&id) != ncclSuccess) return SB_ERR_CUDA;
    memcpy(out, &id, 128); return 0;
}
int sb_comm_init_rank(sb_ctx* c, int world, int rank, const uint8_t id_bytes[128]) { SB_LOCK(c);
    if (!c || !id_bytes || world < 1 || world > 64 || rank < 0 || rank >= world) return fail(c, SB_ERR_ARG, "invalid communicator arguments");
    if (c->comm) return fail(c, SB_ERR_ARG, "context already belongs to a communicator");
    std::string why; NcclApi* nc = nccl_api(&why); if (!nc) return fail(c, SB_ERR_CUDA, why);
    cudaSetDevice(c->device);
    ncclUniqueId id; memcpy(&id, id_bytes, 128);
    NC(c, nc, nc->CommInitRank(&c->comm, world, id, rank));
    c->rank = rank; c->world = world;
    const size_t pb = (size_t)sb_groth16_partials_bytes(c);
    CU(c, cudaMalloc(&c->d_xchg, pb * world));
    CU(c, cudaHostAlloc((void**)&c->h_xchg, pb * (world + 1), cudaHostAllocDefault));
    return 0;
}
int sb_comm_info(sb_ctx* c, int* rank, int* world) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (rank) *rank = c->rank; if (world) *world = c->comm ? c->world : 0;
    return 0;
}
int sb_comm_destroy(sb_ctx* c) { SB_LOCK(c);
    if (!c) return SB_ERR_ARG;
    if (c->comm) {
        cudaSetDevice(c->device); cudaStreamSynchronize(c->stream);
        if (NcclApi* nc = nccl_api(nullptr)) nc->CommDestroy(c->comm);
        c->comm = nullptr; c->rank = 0; c->world = 1;
        if (c->d_xchg) cudaFree(c->d_xchg); if (c->h_xchg) cudaFreeHost(c->h_xchg);
        c->d_xchg = nullptr; c->h_xchg = nullptr;
    }
    return 0;
}
// which rank runs the iNTT -> coset NTT chain of polynomial j (0 = A, 1 = B, 2 = C) when a proof is distributed
int sb_dist_chain_owner(int chain, int world) { return world > 0 ? chain % world : 0; }

// plain (non-Montgomery) r and s: when given, the prover folds s*A + r*B1 + H into the C partial as soon as A and B1 land
// (hidden behind the C and H MSMs), so that the proof assembly after the last MSM is three additions
struct ProofScalars { uint8_t rp[32], sp[32]; };

// The window sums of a proof's MSMs land in the key's device buffer and come back through the context's pinned area.
// Their first sizes hold the table geometries and the plain ones over about a thousand points; a plain MSM over fewer
// points takes narrower windows (3 bits, 86 windows, for 49 points or fewer on BN254), which need more room, so both
// buffers grow to what the geometries of the call need.  Earlier calls have finished with them by now.
static int groth16_wsum_room(sb_ctx* c, Groth16Key* k, size_t dev_bytes, size_t host_bytes) {
    if (dev_bytes > k->wsum_bytes) {
        void* old = k->dWsum; k->dWsum = nullptr; k->wsum_bytes = 0;
        if (old) CU(c, cudaFree(old));
        CU(c, cudaMalloc(&k->dWsum, dev_bytes));
        k->wsum_bytes = dev_bytes;
    }
    if (host_bytes > c->pinned_bytes) {
        uint8_t* old = c->pinned; c->pinned = nullptr; c->pinned_bytes = 0;
        if (old) CU(c, cudaFreeHost(old));
        CU(c, cudaHostAlloc((void**)&c->pinned, host_bytes, cudaHostAllocDefault));
        c->pinned_bytes = host_bytes;
    }
    return 0;
}

// QAP rows -> iNTT -> coset NTT -> [exchange] -> joinABC of K proofs (witness q at dW + q * nVars elements) on stream st, in
// the key's transform buffers batchX / batchY (3Kn elements each: A of every proof, then B, then C).  *hsc = where the H
// scalars went (proof q's at + q * n elements); the ones of [hlo, hlo + hcnt) are computed, K > 1 only with the full range.
// dist: the three chains run on the ranks sb_dist_chain_owner names and send their coset evaluations to every other rank's
// H range (NCCL send/recv); every rank then joins its own H range.
static int groth16_qap_ntt(sb_ctx* c, Groth16Key* k, const void* dW, uint32_t K, uint64_t hlo, uint64_t hcnt, bool dist,
                           cudaStream_t st, uint8_t** hsc) {
    const int cv = c->curve;
    const uint64_t n = k->domainSize, nv = k->nVars;
    const size_t tn = (size_t)K * n * 32;   // bytes of one of A, B, C over the K proofs
    uint8_t* X = (uint8_t*)k->batchX.get(3 * tn);
    uint8_t* Y = (uint8_t*)k->batchY.get(3 * tn);
    if (!X || !Y) return fail(c, SB_ERR_NOMEM, "out of device memory (Groth16 transform buffers)");
    const bool xchg = dist && c->world > 1;
    // Every pass moves the data to the other buffer, so where the coset evaluations end up follows from the pass count:
    // known on ranks that run no chain too, which receive into it.
    const int np = fr_ntt_passes(k->power);
    auto after_ntt = [&](uint8_t* in) { return (np & 1) ? (in == X ? Y : X) : in; };
    uint8_t* const ev = after_ntt(after_ntt(X));
    int my[3], m = 0;
    for (int j = 0; j < 3; j++) if (!xchg || sb_dist_chain_owner(j, c->world) == c->rank) my[m++] = j;
    int rc;
    if (m) {
        // buildABC1 (:147-187)
        { ProfScope pq(&c->stats, PROF_QAP, st);
          rc = fr_qap_rows(cv, k->d_rowptr, k->d_sig, k->d_coef, dW, nv, X, X + tn, X + 2 * tn, n, K, st); c->launches++;
          pq.end(); }
        if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_qap_rows");
        // :64-76  ifft -> batchApplyKey(1, inc) -> fft, with 1/n of the inverse folded into the coset table
        const uint8_t* inc = (k->power == c->fr_s) ? c->shift.data() : c->roots[k->power + 1].data();
        uint8_t ninv[32];
        if (cv == SB_BN254) ninv_bytes<BnFr>(k->power, ninv); else ninv_bytes<BlsFr>(k->power, ninv);
        FrPre pre; rc = get_pre(c, n, ninv, inc, &pre); if (rc) return rc;
        FrNttTables tbi, tbf;
        rc = get_ntt_tab(c, k->power, true, &tbi); if (rc) return rc;
        rc = get_ntt_tab(c, k->power, false, &tbf); if (rc) return rc;
        // the transforms run as one batch per pass (grids fill whole waves): up to four by pointer (one proof's chains, or
        // the ones this rank owns, which need not be adjacent), more as one strided batch of all 3K
        int side = 0, side2 = 0, launches = 0;
        bool landed;
        ProfScope pn(&c->stats, PROF_NTT, st);
        if (m * K <= 4) {
            void* a[4]; void* b[4]; int t = 0;
            for (int i = 0; i < m; i++)
                for (uint32_t q = 0; q < K; q++, t++) { const size_t o = my[i] * tn + q * n * 32; a[t] = X + o; b[t] = Y + o; }
            rc = fr_ntt_batch(cv, a, b, t, k->power, &tbi, nullptr, nullptr, st, &side, &launches);      // unscaled inverse
            if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_ntt_batch");
            void** src = side ? b : a; void** dst = side ? a : b;
            rc = fr_ntt_batch(cv, src, dst, t, k->power, &tbf, &pre, nullptr, st, &side2, &launches);     // coset NTT, 1/n folded in
            if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_ntt_batch");
            landed = (side2 ? dst : src)[0] == ev + my[0] * tn;
        } else {
            rc = fr_ntt_strided(cv, X, Y, 3 * (int)K, k->power, &tbi, nullptr, nullptr, st, &side, &launches);
            if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_ntt_strided");
            uint8_t* src = side ? Y : X; uint8_t* dst = side ? X : Y;
            rc = fr_ntt_strided(cv, src, dst, 3 * (int)K, k->power, &tbf, &pre, nullptr, st, &side2, &launches);
            if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_ntt_strided");
            landed = (side2 ? dst : src) == ev;
        }
        pn.end();
        c->launches += launches;
        if (!landed) return fail(c, SB_ERR_CUDA, "internal: NTT result buffer mismatch");
    }
    if (xchg) {   // coset evaluations of chain j: owner -> every other rank's H range
        NcclApi* nc = nccl_api(nullptr);
        NC(c, nc, nc->GroupStart());
        for (int j = 0; j < 3; j++) {
            const int o = sb_dist_chain_owner(j, c->world);
            uint8_t* evj = ev + j * tn;
            if (o == c->rank) {
                for (int q = 0; q < c->world; q++) {
                    if (q == c->rank) continue;
                    uint64_t qlo, qcnt; sb_shard_range(n, q, c->world, &qlo, &qcnt);
                    if (qcnt) NC(c, nc, nc->Send(evj + qlo * 32, qcnt * 32, ncclUint8, q, c->comm, st));
                }
            } else if (hcnt) NC(c, nc, nc->Recv(evj + hlo * 32, hcnt * 32, ncclUint8, o, c->comm, st));
        }
        NC(c, nc, nc->GroupEnd());
    }
    // joinABC (:320-374) -> plain scalars for the H MSM, into the other buffer (free once the transforms are done)
    uint8_t* const h = ev == X ? Y : X;
    if (hcnt) {
        ProfScope pj(&c->stats, PROF_JOIN, st);
        rc = fr_join_abc(cv, ev + hlo * 32, ev + tn + hlo * 32, ev + 2 * tn + hlo * 32, h + hlo * 32, K * hcnt, st); c->launches++;
        pj.end();
        if (rc) return cuda_fail(c, (cudaError_t)rc, "fr_join_abc");
    }
    *hsc = h;
    return 0;
}

// One of the five MSMs of a sub-batch: its group, one proof's geometry (what combine takes), its window sums in the pinned
// area (len bytes at off, proof q's at off + q * per) and the offset of its partial in a proof's A | B1 | C | H | B2.
struct Groth16Job { const GroupOps* G; MsmGeom g; size_t off, len, per, part; };
struct Groth16Jobs {
    enum { B2, A, B1, C, H };
    Groth16Job job[5];        // B2, A, B1, C, H: the order they are issued and land in; H's region ends the area
    const uint64_t* counts;   // pinned: the sorted entries of the witness and of the H digits
    // sb_last_stat 4 and 5, once every job has landed
    void tally(sb_ctx* c) const { c->stat[4] += 3.0 * (double)counts[0] + (double)counts[1]; c->stat[5] += (double)counts[0]; }
};

// The device work of K proofs (witness q at dW + q * nVars elements) over the witness points [wlo, wlo + wcnt) and the H
// points [hlo, hlo + hcnt), each at most one MSM chunk; K > 1 only with the full ranges.  The witness is sorted once (A,
// B1, B2 and C all multiply it, :84-97); the five bucket pipelines run on their own streams so that the latency-bound
// tails (fold cascade, bucket reduction) of one MSM run beside the throughput-bound accumulation of the next; the H
// scalars (QAP/NTT chain) are produced concurrently.  g_serial_prove serialises everything on one stream (profiling).
// The G2 accumulation goes first: its CTAs (2 x 128 threads x 248 allocated registers per SM) leave no room beside
// them, so no side work that could run beside a G1 accumulation is left waiting behind it.
//   main stream : sort(witness), acc B2, acc A, acc B1, acc C, [wait for the NTT chain], acc H
//   aux[5]      : QAP -> iNTT -> coset NTT -> [exchange] -> joinABC -> sort(H scalars)
//   aux[0..4]   : the tail of job i (fold, reduce, window sum) and its D2H into the pinned area, then pev[2 + i]
// Returns with the work queued and the main stream waiting for all of it; job i's window sums are on the host once
// pev[2 + i] has fired.
static int groth16_issue(sb_ctx* c, Groth16Key* k, const void* dW, uint32_t K, uint64_t wlo, uint64_t wcnt, uint64_t hlo, uint64_t hcnt,
                         bool dist, Groth16Jobs* out) {
    const GroupOps& G1 = c->g1; const GroupOps& G2 = c->g2;
    const uint32_t x1 = G1.xyzz_bytes, x2 = G2.xyzz_bytes;
    const bool serial = g_serial_prove != 0;
    cudaStream_t s0 = c->stream, sN = serial ? s0 : c->aux[5];
    // a key loaded with sb_groth16_load_sharded only holds its own ranges: local indexing
    const bool local = k->n_shards > 1;
    const uint64_t wb = local ? 0 : wlo, hb = local ? 0 : hlo;   // base-set index of the first point
    const bool pre = k->tA != nullptr;
    MsmGeom gw = msm_geometry(wcnt, 32, c->fr_bits), gh = msm_geometry(hcnt, 32, c->fr_bits);
    if (pre) { gw = k->gpW; gw.first = wb; gh = k->gpH; gh.first = hb; }
    MsmGeom gwK = gw, ghK = gh; gwK.K = K; ghK.K = K;
    const size_t w1 = (size_t)gwK.wsum_points() * x1, w2 = (size_t)gwK.wsum_points() * x2, wh = (size_t)ghK.wsum_points() * x1;
    const size_t wtot = 3 * w1 + w2 + wh;
    int rc = groth16_wsum_room(c, k, wtot, wtot + 64);
    if (rc) return rc;
    uint8_t* dws = (uint8_t*)k->dWsum; uint8_t* hws = c->pinned;
    uint64_t* hcounts = (uint64_t*)(c->pinned + wtot);
    CU(c, cudaEventRecord(c->pev[0], s0));                       // witnesses resident
    if (sN != s0) CU(c, cudaStreamWaitEvent(sN, c->pev[0], 0));
    // NTT chain + sort of the H scalars on the side stream
    uint8_t* hsc;
    rc = groth16_qap_ntt(c, k, dW, K, hlo, hcnt, dist, sN, &hsc);
    if (rc) return rc;
    MsmSorted sh;
    rc = msm_sort_entries(hsc + hlo * 32, 32, hcnt, ghK, c->sort_scratch2, sN, &sh, &c->stats);
    if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_sort_entries");
    CU(c, cudaEventRecord(c->pev[1], sN));
    // witness MSMs on the main stream
    MsmSorted sw;
    rc = msm_sort_entries((const uint8_t*)dW + wlo * 32, 32, wcnt, gwK, c->sort_scratch, s0, &sw, &c->stats);
    if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_sort_entries");
    tick(c, 2);
    // the G2 MSM first, then A and B1 (a single proof folds s*A + r*B1 on the host as they land), C, and H last;
    // window sums in the area A | B1 | C | B2 | H, partials in a proof's A | B1 | C | H | B2
    const size_t pw = (size_t)msm_wsum_parts(gw) * gw.windows_per_proof(), ph = (size_t)msm_wsum_parts(gh) * gh.windows_per_proof();
    *out = Groth16Jobs{{{&G2, gw, 3 * w1, w2, pw * x2, 4 * x1}, {&G1, gw, 0, w1, pw * x1, 0}, {&G1, gw, w1, w1, pw * x1, x1},
                        {&G1, gw, 2 * w1, w1, pw * x1, 2 * x1}, {&G1, gh, 3 * w1 + w2, wh, ph * x1, 3 * x1}}, hcounts};
    const void* bases[5] = {pre ? k->tB2 : (const void*)((const uint8_t*)k->dB2 + wb * G2.aff_bytes),
                            pre ? k->tA : (const void*)((const uint8_t*)k->dA + wb * G1.aff_bytes),
                            pre ? k->tB1 : (const void*)((const uint8_t*)k->dB1 + wb * G1.aff_bytes),
                            pre ? k->tC : (const void*)((const uint8_t*)k->dC + wb * G1.aff_bytes),
                            pre ? k->tH : (const void*)((const uint8_t*)k->dH + hb * G1.aff_bytes)};
    for (int i = 0; i < 5; i++) {
        const Groth16Job& j = out->job[i];
        cudaStream_t st = serial ? s0 : c->aux[i];
        if (i == Groth16Jobs::H && sN != s0) CU(c, cudaStreamWaitEvent(s0, c->pev[1], 0));   // H needs the NTT chain
        c->stats.cur_tag = j.G == &G1 ? SB_G1 : SB_G2;
        rc = j.G->buckets(bases[i], i == Groth16Jobs::H ? sh : sw, c->bscr[i], s0, dws + j.off, &c->stats, st, c->pev[8 + i]);
        if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_buckets");
        CU(c, cudaMemcpyAsync(hws + j.off, dws + j.off, j.len, cudaMemcpyDeviceToHost, st));
        if (i == 0) CU(c, cudaMemcpyAsync(&hcounts[0], sw.counts, 8, cudaMemcpyDeviceToHost, st));
        if (i == Groth16Jobs::H) CU(c, cudaMemcpyAsync(&hcounts[1], sh.counts, 8, cudaMemcpyDeviceToHost, st));
        CU(c, cudaEventRecord(c->pev[2 + i], st));
    }
    tick(c, 3);
    // join the side streams back into the main stream
    if (!serial) { for (int i = 0; i < 5; i++) CU(c, cudaStreamWaitEvent(s0, c->pev[2 + i], 0)); CU(c, cudaStreamWaitEvent(s0, c->pev[1], 0)); }
    return 0;
}

// C' = C + H + s*A + r*B1 into the C slot of one proof's partials (A | B1 | C | H | B2): the part of the split assembly
// (groth16_fixed_parts) that depends on the MSMs.  sA = s*A and rB1 = r*B1, which a single proof computes as A and B1 land.
static void groth16_fold(const GroupOps& G1, uint8_t* partials, const uint8_t* sA, const uint8_t* rB1) {
    uint8_t* C = partials + 2 * G1.xyzz_bytes;
    G1.add(C, partials + 3 * G1.xyzz_bytes); G1.add(C, sA); G1.add(C, rB1);
}
static void groth16_fold_scalars(const GroupOps& G1, uint8_t* partials, const ProofScalars& ps) {
    std::vector<uint8_t> sA(G1.xyzz_bytes), rB1(G1.xyzz_bytes);
    G1.times(partials, ps.sp, 32, sA.data());                      // s * A   (src/groth16_prove.js:117: pi_c += s*pi_a)
    G1.times(partials + G1.xyzz_bytes, ps.rp, 32, rB1.data());     // r * B1  (:118)
    groth16_fold(G1, partials, sA.data(), rB1.data());
}

// device part of the prover: returns the five MSM partials (A, B1, C, H | B2) as host XYZZ bytes.
// witness is uploaded to the key's resident witness; null proves from the resident one, or from d_witness when given (a
// witness already on the device: the resident one is left as it is).
// dist: this context is rank c->rank of c->world (sb_comm_init_rank); the witness is uploaded in slices and all-gathered,
// the three transform chains run on different ranks and exchange their coset evaluations (NCCL send/recv), every rank
// then joins and multiplies its own H range.
static int groth16_device(sb_ctx* c, Groth16Key* k, const uint8_t* witness, uint64_t n_witness, int shard, int n_shards, uint8_t* partials,
                          const ProofScalars* ps = nullptr, bool dist = false, const void* d_witness = nullptr) {
    if (witness && n_witness != k->nVars) return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(k->nVars) + ", witness: " + std::to_string(n_witness));
    cudaSetDevice(c->device);
    const uint64_t n = k->domainSize, nv = k->nVars;
    NcclApi* nc = nullptr;
    if (dist) {
        if (!c->comm) return fail(c, SB_ERR_ARG, "context has no communicator: call sb_comm_init_rank first");
        nc = nccl_api(nullptr);
        shard = c->rank; n_shards = c->world;
    }
    const int world = n_shards, rank = shard;
    const void* dW = d_witness ? d_witness : k->dW;
    int rc;
    tick(c, 0);
    if (witness) {
        k->witness_resident = false;
        if (dist && world > 1) {   // every rank uploads 1/world of the witness; NVLink all-gather completes it
            const uint64_t per = (nv + world - 1) / world, lo = std::min(nv, per * (uint64_t)rank), cnt = std::min(nv - lo, per);
            CU(c, h2d(c, (uint8_t*)k->dW + lo * 32, witness + lo * 32, cnt * 32));
            NC(c, nc, nc->AllGather((const uint8_t*)k->dW + per * rank * 32, k->dW, per * 32, ncclUint8, c->comm, c->stream));
        } else CU(c, h2d(c, k->dW, witness, nv * 32));
        k->witness_resident = true;
    } else if (!d_witness && !k->witness_resident) return fail(c, SB_ERR_ARG, "no witness resident for this proving key: call sb_groth16_prove first");
    tick(c, 1);
    prof_begin(c);
    // MSMs (:84-101).  Shard = contiguous point range (SURVEY §8e); shard 0 of 1 = everything.
    uint64_t wlo, wcnt; sb_shard_range(nv, rank, n_shards, &wlo, &wcnt);
    uint64_t hlo, hcnt; sb_shard_range(n, rank, n_shards, &hlo, &hcnt);
    const GroupOps& G1 = c->g1; const GroupOps& G2 = c->g2;
    uint8_t* pA = partials; uint8_t* pB1 = pA + G1.xyzz_bytes; uint8_t* pC = pB1 + G1.xyzz_bytes; uint8_t* pH = pC + G1.xyzz_bytes; uint8_t* pB2 = pH + G1.xyzz_bytes;
    memset(partials, 0, 4 * G1.xyzz_bytes + G2.xyzz_bytes);
    std::vector<uint8_t> sA(G1.xyzz_bytes, 0), rB1(G1.xyzz_bytes, 0);
    const uint64_t MAXC = 1ull << (g_msm_chunk_log > 0 ? g_msm_chunk_log : 23);   // points per MSM chunk
    const bool local = k->n_shards > 1;
    if (local && (shard != k->shard || n_shards != k->n_shards)) return fail(c, SB_ERR_ARG, "proving key was loaded for a different shard");
    const uint64_t wb = local ? 0 : wlo, hb = local ? 0 : hlo;   // base-set index of this call's first point
    const bool overlapped = wcnt <= MAXC && hcnt <= MAXC && wcnt > 0 && hcnt > 0 && c->pinned;
    if (dist && world > 1 && !overlapped) return fail(c, SB_ERR_ARG, "distributed proving needs at least one point per rank and shards of at most 2^23 points");
    if (overlapped) {
        Groth16Jobs t;
        rc = groth16_issue(c, k, dW, 1, wlo, wcnt, hlo, hcnt, dist, &t);
        if (rc) return rc;
        // host recombination as each MSM lands (overlaps with the MSMs still running)
        for (int i = 0; i < 5; i++) {
            const Groth16Job& j = t.job[i];
            CU(c, cudaEventSynchronize(c->pev[2 + i]));
            j.G->combine(c->pinned + j.off, j.g, partials + j.part);
            if (ps && i == Groth16Jobs::A) G1.times(pA, ps->sp, 32, sA.data());      // s * A   (src/groth16_prove.js:117: pi_c += s*pi_a)
            if (ps && i == Groth16Jobs::B1) G1.times(pB1, ps->rp, 32, rB1.data());   // r * B1  (:118)
        }
        t.tally(c);
    } else {
    uint8_t* hsc;
    rc = groth16_qap_ntt(c, k, dW, 1, hlo, hcnt, dist, c->stream, &hsc); if (rc) return rc;
    tick(c, 2);
    for (uint64_t off = 0; off < wcnt; off += MAXC) {
        uint64_t cn = std::min(MAXC, wcnt - off), base = wb + off;
        MsmGeom g = msm_geometry(cn, 32, c->fr_bits);
        MsmSorted s;
        rc = msm_sort_entries((const uint8_t*)dW + (wlo + off) * 32, 32, cn, g, c->sort_scratch, c->stream, &s, &c->stats);
        if (rc) return cuda_fail(c, (cudaError_t)rc, "msm_sort_entries");
        size_t w1 = (size_t)g.wsum_points() * G1.xyzz_bytes, w2 = (size_t)g.wsum_points() * G2.xyzz_bytes;
        rc = groth16_wsum_room(c, k, 3 * w1 + w2, 0);
        if (rc) return rc;
        uint8_t* ws = (uint8_t*)k->dWsum;
        c->stats.cur_tag = SB_G1;
        rc = G1.buckets((const uint8_t*)k->dA + base * G1.aff_bytes, s, c->bucket_scratch, c->stream, ws, &c->stats, nullptr, nullptr); if (rc) return cuda_fail(c, (cudaError_t)rc, "msm A");
        rc = G1.buckets((const uint8_t*)k->dB1 + base * G1.aff_bytes, s, c->bucket_scratch, c->stream, ws + w1, &c->stats, nullptr, nullptr); if (rc) return cuda_fail(c, (cudaError_t)rc, "msm B1");
        rc = G1.buckets((const uint8_t*)k->dC + base * G1.aff_bytes, s, c->bucket_scratch, c->stream, ws + 2 * w1, &c->stats, nullptr, nullptr); if (rc) return cuda_fail(c, (cudaError_t)rc, "msm C");
        c->stats.cur_tag = SB_G2;
        rc = G2.buckets((const uint8_t*)k->dB2 + base * G2.aff_bytes, s, c->bucket_scratch, c->stream, ws + 3 * w1, &c->stats, nullptr, nullptr); if (rc) return cuda_fail(c, (cudaError_t)rc, "msm B2");
        std::vector<uint8_t> hw(3 * w1 + w2);
        uint64_t entries = 0;
        CU(c, cudaMemcpyAsync(hw.data(), ws, hw.size(), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaMemcpyAsync(&entries, s.counts, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        c->stat[4] += 3.0 * (double)entries; c->stat[5] += (double)entries;
        G1.combine(hw.data(), g, pA); G1.combine(hw.data() + w1, g, pB1); G1.combine(hw.data() + 2 * w1, g, pC); G2.combine(hw.data() + 3 * w1, g, pB2);
    }
    tick(c, 3);
    if (hcnt) {
        rc = msm_dev_accumulate(c, G1, (const uint8_t*)k->dH + hb * G1.aff_bytes, hsc + hlo * 32, 32, hcnt, pH);
        if (rc) return rc;
    }
    if (ps) { G1.times(pA, ps->sp, 32, sA.data()); G1.times(pB1, ps->rp, 32, rB1.data()); }
    }
    if (ps) {   // C' = C + H + s*A + r*B1;  the B1 and H slots are spent
        groth16_fold(G1, partials, sA.data(), rB1.data());
        memset(pB1, 0, G1.xyzz_bytes); memset(pH, 0, G1.xyzz_bytes);
    }
    tick(c, 4);
    cudaEventSynchronize(c->ev[4]);
    prof_end(c);
    c->last_ms[0] = elapsed(c, 0, 4); c->last_ms[1] = elapsed(c, 0, 1); c->last_ms[2] = elapsed(c, 1, 2); c->last_ms[3] = elapsed(c, 2, 3); c->last_ms[4] = elapsed(c, 3, 4);
    return 0;
}

// host part: proof assembly, src/groth16_prove.js:103-132

struct VkPoints { const uint8_t *alpha1, *beta1, *beta2, *delta1, *delta2; };
static void plain_scalars(int curve, const uint8_t r[32], const uint8_t s[32], uint8_t rp[32], uint8_t sp[32], uint8_t rsp[32]) {
    uint8_t rs[32];
    if (curve == SB_BN254) {
        fr_from_mont_bytes<BnFr>(r, rp); fr_from_mont_bytes<BnFr>(s, sp);
        Fp<BnFr> a, b; memcpy(&a, r, 32); memcpy(&b, s, 32); a = Fp<BnFr>::mul(a, b); memcpy(rs, &a, 32);
        fr_from_mont_bytes<BnFr>(rs, rsp);
    } else {
        fr_from_mont_bytes<BlsFr>(r, rp); fr_from_mont_bytes<BlsFr>(s, sp);
        Fp<BlsFr> a, b; memcpy(&a, r, 32); memcpy(&b, s, 32); a = Fp<BlsFr>::mul(a, b); memcpy(rs, &a, 32);
        fr_from_mont_bytes<BlsFr>(rs, rsp);
    }
}

// The assembly is split so that nothing but three additions and three normalisations follows the last MSM:
//   pi_a = A + [alpha1 + r*delta1],  pi_b = B2 + [beta2 + s*delta2],
//   pi_c = C + H + s*pi_a + r*pib1 - rs*delta1 = [C + H + s*A + r*B1] + [s*alpha1 + r*beta1 + rs*delta1]
// The bracketed fixed parts depend only on the key and (r, s): a helper thread computes them while the GPU works;
// the C bracket is folded (groth16_fold) by groth16_device as A and B1 land, or per proof on the host.
struct FixedParts { std::vector<uint8_t> Fa, Fb, Fc; };
// g2_thread: the G2 multiple runs on a thread of its own (a single proof's latency); false runs it in place (batch pool)
static FixedParts groth16_fixed_parts(int curve, const GroupOps& G1, const GroupOps& G2, const VkPoints vk, const uint8_t* r, const uint8_t* s,
                                      bool g2_thread = true) {
    const uint32_t x1 = G1.xyzz_bytes, x2 = G2.xyzz_bytes;
    uint8_t rp[32], sp[32], rsp[32];
    plain_scalars(curve, r, s, rp, sp, rsp);
    FixedParts f; f.Fa.assign(x1, 0); f.Fb.assign(x2, 0); f.Fc.assign(x1, 0);
    std::vector<uint8_t> a1(x1), b1(x1), d1(x1), b2(x2), d2(x2), t1(x1), t2(x2);
    G1.from_affine(vk.alpha1, a1.data()); G1.from_affine(vk.beta1, b1.data()); G1.from_affine(vk.delta1, d1.data());
    G2.from_affine(vk.beta2, b2.data()); G2.from_affine(vk.delta2, d2.data());
    std::future<void> g2 = std::async(g2_thread ? std::launch::async : std::launch::deferred, [&]() { G2.times(d2.data(), sp, 32, t2.data()); });   // the one G2 multiple
    G1.times(d1.data(), rp, 32, t1.data()); f.Fa = a1; G1.add(f.Fa.data(), t1.data());
    G1.times(a1.data(), sp, 32, f.Fc.data());
    G1.times(b1.data(), rp, 32, t1.data()); G1.add(f.Fc.data(), t1.data());
    G1.times(d1.data(), rsp, 32, t1.data()); G1.add(f.Fc.data(), t1.data());
    g2.get();
    f.Fb = b2; G2.add(f.Fb.data(), t2.data());
    return f;
}
static void groth16_finish_folded(const GroupOps& G1, const GroupOps& G2, const FixedParts& f, const uint8_t* partials, uint8_t* proof) {
    const uint32_t x1 = G1.xyzz_bytes, x2 = G2.xyzz_bytes;
    std::vector<uint8_t> A(partials, partials + x1), C(partials + 2 * x1, partials + 3 * x1), B2(partials + 4 * x1, partials + 4 * x1 + x2);
    G1.add(A.data(), f.Fa.data()); G2.add(B2.data(), f.Fb.data()); G1.add(C.data(), f.Fc.data());
    G1.to_affine(A.data(), proof);
    G2.to_affine(B2.data(), proof + G1.aff_bytes);
    G1.to_affine(C.data(), proof + G1.aff_bytes + G2.aff_bytes);
}
// The proof from the partials of n_shards shards (n_shards x (A | B1 | C | H | B2), XYZZ bytes): their sums, folded and
// finished as above.
static void groth16_assemble_host(int curve, const GroupOps& G1, const GroupOps& G2, const VkPoints& vk, const uint8_t* all, int n_shards,
                                  const uint8_t r[32], const uint8_t s[32], uint8_t* proof) {
    const uint32_t x1 = G1.xyzz_bytes, pb = 4 * x1 + G2.xyzz_bytes;
    std::vector<uint8_t> acc(pb, 0);
    for (int i = 0; i < n_shards; i++) {
        const uint8_t* p = all + (size_t)i * pb;
        for (int j = 0; j < 4; j++) G1.add(acc.data() + j * x1, p + j * x1);
        G2.add(acc.data() + 4 * x1, p + 4 * x1);
    }
    ProofScalars ps; uint8_t rsp[32]; plain_scalars(curve, r, s, ps.rp, ps.sp, rsp);
    groth16_fold_scalars(G1, acc.data(), ps);
    groth16_finish_folded(G1, G2, groth16_fixed_parts(curve, G1, G2, vk, r, s, false), acc.data(), proof);
}
static int groth16_prove_folded(sb_ctx* c, Groth16Key* k, const uint8_t* witness, uint64_t n_witness, const uint8_t r[32], const uint8_t s[32], uint8_t* proof,
                                const void* d_witness = nullptr) {
    VkPoints vk{k->alpha1.data(), k->beta1.data(), k->beta2.data(), k->delta1.data(), k->delta2.data()};
    const int curve = c->curve; const GroupOps G1 = c->g1, G2 = c->g2;
    std::future<FixedParts> fixed = std::async(std::launch::async, [=]() { return groth16_fixed_parts(curve, G1, G2, vk, r, s); });
    ProofScalars ps; uint8_t rsp[32]; plain_scalars(curve, r, s, ps.rp, ps.sp, rsp);
    std::vector<uint8_t> partials(sb_groth16_partials_bytes(c));
    int rc = groth16_device(c, k, witness, n_witness, 0, 1, partials.data(), &ps, false, d_witness);
    FixedParts f = fixed.get();
    if (rc) return rc;
    groth16_finish_folded(c->g1, c->g2, f, partials.data(), proof);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- Groth16 batches
// sb_groth16_prove_batch: K proofs against one key, sub-batch by sub-batch.  A sub-batch of K' proofs runs the single
// proof's pipeline (groth16_issue) once with K' times the work per launch: one QAP launch over K' witnesses, one strided NTT
// batch of 3K' transforms per pass, one joinABC over K'n elements, one sort of the K' witnesses' digits (shared by A, B1, B2
// and C) and one of the K' H-scalar vectors, five bucket pipelines whose windows are the K' proofs' windows side by side
// (MsmGeom::K), five downloads of the window sums.  Recombination and proof assembly run per proof on host threads.

// What one more proof of a sub-batch costs in device memory: its witness, six n-element arrays (the 3n transform data and
// its 3n scratch; the H scalars reuse the scratch), the sorted entries of its witness and H digits, and its share of the
// five bucket pipelines (K'·B XYZZ buckets per MSM, G1 and G2).
static size_t groth16_batch_footprint(const sb_ctx* c, const Groth16Key* k, const MsmGeom& gw, const MsmGeom& gh) {
    const uint64_t n = k->domainSize, nv = k->nVars;
    const size_t x1 = c->g1.xyzz_bytes, x2 = c->g2.xyzz_bytes;
    const uint64_t ew = nv * (uint64_t)gw.W, eh = n * (uint64_t)gh.W;
    const uint64_t bw = (uint64_t)gw.windows_per_proof() * gw.B, bh = (uint64_t)gh.windows_per_proof() * gh.B;
    return (size_t)(nv + 6 * n) * 32 + sort_batch_bytes(ew) + sort_batch_bytes(eh)
         + 3 * msm_batch_bytes(ew, bw, x1) + msm_batch_bytes(ew, bw, x2) + msm_batch_bytes(eh, bh, x1);
}

// Keys whose witness or H side is longer than one MSM chunk (2^23 points, sb_set_tuning(6) lowers it): the batched sort
// would hold every entry of a proof at once, so each proof goes through the single-proof path, which cuts its MSMs into
// chunks.  Each witness goes to the batch's witness buffer, so the resident witness is not touched.
static int groth16_prove_batch_chunked(sb_ctx* c, Groth16Key* k, const uint8_t* witnesses, uint32_t count,
                                       const uint8_t* r, const uint8_t* s, uint8_t* proofs) {
    const uint64_t nv = k->nVars;
    const uint32_t proof_bytes = 2 * c->g1.aff_bytes + c->g2.aff_bytes;
    void* dW = k->batchW.get(nv * 32);
    if (!dW) return fail(c, SB_ERR_NOMEM, "out of device memory (Groth16 batch witness)");
    tick(c, 5);
    for (uint32_t i = 0; i < count; i++) {
        CU(c, h2d(c, dW, witnesses + (size_t)i * nv * 32, nv * 32));
        int rc = groth16_prove_folded(c, k, nullptr, nv, r + 32 * (size_t)i, s + 32 * (size_t)i, proofs + (size_t)i * proof_bytes, dW);
        if (rc) return rc;
    }
    tick(c, 6);
    CU(c, cudaEventSynchronize(c->ev[6]));
    c->last_ms[0] = elapsed(c, 5, 6);
    return 0;
}

// host_threads: the host pool's size, 0 = one thread per core (a multi-context batch gives each rank its share of the cores)
static int groth16_prove_batch_impl(sb_ctx* c, Groth16Key* k, const uint8_t* witnesses, uint32_t count,
                                    const uint8_t* r, const uint8_t* s, uint8_t* proofs, unsigned host_threads = 0) {
    cudaSetDevice(c->device);
    const uint64_t n = k->domainSize, nv = k->nVars;
    const uint64_t MAXC = 1ull << (g_msm_chunk_log > 0 ? g_msm_chunk_log : 23);
    if (nv > MAXC || n > MAXC) return groth16_prove_batch_chunked(c, k, witnesses, count, r, s, proofs);
    const int cv = c->curve;
    const GroupOps G1 = c->g1, G2 = c->g2;
    const uint32_t x1 = G1.xyzz_bytes, x2 = G2.xyzz_bytes, pb = 4 * x1 + x2, proof_bytes = 2 * G1.aff_bytes + G2.aff_bytes;
    MsmGeom gw = msm_geometry(nv, 32, c->fr_bits), gh = msm_geometry(n, 32, c->fr_bits);
    const bool pre = k->tA != nullptr;
    if (pre) { gw = k->gpW; gw.first = 0; gh = k->gpH; gh.first = 0; }
    // 3K' transforms per NTT launch: the grid's y dimension (65535) bounds K' as well
    const uint64_t key_limit = std::min({msm_batch_limit(nv, gw.c, gw.W, gw.precomp), msm_batch_limit(n, gh.c, gh.W, gh.precomp), (uint64_t)65535 / 3});
    const uint32_t KB = batch_size(c, count, key_limit, groth16_batch_footprint(c, k, gw, gh), k->batchW.cap + k->batchX.cap + k->batchY.cap);
    // per proof: the five partials A | B1 | C | H | B2, then the proof
    std::vector<uint8_t> allp((size_t)count * pb, 0);
    std::vector<FixedParts> fixed(count);
    const VkPoints vk{k->alpha1.data(), k->beta1.data(), k->beta2.data(), k->delta1.data(), k->delta2.data()};
    // Host work on one pool of at most one thread per core, declared after everything its tasks touch: leaving this
    // function (also on an error) runs the queued tasks and joins.  The fixed parts go first, so they overlap the GPU work.
    HostPool pool(std::min<unsigned>(count, host_threads ? host_threads : std::max(1u, std::thread::hardware_concurrency())));
    for (uint32_t i = 0; i < count; i++)
        pool.submit([&, i]() { fixed[i] = groth16_fixed_parts(cv, G1, G2, vk, r + 32 * (size_t)i, s + 32 * (size_t)i, false); });
    int rc;
    tick(c, 0);
    prof_begin(c);
    for (uint32_t k0 = 0; k0 < count; k0 += KB) {
        const uint32_t kb = std::min(KB, count - k0);
        const size_t tn = (size_t)kb * n * 32;   // bytes of one of A, B, C over the sub-batch
        uint8_t* dW = (uint8_t*)k->batchW.get((size_t)kb * nv * 32);
        uint8_t* X = (uint8_t*)k->batchX.get(3 * tn);
        uint8_t* Y = (uint8_t*)k->batchY.get(3 * tn);
        if (!dW || !X || !Y) return fail(c, SB_ERR_NOMEM, "out of device memory (Groth16 batch of " + std::to_string(kb) + " proofs)");
        CU(c, h2d(c, dW, witnesses + (size_t)k0 * nv * 32, (size_t)kb * nv * 32));
        Groth16Jobs t;
        rc = groth16_issue(c, k, dW, kb, 0, nv, 0, n, false, &t);
        if (rc) return rc;
        // the pinned area serves the next sub-batch: the host work gets its own copy, taken job by job as each lands, and
        // runs while the GPU goes on
        auto host = std::make_shared<std::vector<uint8_t>>(t.job[4].off + t.job[4].len);
        for (int i = 0; i < 5; i++) {
            CU(c, cudaEventSynchronize(c->pev[2 + i]));
            memcpy(host->data() + t.job[i].off, c->pinned + t.job[i].off, t.job[i].len);
        }
        t.tally(c);
        for (uint32_t p = k0; p < k0 + kb; p++) pool.submit([&, host, t, p, k0]() {
            const size_t q = p - k0;
            uint8_t* part = allp.data() + (size_t)p * pb;
            for (const Groth16Job& j : t.job) j.G->combine(host->data() + j.off + q * j.per, j.g, part + j.part);
            ProofScalars ps; uint8_t rsp[32]; plain_scalars(cv, r + 32 * (size_t)p, s + 32 * (size_t)p, ps.rp, ps.sp, rsp);
            groth16_fold_scalars(G1, part, ps);
        });
    }
    pool.wait();   // every fixed part and every folded partial
    for (uint32_t p = 0; p < count; p++)
        pool.submit([&, p]() { groth16_finish_folded(G1, G2, fixed[p], allp.data() + (size_t)p * pb, proofs + (size_t)p * proof_bytes); });
    pool.wait();
    tick(c, 1);
    CU(c, cudaEventSynchronize(c->ev[1]));
    prof_end(c);
    c->last_ms[0] = elapsed(c, 0, 1);
    return 0;
}

int sb_groth16_prove_batch(sb_ctx* c, uint64_t h, const uint8_t* witnesses, uint64_t n_witness, uint32_t count,
                           const uint8_t* r, const uint8_t* s, uint8_t* proofs) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (k->n_shards > 1) return fail(c, SB_ERR_ARG, "proving key was loaded sharded: use sb_groth16_prove_shard + sb_groth16_finish");
    if (n_witness != k->nVars) return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(k->nVars) + ", witness: " + std::to_string(n_witness));
    if (count == 0) return SB_OK;
    if (!witnesses || !r || !s || !proofs) return fail(c, SB_ERR_ARG, "null argument");
    return groth16_prove_batch_impl(c, k, witnesses, count, r, s, proofs);
}

int sb_groth16_prove(sb_ctx* c, uint64_t h, const uint8_t* witness, uint64_t n_witness, const uint8_t r[32], const uint8_t s[32], uint8_t* proof) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (k->n_shards > 1) return fail(c, SB_ERR_ARG, "proving key was loaded sharded: use sb_groth16_prove_shard + sb_groth16_finish");
    if (!witness || !r || !s || !proof) return fail(c, SB_ERR_ARG, "null argument");
    return groth16_prove_folded(c, k, witness, n_witness, r, s, proof);
}
int sb_groth16_prove_resident(sb_ctx* c, uint64_t h, const uint8_t r[32], const uint8_t s[32], uint8_t* proof) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (k->n_shards > 1) return fail(c, SB_ERR_ARG, "proving key was loaded sharded: use sb_groth16_prove_shard + sb_groth16_finish");
    if (!r || !s || !proof) return fail(c, SB_ERR_ARG, "null argument");
    return groth16_prove_folded(c, k, nullptr, k->nVars, r, s, proof);
}
int sb_groth16_prove_shard(sb_ctx* c, uint64_t h, const uint8_t* witness, uint64_t n_witness, int shard, int n_shards, uint8_t* partials_out) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (n_shards < 1 || shard < 0 || shard >= n_shards) return fail(c, SB_ERR_ARG, "invalid shard");
    return groth16_device(c, k, witness, n_witness, shard, n_shards, partials_out);
}
int sb_groth16_finish(sb_ctx* c, uint64_t h, const uint8_t* all, int n_shards, const uint8_t r[32], const uint8_t s[32], uint8_t* proof) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    const VkPoints vk{k->alpha1.data(), k->beta1.data(), k->beta2.data(), k->delta1.data(), k->delta2.data()};
    groth16_assemble_host(c->curve, c->g1, c->g2, vk, all, n_shards, r, s, proof);
    return 0;
}

// One proof across the ranks of a communicator (collective: every rank calls it with the same witness, r and s).
// witness may be null on every rank to reuse the resident one.  proof_affine_out may be null on ranks that do not need
// the proof; ranks that pass a buffer all receive the same bytes.
int sb_groth16_prove_dist(sb_ctx* c, uint64_t h, const uint8_t* witness, uint64_t n_witness, const uint8_t r[32], const uint8_t s[32], uint8_t* proof) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    if (!c->comm) return fail(c, SB_ERR_ARG, "context has no communicator: call sb_comm_init_rank first");
    if (!r || !s) return fail(c, SB_ERR_ARG, "null argument");
    NcclApi* nc = nccl_api(nullptr);
    VkPoints vk{k->alpha1.data(), k->beta1.data(), k->beta2.data(), k->delta1.data(), k->delta2.data()};
    const int curve = c->curve; const GroupOps G1 = c->g1, G2 = c->g2;
    std::future<FixedParts> fixed;
    if (proof) fixed = std::async(std::launch::async, [=]() { return groth16_fixed_parts(curve, G1, G2, vk, r, s); });
    ProofScalars ps; uint8_t rsp[32]; plain_scalars(curve, r, s, ps.rp, ps.sp, rsp);
    const size_t pb = sb_groth16_partials_bytes(c);
    uint8_t* mine = c->h_xchg + pb * c->world;
    int rc = groth16_device(c, k, witness, n_witness, c->rank, c->world, mine, &ps, true);
    if (rc) { if (proof) fixed.get(); return rc; }
    cudaError_t e = cudaMemcpyAsync((uint8_t*)c->d_xchg + pb * c->rank, mine, pb, cudaMemcpyHostToDevice, c->stream);
    ncclResult_t nr = ncclSuccess;
    if (e == cudaSuccess) nr = nc->AllGather((const uint8_t*)c->d_xchg + pb * c->rank, c->d_xchg, pb, ncclUint8, c->comm, c->stream);
    if (e == cudaSuccess && nr == ncclSuccess && proof) e = cudaMemcpyAsync(c->h_xchg, c->d_xchg, pb * c->world, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (proof) {
        FixedParts f = fixed.get();
        if (e == cudaSuccess && nr == ncclSuccess) {
            const uint32_t x1 = G1.xyzz_bytes;
            std::vector<uint8_t> acc(pb, 0);
            for (int i = 0; i < c->world; i++) {
                const uint8_t* p = c->h_xchg + (size_t)i * pb;
                G1.add(acc.data(), p); G1.add(acc.data() + 2 * x1, p + 2 * x1); G2.add(acc.data() + 4 * x1, p + 4 * x1);
            }
            groth16_finish_folded(G1, G2, f, acc.data(), proof);
        }
    }
    if (nr != ncclSuccess) return fail(c, SB_ERR_CUDA, std::string("ncclAllGather: ") + nc->GetErrorString(nr));
    if (e != cudaSuccess) return cuda_fail(c, e, "partial exchange");
    return 0;
}

// ---- single-process multi-GPU convenience (what a Node addon calls): one context per device, one host thread per
// context inside each call.  SURVEY §8b: sb_create(curve, device_ids, n_devices) with the communicator built here.
int sb_create_multi(int curve, const int* device_ids, int n_devices, sb_ctx** out) {
    if (!device_ids || !out || n_devices < 1 || n_devices > 64) return SB_ERR_ARG;
    for (int i = 0; i < n_devices; i++) out[i] = nullptr;
    int rc = 0;
    for (int i = 0; i < n_devices && !rc; i++) rc = sb_create(curve, device_ids[i], &out[i]);
    uint8_t id[128];
    if (!rc && n_devices > 1) rc = sb_comm_unique_id(id);
    if (!rc && n_devices > 1) {
        std::vector<std::future<int>> f;
        for (int i = 0; i < n_devices; i++) f.push_back(std::async(std::launch::async, [=]() { return sb_comm_init_rank(out[i], n_devices, i, id); }));
        for (auto& x : f) { int r = x.get(); if (r && !rc) rc = r; }
    }
    if (rc) { for (int i = 0; i < n_devices; i++) { if (out[i]) sb_destroy(out[i]); out[i] = nullptr; } }
    return rc;
}
int sb_groth16_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!ctxs || !zkey || !handles || n < 1) return SB_ERR_ARG;
    std::vector<std::future<int>> f;
    for (int i = 0; i < n; i++) f.push_back(std::async(std::launch::async, [=]() { return sb_groth16_load_sharded(ctxs[i], zkey, zkey_len, i, n, &handles[i]); }));
    int rc = 0; for (auto& x : f) { int r = x.get(); if (r && !rc) rc = r; }
    return rc;
}
int sb_groth16_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                           const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out) {
    if (!ctxs || !handles || n < 1 || !proof_affine_out) return SB_ERR_ARG;
    if (n == 1) return sb_groth16_prove(ctxs[0], handles[0], witness, n_witness, r, s, proof_affine_out);
    for (int i = 0; i < n; i++) {   // before any rank enters the collective: a refusal on some ranks only would leave the others waiting
        SB_LOCK(ctxs[i]);
        const Groth16Key* k = get_key(ctxs[i], handles[i]);
        if (k && k->replica_id) return fail(ctxs[0], SB_ERR_ARG, "sb_groth16_prove_multi: the key of rank " + std::to_string(i) +
                                                                     " is a replica of sb_groth16_load_replicas: prove with sb_groth16_prove_batch_multi");
    }
    std::vector<std::future<int>> f;
    for (int i = 0; i < n; i++)
        f.push_back(std::async(std::launch::async, [=]() { return sb_groth16_prove_dist(ctxs[i], handles[i], witness, n_witness, r, s, i == 0 ? proof_affine_out : nullptr); }));
    int rc = 0; for (auto& x : f) { int r2 = x.get(); if (r2 && !rc) rc = r2; }
    return rc;
}

// ---- host-only helpers (no context, no device): the combine/assembly half of the multi-GPU path, testable on CPU
static void host_ops(int curve, GroupOps& g1, GroupOps& g2) {
    if (curve == SB_BN254) { g1 = SB_GROUP_OPS(bn254_g1, 64); g2 = SB_GROUP_OPS(bn254_g2, 128); }
    else { g1 = SB_GROUP_OPS(bls12381_g1, 96); g2 = SB_GROUP_OPS(bls12381_g2, 192); }
}
int sb_host_sum_partials(int curve, int group, const uint8_t* partials, int count, uint8_t* out_jacobian) {
    if ((curve != SB_BN254 && curve != SB_BLS12_381) || (group != SB_G1 && group != SB_G2) || count < 0) return SB_ERR_ARG;
    GroupOps g1, g2; host_ops(curve, g1, g2);
    const GroupOps& G = group == SB_G1 ? g1 : g2;
    std::vector<uint8_t> acc(G.xyzz_bytes, 0);
    for (int i = 0; i < count; i++) G.add(acc.data(), partials + (size_t)i * G.xyzz_bytes);
    G.to_jacobian(acc.data(), out_jacobian);
    return 0;
}
int sb_host_partial_from_affine(int curve, int group, const uint8_t* affine, uint8_t* partial_out) {
    if ((curve != SB_BN254 && curve != SB_BLS12_381) || (group != SB_G1 && group != SB_G2)) return SB_ERR_ARG;
    GroupOps g1, g2; host_ops(curve, g1, g2);
    (group == SB_G1 ? g1 : g2).from_affine(affine, partial_out);
    return 0;
}
uint32_t sb_host_partial_bytes(int curve, int group) {
    GroupOps g1, g2; if (curve != SB_BN254 && curve != SB_BLS12_381) return 0; host_ops(curve, g1, g2);
    return group == SB_G1 ? g1.xyzz_bytes : g2.xyzz_bytes;
}
int sb_host_groth16_finish(int curve, const uint8_t* vk_alpha1, const uint8_t* vk_beta1, const uint8_t* vk_beta2,
                           const uint8_t* vk_delta1, const uint8_t* vk_delta2, const uint8_t* partials_all_ranks, int n_shards,
                           const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out) {
    if ((curve != SB_BN254 && curve != SB_BLS12_381) || n_shards < 1) return SB_ERR_ARG;
    GroupOps G1, G2; host_ops(curve, G1, G2);
    const VkPoints vk{vk_alpha1, vk_beta1, vk_beta2, vk_delta1, vk_delta2};
    groth16_assemble_host(curve, G1, G2, vk, partials_all_ranks, n_shards, r, s, proof_affine_out);
    return 0;
}
// point range of shard `shard` of `n_shards` over `total` points (the split sb_groth16_prove_shard uses)
void sb_shard_range(uint64_t total, int shard, int n_shards, uint64_t* first, uint64_t* count) {
    uint64_t per = (total + n_shards - 1) / n_shards, lo = std::min(total, per * (uint64_t)shard);
    *first = lo; *count = std::min(total - lo, per);
}

int sb_groth16_prove_wtns(sb_ctx* c, uint64_t h, const uint8_t* w, uint64_t wlen, const uint8_t r[32], const uint8_t s[32], uint8_t* proof) { SB_LOCK(c);
    Groth16Key* k = get_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid groth16 handle");
    Wtns wt; std::string err;
    if (wtns_parse(w, wlen, wt, err)) return fail(c, SB_ERR_FORMAT, err);
    if (!modulus_matches(wt.q, wt.n8, c->curve, true)) return fail(c, SB_ERR_ARG, "Curve of the witness does not match the curve of the proving key");
    return sb_groth16_prove(c, h, wt.values.p, wt.nWitness, r, s, proof);
}

}  // extern "C"

// ================================================================================================================
// PLONK (src/plonk_prove.js) — templates live outside the extern "C" block
#include "api_plonk.inl"
#include "api_fflonk.inl"
#include "api_verify.inl"

// ---- one PLONK / fflonk proof on several devices (sb_plonk_load_multi .. sb_fflonk_prove_multi)
// a key of a multi load holds one PTau range only, so the single-device entries refuse it
#define MULTI_HANDLE(proto) "this " #proto " key is one shard of sb_" #proto "_load_multi: prove with sb_" #proto "_prove_multi"

// sb_*_load_multi: argument checks, then rank i's part loaded by load(ctxs[i], i, id, &handles[i]) on its own thread (under
// that context's lock).  A rank on another device than rank 0 gets peer access to rank 0's device where the devices allow
// it (otherwise the peer copies stage through the host).  If a rank fails, the handles made are released and rank 0's
// context reports the failing rank's code and message.
// Checks every sb_*_load_multi / sb_*_prove_multi call starts with, before any context is touched: the message of a
// refusal is kept for the calling thread only (what sb_last_error(ctxs[0]) returns to it).
static int multi_ctx_args(sb_ctx* const* ctxs, int n, const char* name) {
    if (!ctxs || n < 1 || n > 64) return SB_ERR_ARG;
    for (int i = 0; i < n; i++) if (!ctxs[i]) return SB_ERR_ARG;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < i; j++)
            if (ctxs[i] == ctxs[j]) {
                t_err_ctx = ctxs[0];
                t_err = std::string(name) + ": context " + std::to_string(i) + " is context " + std::to_string(j) + " again";
                return SB_ERR_ARG;
            }
    return 0;
}

// id numbers the call (g_multi_loads).  sb_*_load_replicas passes peer = false: its ranks never copy between devices.
static int load_multi(sb_ctx* const* ctxs, int n, uint64_t* handles, const std::function<int(sb_ctx*, int, uint64_t, uint64_t*)>& load,
                      int (*release)(sb_ctx*, uint64_t), const char* name, bool peer = true) {
    if (int rc = multi_ctx_args(ctxs, n, name)) return rc;
    if (!handles) return fail(ctxs[0], SB_ERR_ARG, "null argument");
    for (int i = 0; i < n; i++) handles[i] = 0;
    const uint64_t id = ++g_multi_loads;
    std::vector<std::future<int>> f;
    for (int i = 0; i < n; i++)
        f.push_back(std::async(std::launch::async, [&, i]() {
            sb_ctx* c = ctxs[i];
            SB_LOCK(c);
            cudaSetDevice(c->device);
            int rc = load(c, i, id, &handles[i]);
            const int d0 = ctxs[0]->device;
            int can = 0;
            if (!rc && peer && c->device != d0 && cudaDeviceCanAccessPeer(&can, c->device, d0) == cudaSuccess && can) {
                cudaError_t e = cudaDeviceEnablePeerAccess(d0, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) rc = cuda_fail(c, e, "cudaDeviceEnablePeerAccess");
                cudaGetLastError();
            }
            return rc;
        }));
    std::vector<int> rcs(n);
    for (int i = 0; i < n; i++) rcs[i] = f[i].get();
    for (int i = 0; i < n; i++) {
        if (!rcs[i]) continue;
        const std::string msg = ctxs[i]->err;
        for (int j = 0; j < n; j++) if (handles[j]) { release(ctxs[j], handles[j]); handles[j] = 0; }
        return fail(ctxs[0], rcs[i], msg);
    }
    return 0;
}

// Whether keys[i] = k is rank i of the load keys[0] = k0 belongs to: one sb_*_load_multi call (n = 1: a single-device key),
// or one sb_*_load_replicas call.
template <class K> static bool multi_rank(const K* k, const K* k0, int i, int n) {
    return n == 1 ? k->multi_id == 0 : (k->multi_id && k->multi_id == k0->multi_id && k->rank == i && k->n_ranks == n);
}
template <class K> static bool replica_rank(const K* k, const K* k0, int i, int n) {
    return k->replica_id && k->replica_id == k0->replica_id && k->replica == i && k->n_replicas == n;
}

// Argument checks of sb_*_prove_multi and sb_*_prove_batch_multi, before any device work: pointers, n, distinct contexts of
// one curve.  Then every context is locked (in address order, so that calls on overlapping sets of contexts cannot
// deadlock) and the handles are checked: same_load(keys[i], keys[0], i, n) for every rank.
template <class K> static int prove_multi_args(sb_ctx* const* ctxs, const uint64_t* handles, int n, const void* witness, const void* blinders,
                                               const void* proof, K* (*get)(sb_ctx*, uint64_t), const char* name,
                                               std::vector<std::unique_lock<std::recursive_mutex>>& locks, std::vector<K*>& keys,
                                               bool (*same_load)(const K*, const K*, int, int) = multi_rank<K>, const char* load = "load_multi") {
    if (int rc = multi_ctx_args(ctxs, n, name)) return rc;
    sb_ctx* c0 = ctxs[0];
    if (!handles || !witness || !blinders || !proof) return fail(c0, SB_ERR_ARG, "null argument");
    for (int i = 0; i < n; i++)
        if (ctxs[i]->curve != c0->curve) return fail(c0, SB_ERR_ARG, std::string(name) + ": the contexts are not all of one curve");
    std::vector<sb_ctx*> order(ctxs, ctxs + n);
    std::sort(order.begin(), order.end(), std::less<sb_ctx*>());
    for (sb_ctx* c : order) locks.emplace_back(c->mu);
    keys.assign(n, nullptr);
    for (int i = 0; i < n; i++) {
        keys[i] = get(ctxs[i], handles[i]);
        if (!keys[i]) return fail(c0, SB_ERR_ARG, std::string(name) + ": invalid handle of rank " + std::to_string(i));
    }
    for (int i = 0; i < n; i++)
        if (!same_load(keys[i], keys[0], i, n))
            return fail(c0, SB_ERR_ARG, std::string(name) + ": the handles do not come from one " + load + " call of these " + std::to_string(n) + " contexts, in this order");
    return 0;
}

// sb_*_prove_batch_multi after its argument checks, with every context locked: rank i proves the proofs
// [lo, lo + cnt) = sb_shard_range(count, i, n) with prove(i, lo, cnt, statuses of those proofs or null) on a host thread of
// its own.  with_status (PLONK / fflonk): the per-proof statuses are collected and copied to status_out (when not null)
// unless a rank failed for another reason than refused proofs.  Returns 0; or the lowest such rank's code, with its message
// on ctxs[0]; or SB_ERR_ARG with the text of the lowest-index refused proof, which is the message of the lowest rank that
// refused one (each rank reports its own lowest).  sb_last_ms(ctxs[0], 0) = the host wall clock of the call;
// sb_last_ms(ctxs[i], 0), i > 0 = rank i's batch (0 for an empty range).
static int batch_multi_run(sb_ctx* const* ctxs, int n, uint32_t count, bool with_status, int32_t* status_out,
                           const std::function<int(int, uint32_t, uint32_t, int32_t*)>& prove) {
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<int32_t> status(with_status ? count : 0, 0);
    std::vector<std::future<int>> f;
    for (int i = 0; i < n; i++)
        f.push_back(std::async(std::launch::async, [&, i]() {
            uint64_t lo, cnt; sb_shard_range(count, i, n, &lo, &cnt);
            ctxs[i]->last_ms[0] = 0;
            if (!cnt) return 0;
            cudaSetDevice(ctxs[i]->device);
            return prove(i, (uint32_t)lo, (uint32_t)cnt, with_status ? status.data() + lo : nullptr);
        }));
    std::vector<int> rcs(n);
    for (int i = 0; i < n; i++) rcs[i] = f[i].get();
    ctxs[0]->last_ms[0] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    int refused = -1;
    for (int i = 0; i < n; i++) {
        if (!rcs[i]) continue;
        uint64_t lo, cnt; sb_shard_range(count, i, n, &lo, &cnt);
        const bool any = with_status && std::any_of(status.begin() + lo, status.begin() + lo + cnt, [](int32_t s) { return s != 0; });
        if (rcs[i] != SB_ERR_ARG || !any) return fail(ctxs[0], rcs[i], ctxs[i]->err);
        if (refused < 0) refused = i;
    }
    if (status_out) memcpy(status_out, status.data(), status.size() * sizeof(int32_t));
    return refused < 0 ? 0 : fail(ctxs[0], SB_ERR_ARG, ctxs[refused]->err);
}

extern "C" {

int sb_plonk_load(sb_ctx* c, const uint8_t* zkey, uint64_t len, uint64_t* handle) { SB_LOCK(c);
    if (!c || !zkey || !handle) return SB_ERR_ARG;
    cudaSetDevice(c->device);
    return c->curve == SB_BN254 ? plonk_load_impl<BnFr>(c, zkey, len, handle) : plonk_load_impl<BlsFr>(c, zkey, len, handle);
}
// maps the file read-only and hands it to the byte loader: the sections are read once, front to back, through the pinned
// staging buffers (h2d), so the key never sits in anonymous host memory
static int load_mapped(sb_ctx* c, const char* path, uint64_t* handle, int (*load)(sb_ctx*, const uint8_t*, uint64_t, uint64_t*)) {
    if (!c || !path || !handle) return SB_ERR_ARG;
    int fd = open(path, O_RDONLY);
    if (fd < 0) return fail(c, SB_ERR_FORMAT, std::string("cannot open ") + path);
    struct stat st;
    if (fstat(fd, &st) != 0 || st.st_size <= 0) { close(fd); return fail(c, SB_ERR_FORMAT, std::string("cannot stat ") + path); }
    void* p = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (p == MAP_FAILED) return fail(c, SB_ERR_FORMAT, std::string("cannot map ") + path);
    madvise(p, (size_t)st.st_size, MADV_SEQUENTIAL);
    int rc = load(c, (const uint8_t*)p, (uint64_t)st.st_size, handle);
    munmap(p, (size_t)st.st_size);
    return rc;
}
int sb_groth16_load_file(sb_ctx* c, const char* path, uint64_t* handle) { SB_LOCK(c); return load_mapped(c, path, handle, sb_groth16_load); }
int sb_plonk_load_file(sb_ctx* c, const char* path, uint64_t* handle) { SB_LOCK(c); return load_mapped(c, path, handle, sb_plonk_load); }
static PlonkKeyDev* get_plonk_key(sb_ctx* c, uint64_t h) { return (c && h >= 1 && h <= c->plonk_keys.size()) ? c->plonk_keys[h - 1] : nullptr; }
int sb_plonk_info(sb_ctx* c, uint64_t h, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_size, uint32_t* n_additions) { SB_LOCK(c);
    PlonkKeyDev* k = get_plonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid plonk handle");
    if (n_vars) *n_vars = k->z.nVars; if (n_public) *n_public = k->z.nPublic; if (domain_size) *domain_size = k->z.n; if (n_additions) *n_additions = k->z.nAdditions;
    return 0;
}
uint32_t sb_plonk_proof_bytes(sb_ctx* c) { return c ? 9 * c->g1.aff_bytes + 6 * 32 : 0; }
int sb_plonk_prove(sb_ctx* c, uint64_t h, const uint8_t* witness, uint64_t n_witness, const uint8_t* blinders, uint8_t* proof) { SB_LOCK(c);
    PlonkKeyDev* k = get_plonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid plonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(plonk));
    if (!witness || !blinders || !proof) return fail(c, SB_ERR_ARG, "null argument");
    cudaSetDevice(c->device);
    return c->curve == SB_BN254 ? plonk_prove_impl<BnFq, BnFr>(c, k, witness, n_witness, blinders, proof)
                                : plonk_prove_impl<BlsFq, BlsFr>(c, k, witness, n_witness, blinders, proof);
}
int sb_plonk_prove_resident(sb_ctx* c, uint64_t h, const uint8_t* blinders, uint8_t* proof) { SB_LOCK(c);
    PlonkKeyDev* k = get_plonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid plonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(plonk));
    if (!blinders || !proof) return fail(c, SB_ERR_ARG, "null argument");
    if (!k->n_wit_resident) return fail(c, SB_ERR_ARG, "no witness resident for this proving key: call sb_plonk_prove first");
    cudaSetDevice(c->device);
    return c->curve == SB_BN254 ? plonk_prove_impl<BnFq, BnFr>(c, k, nullptr, 0, blinders, proof)
                                : plonk_prove_impl<BlsFq, BlsFr>(c, k, nullptr, 0, blinders, proof);
}
int sb_plonk_prove_batch(sb_ctx* c, uint64_t h, const uint8_t* witnesses, uint64_t n_witness, uint32_t count, const uint8_t* blinders,
                         uint8_t* proofs, int32_t* status) { SB_LOCK(c);
    PlonkKeyDev* k = get_plonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid plonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(plonk));
    if (n_witness != (uint64_t)k->z.nVars - k->z.nAdditions)                                          // plonk_prove.js:66-68
        return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(k->z.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k->z.nAdditions));
    if (count == 0) return SB_OK;
    if (!witnesses || !blinders || !proofs) return fail(c, SB_ERR_ARG, "null argument");
    cudaSetDevice(c->device);
    return c->curve == SB_BN254 ? plonk_prove_batch_impl<BnFq, BnFr>(c, k, witnesses, n_witness, count, blinders, proofs, status)
                                : plonk_prove_batch_impl<BlsFq, BlsFr>(c, k, witnesses, n_witness, count, blinders, proofs, status);
}
int sb_plonk_release(sb_ctx* c, uint64_t h) { SB_LOCK(c);
    PlonkKeyDev* k = get_plonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid plonk handle");
    cudaSetDevice(c->device); cudaStreamSynchronize(c->stream);
    plonk_free_key(k); c->plonk_keys[h - 1] = nullptr;
    return 0;
}

// ---- fflonk (src/fflonk_prove.js)
int sb_fflonk_load(sb_ctx* c, const uint8_t* zkey, uint64_t len, uint64_t* handle) { SB_LOCK(c);
    if (!c || !zkey || !handle) return SB_ERR_ARG;
    if (c->curve != SB_BN254) return fail(c, SB_ERR_ARG, "fflonk is defined on bn128 only (src/fflonk_setup.js:534-557)");
    cudaSetDevice(c->device);
    return fflonk_load_impl<BnFr>(c, zkey, len, handle);
}
int sb_fflonk_load_file(sb_ctx* c, const char* path, uint64_t* handle) { SB_LOCK(c); return load_mapped(c, path, handle, sb_fflonk_load); }
static FflonkKeyDev* get_fflonk_key(sb_ctx* c, uint64_t h) { return (c && h >= 1 && h <= c->fflonk_keys.size()) ? c->fflonk_keys[h - 1] : nullptr; }
int sb_fflonk_info(sb_ctx* c, uint64_t h, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_size, uint32_t* n_additions) { SB_LOCK(c);
    FflonkKeyDev* k = get_fflonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid fflonk handle");
    if (n_vars) *n_vars = k->z.nVars; if (n_public) *n_public = k->z.nPublic; if (domain_size) *domain_size = k->z.n; if (n_additions) *n_additions = k->z.nAdditions;
    return 0;
}
uint32_t sb_fflonk_proof_bytes(sb_ctx* c) { return c ? 4 * c->g1.aff_bytes + 16 * 32 : 0; }
int sb_fflonk_prove(sb_ctx* c, uint64_t h, const uint8_t* witness, uint64_t n_witness, const uint8_t* blinders, uint8_t* proof) { SB_LOCK(c);
    FflonkKeyDev* k = get_fflonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid fflonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(fflonk));
    if (!witness || !blinders || !proof) return fail(c, SB_ERR_ARG, "null argument");
    cudaSetDevice(c->device);
    return fflonk_prove_impl<BnFq, BnFr>(c, k, witness, n_witness, blinders, proof);
}
int sb_fflonk_prove_resident(sb_ctx* c, uint64_t h, const uint8_t* blinders, uint8_t* proof) { SB_LOCK(c);
    FflonkKeyDev* k = get_fflonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid fflonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(fflonk));
    if (!blinders || !proof) return fail(c, SB_ERR_ARG, "null argument");
    if (!k->n_wit_resident) return fail(c, SB_ERR_ARG, "no witness resident for this proving key: call sb_fflonk_prove first");
    cudaSetDevice(c->device);
    return fflonk_prove_impl<BnFq, BnFr>(c, k, nullptr, 0, blinders, proof);
}
int sb_fflonk_prove_batch(sb_ctx* c, uint64_t h, const uint8_t* witnesses, uint64_t n_witness, uint32_t count, const uint8_t* blinders,
                          uint8_t* proofs, int32_t* status) { SB_LOCK(c);
    FflonkKeyDev* k = get_fflonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid fflonk handle");
    if (k->multi_id) return fail(c, SB_ERR_ARG, MULTI_HANDLE(fflonk));
    if (n_witness != (uint64_t)k->z.nVars - k->z.nAdditions)                                          // fflonk_prove.js:79-81
        return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(k->z.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k->z.nAdditions));
    if (count == 0) return SB_OK;
    if (!witnesses || !blinders || !proofs) return fail(c, SB_ERR_ARG, "null argument");
    cudaSetDevice(c->device);
    return fflonk_prove_batch_impl<BnFq, BnFr>(c, k, witnesses, n_witness, count, blinders, proofs, status);
}
int sb_fflonk_release(sb_ctx* c, uint64_t h) { SB_LOCK(c);
    FflonkKeyDev* k = get_fflonk_key(c, h); if (!k) return fail(c, SB_ERR_ARG, "invalid fflonk handle");
    cudaSetDevice(c->device); cudaStreamSynchronize(c->stream);
    fflonk_free_key(k); c->fflonk_keys[h - 1] = nullptr;
    return 0;
}

int sb_plonk_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!zkey) return SB_ERR_ARG;
    return load_multi(ctxs, n, handles, [=](sb_ctx* c, int i, uint64_t id, uint64_t* h) {
        return c->curve == SB_BN254 ? plonk_load_impl<BnFr>(c, zkey, zkey_len, h, i, n, n > 1 ? id : 0)
                                    : plonk_load_impl<BlsFr>(c, zkey, zkey_len, h, i, n, n > 1 ? id : 0);
    }, sb_plonk_release, "sb_plonk_load_multi");
}
int sb_plonk_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                         const uint8_t* blinders, uint8_t* proof) {
    std::vector<std::unique_lock<std::recursive_mutex>> locks; std::vector<PlonkKeyDev*> keys;
    int rc = prove_multi_args(ctxs, handles, n, witness, blinders, proof, get_plonk_key, "sb_plonk_prove_multi", locks, keys);
    if (rc) return rc;
    sb_ctx* c = ctxs[0];
    if (n == 1) return sb_plonk_prove(c, handles[0], witness, n_witness, blinders, proof);
    cudaSetDevice(c->device);
    PlonkRanks rk{ctxs, (PlonkKeyBase* const*)nullptr, n, nullptr};
    std::vector<PlonkKeyBase*> base(keys.begin(), keys.end()); rk.keys = base.data();
    CU(c, cudaEventCreateWithFlags(&rk.ready, cudaEventDisableTiming));
    if (c->curve == SB_BN254) { CudaShardedBackend<Fp<BnFr>, CudaPlonkBackend> be; be.ranks = &rk; rc = plonk_prove_impl<BnFq, BnFr>(c, keys[0], witness, n_witness, blinders, proof, be); }
    else { CudaShardedBackend<Fp<BlsFr>, CudaPlonkBackend> be; be.ranks = &rk; rc = plonk_prove_impl<BlsFq, BlsFr>(c, keys[0], witness, n_witness, blinders, proof, be); }
    cudaEventDestroy(rk.ready);
    return rc;
}
int sb_fflonk_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!zkey) return SB_ERR_ARG;
    return load_multi(ctxs, n, handles, [=](sb_ctx* c, int i, uint64_t id, uint64_t* h) {
        if (c->curve != SB_BN254) return fail(c, SB_ERR_ARG, "fflonk is defined on bn128 only (src/fflonk_setup.js:534-557)");
        return fflonk_load_impl<BnFr>(c, zkey, zkey_len, h, i, n, n > 1 ? id : 0);
    }, sb_fflonk_release, "sb_fflonk_load_multi");
}
int sb_fflonk_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                          const uint8_t* blinders, uint8_t* proof) {
    std::vector<std::unique_lock<std::recursive_mutex>> locks; std::vector<FflonkKeyDev*> keys;
    int rc = prove_multi_args(ctxs, handles, n, witness, blinders, proof, get_fflonk_key, "sb_fflonk_prove_multi", locks, keys);
    if (rc) return rc;
    sb_ctx* c = ctxs[0];
    if (n == 1) return sb_fflonk_prove(c, handles[0], witness, n_witness, blinders, proof);
    cudaSetDevice(c->device);
    PlonkRanks rk{ctxs, (PlonkKeyBase* const*)nullptr, n, nullptr};
    std::vector<PlonkKeyBase*> base(keys.begin(), keys.end()); rk.keys = base.data();
    CU(c, cudaEventCreateWithFlags(&rk.ready, cudaEventDisableTiming));
    CudaShardedBackend<Fp<BnFr>, CudaFflonkBackend> be; be.ranks = &rk;
    rc = fflonk_prove_impl<BnFq, BnFr>(c, keys[0], witness, n_witness, blinders, proof, be);
    cudaEventDestroy(rk.ready);
    return rc;
}

}  // extern "C"

// ---- batches of one key on several devices (sb_*_load_replicas, sb_*_prove_batch_multi)
// sb_*_load_replicas: load_multi with the whole key on every context, each handle marked as replica i of the call.
template <class K> static int load_replicas(sb_ctx* const* ctxs, int n, uint64_t* handles, const std::function<int(sb_ctx*, uint64_t*)>& load,
                                            std::vector<K*> sb_ctx::*keys, int (*release)(sb_ctx*, uint64_t), const char* name) {
    return load_multi(ctxs, n, handles, [&](sb_ctx* c, int i, uint64_t id, uint64_t* h) {
        int rc = load(c, h);
        if (!rc) { K* k = (c->*keys)[*h - 1]; k->replica_id = id; k->replica = i; k->n_replicas = n; }
        return rc;
    }, release, name, false);
}

extern "C" {

int sb_groth16_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!zkey) return SB_ERR_ARG;
    return load_replicas<Groth16Key>(ctxs, n, handles, [=](sb_ctx* c, uint64_t* h) { return groth16_load_impl(c, zkey, zkey_len, 0, 1, h); },
                                     &sb_ctx::keys, sb_groth16_release, "sb_groth16_load_replicas");
}
int sb_plonk_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!zkey) return SB_ERR_ARG;
    return load_replicas<PlonkKeyDev>(ctxs, n, handles, [=](sb_ctx* c, uint64_t* h) { return sb_plonk_load(c, zkey, zkey_len, h); },
                                      &sb_ctx::plonk_keys, sb_plonk_release, "sb_plonk_load_replicas");
}
int sb_fflonk_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles) {
    if (!zkey) return SB_ERR_ARG;
    return load_replicas<FflonkKeyDev>(ctxs, n, handles, [=](sb_ctx* c, uint64_t* h) { return sb_fflonk_load(c, zkey, zkey_len, h); },
                                       &sb_ctx::fflonk_keys, sb_fflonk_release, "sb_fflonk_load_replicas");
}

int sb_groth16_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses, uint64_t n_witness,
                                 uint32_t count, const uint8_t* r, const uint8_t* s, uint8_t* proofs) {
    std::vector<std::unique_lock<std::recursive_mutex>> locks; std::vector<Groth16Key*> keys;
    int rc = prove_multi_args(ctxs, handles, n, witnesses, r && s ? r : nullptr, proofs, get_key, "sb_groth16_prove_batch_multi", locks, keys,
                              replica_rank<Groth16Key>, "load_replicas");
    if (rc) return rc;
    sb_ctx* c = ctxs[0];
    if (n == 1) return sb_groth16_prove_batch(c, handles[0], witnesses, n_witness, count, r, s, proofs);
    if (n_witness != keys[0]->nVars) return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(keys[0]->nVars) + ", witness: " + std::to_string(n_witness));
    if (count == 0) return SB_OK;
    // the ranks' host pools share the cores
    const unsigned threads = std::max(1u, std::thread::hardware_concurrency() / n);
    const size_t pb = 2 * c->g1.aff_bytes + c->g2.aff_bytes;
    return batch_multi_run(ctxs, n, count, false, nullptr, [&](int i, uint32_t lo, uint32_t cnt, int32_t*) {
        return groth16_prove_batch_impl(ctxs[i], keys[i], witnesses + (size_t)lo * n_witness * 32, cnt, r + (size_t)lo * 32, s + (size_t)lo * 32,
                                        proofs + lo * pb, threads);
    });
}
int sb_plonk_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses, uint64_t n_witness,
                               uint32_t count, const uint8_t* blinders, uint8_t* proofs, int32_t* status) {
    std::vector<std::unique_lock<std::recursive_mutex>> locks; std::vector<PlonkKeyDev*> keys;
    int rc = prove_multi_args(ctxs, handles, n, witnesses, blinders, proofs, get_plonk_key, "sb_plonk_prove_batch_multi", locks, keys,
                              replica_rank<PlonkKeyDev>, "load_replicas");
    if (rc) return rc;
    sb_ctx* c = ctxs[0];
    if (n == 1) return sb_plonk_prove_batch(c, handles[0], witnesses, n_witness, count, blinders, proofs, status);
    const PlonkZkey& z = keys[0]->z;
    if (n_witness != (uint64_t)z.nVars - z.nAdditions)
        return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(z.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(z.nAdditions));
    if (count == 0) return SB_OK;
    const size_t pb = sb_plonk_proof_bytes(c);
    return batch_multi_run(ctxs, n, count, true, status, [&](int i, uint32_t lo, uint32_t cnt, int32_t* st) {
        const uint8_t* w = witnesses + (size_t)lo * n_witness * 32; const uint8_t* b = blinders + (size_t)lo * 11 * 32;
        return c->curve == SB_BN254 ? plonk_prove_batch_impl<BnFq, BnFr>(ctxs[i], keys[i], w, n_witness, cnt, b, proofs + lo * pb, st)
                                    : plonk_prove_batch_impl<BlsFq, BlsFr>(ctxs[i], keys[i], w, n_witness, cnt, b, proofs + lo * pb, st);
    });
}
int sb_fflonk_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses, uint64_t n_witness,
                                uint32_t count, const uint8_t* blinders, uint8_t* proofs, int32_t* status) {
    std::vector<std::unique_lock<std::recursive_mutex>> locks; std::vector<FflonkKeyDev*> keys;
    int rc = prove_multi_args(ctxs, handles, n, witnesses, blinders, proofs, get_fflonk_key, "sb_fflonk_prove_batch_multi", locks, keys,
                              replica_rank<FflonkKeyDev>, "load_replicas");
    if (rc) return rc;
    sb_ctx* c = ctxs[0];
    if (n == 1) return sb_fflonk_prove_batch(c, handles[0], witnesses, n_witness, count, blinders, proofs, status);
    const FflonkZkey& z = keys[0]->z;
    if (n_witness != (uint64_t)z.nVars - z.nAdditions)
        return fail(c, SB_ERR_ARG, "Invalid witness length. Circuit: " + std::to_string(z.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(z.nAdditions));
    if (count == 0) return SB_OK;
    const size_t pb = sb_fflonk_proof_bytes(c);
    return batch_multi_run(ctxs, n, count, true, status, [&](int i, uint32_t lo, uint32_t cnt, int32_t* st) {
        return fflonk_prove_batch_impl<BnFq, BnFr>(ctxs[i], keys[i], witnesses + (size_t)lo * n_witness * 32, n_witness, cnt,
                                                   blinders + (size_t)lo * 9 * 32, proofs + lo * pb, st);
    });
}

}  // extern "C"
