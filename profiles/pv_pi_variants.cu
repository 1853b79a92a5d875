// pv_pi_variants.cu — the two forms of PI(xi) = -sum s_i L_{i+1}(xi) and L_1(xi) the PLONK / fflonk verifiers could use,
// timed against each other (profiles/bench_pv_pi.py builds and runs this):
//   batched    one thread per proof: verify_plonk.cuh's pv_pi, the sum as one fraction, one inversion per proof
//   per_input  one thread per (proof, public input) computing L_{i+1} with its own inversion and s_i L_{i+1}, then one
//              thread per proof summing the terms
// Both run on the same random xi, zh and signals; the results are compared before any time is printed.
//   pv_pi_variants COUNT N_PUBLIC REPS  ->  one JSON line per curve
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
#include "../snarkjs_b200/csrc/verify_plonk.cuh"
using namespace sb;

template <class P> __global__ void k_batched(const FrF<P>* xi, const FrF<P>* zh, FrF<P> w, uint32_t power, const FrPlain* pub, uint32_t np,
                                             uint32_t count, FrF<P>* pi, FrF<P>* l1) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < count) pv_pi<P>(xi[k], zh[k], w, power, pub + (uint64_t)k * np, np, l1[k], pi[k]);
}
template <class P> __global__ void k_terms(const FrF<P>* xi, const FrF<P>* zh, const FrF<P>* wpow, FrF<P> nf, const FrPlain* pub, uint32_t np,
                                           uint64_t n, FrF<P>* term, FrF<P>* l1) {
    typedef FrF<P> R;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint64_t k = t / np;
    const uint32_t i = (uint32_t)(t % np);
    const R L = fr_div(R::mul(wpow[i], zh[k]), R::mul(nf, R::sub(xi[k], wpow[i])));
    term[t] = R::mul(fr_mont<P>(pub[t]), L);
    if (i == 0) l1[k] = L;
}
template <class P> __global__ void k_sum(const FrF<P>* term, uint32_t np, uint32_t count, FrF<P>* pi) {
    typedef FrF<P> R;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    R s = R::zero();
    for (uint32_t i = 0; i < np; i++) s = R::sub(s, term[(uint64_t)k * np + i]);
    pi[k] = s;
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <class P> static void run(const char* name, uint32_t count, uint32_t np, int reps) {
    typedef FrF<P> R;
    const uint32_t power = 20;
    std::mt19937_64 rng(7);
    auto rnd = [&]() { FrPlain p; for (int i = 0; i < 8; i++) p.v[i] = (uint32_t)rng(); p.v[7] &= 0x0fffffffu; return p; };
    std::vector<R> xi(count), zh(count);
    for (uint32_t k = 0; k < count; k++) { xi[k] = fr_mont<P>(rnd()); zh[k] = fr_mont<P>(rnd()); }
    std::vector<FrPlain> pub((size_t)count * np);
    for (auto& p : pub) p = rnd();
    const R w = fr_mont<P>(rnd());
    R nf = R::one();
    for (uint32_t i = 0; i < power; i++) nf = R::dbl(nf);
    std::vector<R> wpow(np);
    R wq = R::one();
    for (uint32_t i = 0; i < np; i++) { wpow[i] = wq; wq = R::mul(wq, w); }
    R *d_xi, *d_zh, *d_wpow, *d_pi[2], *d_l1[2], *d_term;
    FrPlain* d_pub;
    const uint64_t n = (uint64_t)count * np;
    CK(cudaMalloc(&d_xi, count * sizeof(R))); CK(cudaMalloc(&d_zh, count * sizeof(R))); CK(cudaMalloc(&d_wpow, np * sizeof(R)));
    CK(cudaMalloc(&d_pub, n * sizeof(FrPlain))); CK(cudaMalloc(&d_term, n * sizeof(R)));
    for (int v = 0; v < 2; v++) { CK(cudaMalloc(&d_pi[v], count * sizeof(R))); CK(cudaMalloc(&d_l1[v], count * sizeof(R))); }
    CK(cudaMemcpy(d_xi, xi.data(), count * sizeof(R), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_zh, zh.data(), count * sizeof(R), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_wpow, wpow.data(), np * sizeof(R), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_pub, pub.data(), n * sizeof(FrPlain), cudaMemcpyHostToDevice));
    const unsigned bc = (count + VERIFY_THREADS - 1) / VERIFY_THREADS, bn = (unsigned)((n + 127) / 128);
    auto batched = [&]() { k_batched<P><<<bc, VERIFY_THREADS>>>(d_xi, d_zh, w, power, d_pub, np, count, d_pi[0], d_l1[0]); };
    auto per_input = [&]() {
        k_terms<P><<<bn, 128>>>(d_xi, d_zh, d_wpow, nf, d_pub, np, n, d_term, d_l1[1]);
        k_sum<P><<<bc, VERIFY_THREADS>>>(d_term, np, count, d_pi[1]);
    };
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best[2] = {1e30f, 1e30f};
    for (int rep = 0; rep <= reps; rep++) {          // rep 0 warms both up; the two alternate
        for (int v = 0; v < 2; v++) {
            CK(cudaEventRecord(e0));
            if (v == 0) batched(); else per_input();
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep && ms < best[v]) best[v] = ms;
        }
    }
    std::vector<R> pi0(count), pi1(count), l0(count), l1(count);
    CK(cudaMemcpy(pi0.data(), d_pi[0], count * sizeof(R), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(pi1.data(), d_pi[1], count * sizeof(R), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(l0.data(), d_l1[0], count * sizeof(R), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(l1.data(), d_l1[1], count * sizeof(R), cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < count; k++)
        if (!(pi0[k] == pi1[k]) || !(l0[k] == l1[k])) { fprintf(stderr, "%s: the two forms differ at proof %u\n", name, k); exit(2); }
    printf("{\"fr\": \"%s\", \"count\": %u, \"n_public\": %u, \"batched_ms\": %.4f, \"per_input_ms\": %.4f}\n", name, count, np, best[0], best[1]);
    cudaFree(d_xi); cudaFree(d_zh); cudaFree(d_wpow); cudaFree(d_pub); cudaFree(d_term);
    for (int v = 0; v < 2; v++) { cudaFree(d_pi[v]); cudaFree(d_l1[v]); }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
}

int main(int argc, char** argv) {
    if (argc != 4) { fprintf(stderr, "usage: %s COUNT N_PUBLIC REPS\n", argv[0]); return 1; }
    const uint32_t count = (uint32_t)atoi(argv[1]), np = (uint32_t)atoi(argv[2]);
    const int reps = atoi(argv[3]);
    if (!count || !np) { fprintf(stderr, "COUNT and N_PUBLIC must be positive\n"); return 1; }
    run<BnFq>("bn254", count, np, reps);
    run<BlsFq>("bls12381", count, np, reps);
    return 0;
}
