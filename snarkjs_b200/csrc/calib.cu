// calib.cu — calibration micro-kernels for the integer-pipe roofline (SURVEY.md §8d): the measured rate of
// IMAD.WIDE.U32 (the instruction that carries >95% of the work) and of back-to-back register-resident
// Montgomery multiplies.  bench.py reports kernel throughput against these measured peaks.
#include <cuda_runtime.h>
#include "fp.cuh"
namespace sb {
__global__ void __launch_bounds__(256) k_calib_imad(uint64_t* out, int iters, uint32_t a, uint32_t b) {
    uint64_t acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = threadIdx.x + j;
    uint32_t x = a + threadIdx.x, y = b;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
#pragma unroll
            for (int j = 0; j < 8; j++) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[j]) : "r"((uint32_t)acc[(j + 3) & 7]), "r"(y));   // data dependent multiplicand: no strength reduction
        }
    }
    uint64_t s = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) s ^= acc[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void __launch_bounds__(256) k_calib_modmul(uint32_t* out, int iters) {
    typedef Fp<BnFq> F;
    F a = F::one(), b = F::r2(), c = F::one(), d = F::r2();
    a.v[0] += threadIdx.x; c.v[1] += blockIdx.x + 3 * threadIdx.x; b.v[2] ^= threadIdx.x; d.v[3] += 7 * threadIdx.x;   // every chain is per-thread (nothing for the uniform datapath)
    for (int it = 0; it < iters; it++) { a = F::mul(a, b); c = F::mul(c, d); b = F::mul(b, a); d = F::mul(d, c); }
    F r = F::add(F::add(a, b), F::add(c, d));
    out[blockIdx.x * blockDim.x + threadIdx.x] = r.v[0] ^ r.v[7];
}
// ---- FP64 exploration: the GPU has a full-rate FP64 pipe that the integer kernels leave idle.  A 52-bit
// limb product needs two DFMAs (high and low half, Emmart's fma_rz trick), one DADD and two 64-bit integer adds.
__global__ void __launch_bounds__(256) k_calib_dfma(double* out, int iters) {
    double acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 1.0 + threadIdx.x * 1e-3 + j;
    const double b = 1.0000001, cst = 0.5;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
#pragma unroll
            for (int j = 0; j < 8; j++) acc[j] = __fma_rz(acc[j], b, cst);
        }
    }
    double s = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) s += acc[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// one "52-bit limb product" = hi/lo split by two fma_rz + one add, both halves accumulated as 64-bit integers
__device__ __forceinline__ void limb_product(double a, double b, long long& sh, long long& sl) {
    const double c1 = 20282409603651670423947251286016.0;            // 2^104
    const double c2 = 20282409603651674927546878656512.0;            // 2^104 + 2^52
    double hi = __fma_rz(a, b, c1);
    double sub = c2 - hi;
    double lo = __fma_rz(a, b, sub);
    sh += __double_as_longlong(hi);
    sl += __double_as_longlong(lo);
}
// mode 0: every warp does limb products; mode 1: even warps limb products, odd warps Montgomery multiplies (co-issue test)
__global__ void __launch_bounds__(256) k_calib_limbprod(long long* out, int iters, int mode) {
    const int warp = threadIdx.x >> 5;
    if (mode == 1 && (warp & 1)) {
        typedef Fp<BnFq> F;
        F a = F::one(), b = F::r2(), c = F::one(), d = F::r2();
        a.v[0] += threadIdx.x; c.v[1] += blockIdx.x + 3 * threadIdx.x; b.v[2] ^= threadIdx.x; d.v[3] += 7 * threadIdx.x;
        for (int it = 0; it < iters / 4; it++) { a = F::mul(a, b); c = F::mul(c, d); b = F::mul(b, a); d = F::mul(d, c); }
        F r = F::add(F::add(a, b), F::add(c, d));
        out[blockIdx.x * blockDim.x + threadIdx.x] = r.v[0] ^ r.v[7];
        return;
    }
    double a[5], b[5];
#pragma unroll
    for (int j = 0; j < 5; j++) { a[j] = 4503599627370495.0 - threadIdx.x - j; b[j] = 4503599627370001.0 - 3 * threadIdx.x - 7 * j; }
    long long sh = 0, sl = 0;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 5; i++) {
#pragma unroll
            for (int j = 0; j < 5; j++) limb_product(a[i], b[j], sh, sl);
        }
        a[it % 5] -= 2.0;           // keep the compiler from hoisting the products
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = sh ^ sl;
}

// returns operations per second (what = 0: IMAD.WIDE.U32, 1: BN254 Fq Montgomery multiplies), <0 on error
double calibrate(int what, cudaStream_t stream) {
    int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int blocks = sms * 8, threads = 256;
    void* buf = nullptr; if (cudaMalloc(&buf, (size_t)blocks * threads * 8) != cudaSuccess) return -1;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = what == 0 ? 4096 : what == 1 ? 512 : what == 2 ? 4096 : 256;
    double best = 0;
    for (int rep = 0; rep < 4; rep++) {
        cudaEventRecord(e0, stream);
        if (what == 0) k_calib_imad<<<blocks, threads, 0, stream>>>((uint64_t*)buf, iters, 12345u + rep, 0x9e3779b9u);
        else if (what == 1) k_calib_modmul<<<blocks, threads, 0, stream>>>((uint32_t*)buf, iters);
        else if (what == 2) k_calib_dfma<<<blocks, threads, 0, stream>>>((double*)buf, iters);
        else k_calib_limbprod<<<blocks, threads, 0, stream>>>((long long*)buf, iters, what == 4 ? 1 : 0);
        cudaEventRecord(e1, stream);
        if (cudaEventSynchronize(e1) != cudaSuccess) { best = -1; break; }
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        // what: 0 IMAD.WIDE, 1 modmul, 2 DFMA, 3 limb products (all warps), 4 limb products counted on the even warps
        // while the odd warps run Montgomery multiplies (the returned rate is the limb products of the even warps only)
        double ops = (double)blocks * threads * iters * (what == 0 ? 64.0 : what == 1 ? 4.0 : what == 2 ? 64.0 : what == 3 ? 25.0 : 12.5);
        if (rep > 0 && ms > 0) best = ops / (ms * 1e-3) > best ? ops / (ms * 1e-3) : best;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(buf);
    return best;
}
}
