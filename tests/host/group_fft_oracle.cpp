// group_fft_oracle.cpp — CPU reference for the group FFT and group batchApplyKey (test infrastructure).
//
// Built on the CPU oracle's field and Jacobian-point restatement, which it includes unchanged; tests/gfft_oracle.py
// compiles this file into a temporary shared library and calls the two extern "C" functions below.
//
// Group FFT (buildFFT$3 _fft, build/snarkjs.js:14675-14918): radix-2 over natural-order points, every twiddle applied
// with timesFr (fromMontgomery + timesScalar, g?m_fftMix / g?m_fftJoin).  The inverse is the forward transform scaled by
// n^-1 with x[k] = X[(n-k) mod n] (g?m_fftFinal plus the reversed chunk order, 14896-14905).  Points are affine (2
// coordinates, all-zero = infinity) or Jacobian (3 coordinates, Z = 0 = infinity); Jacobian output is not normalised.
#include "../../oracle/snark_oracle.cpp"

template <class J> static J load_point(const uint8_t* in, int in_jac, u64 i) {
    J p;
    if (in_jac) { memcpy(&p, in + i * sizeof(J), sizeof(J)); return p; }
    typename J::Aff a; memcpy(&a, in + i * sizeof(a), sizeof(a));
    return J::from_affine(a);
}
template <class J> static void store_point(const J& p, int out_jac, uint8_t* out, u64 i) {
    if (out_jac) { memcpy(out + i * sizeof(J), &p, sizeof(J)); return; }
    typename J::Aff a = J::to_affine(p); memcpy(out + i * sizeof(a), &a, sizeof(a));
}
template <class GF, class T> static int group_fft(const uint8_t* in, int in_jac, u64 n, int inverse, int out_jac, uint8_t* out,
                                                  const Roots<T>& R) {
    typedef Jac<GF> J; typedef Fp<T> F;
    if (n == 0 || (n & (n - 1))) return -1;
    int bits = log2u(n);
    if (bits > R.s) return -2;
    std::vector<J> a(n);
    for (u64 i = 0; i < n; i++) a[bitrev(i, bits)] = load_point<J>(in, in_jac, i);
    for (int st = 1; st <= bits; st++) {
        u64 m = 1ull << st, mh = m >> 1;
        std::vector<F> tw(mh); F t = F::one();
        for (u64 j = 0; j < mh; j++) { tw[j] = F::from_mont(t); t = F::mul(t, R.w[st]); }
#pragma omp parallel for schedule(dynamic, 64)
        for (long long k = 0; k < (long long)(n / 2); k++) {
            u64 blk = (u64)k / mh, j = (u64)k % mh;
            u64 i0 = blk * m + j, i1 = i0 + mh;
            J x = J::times(a[i1], (const uint8_t*)tw[j].v, 32);
            J u = a[i0];
            a[i0] = J::add(u, x);
            a[i1] = J::add(u, J::neg(x));
        }
    }
    if (inverse) {
        F two = F::add(F::one(), F::one()), nn = F::one();
        for (int i = 0; i < bits; i++) nn = F::mul(nn, two);
        F ninv = F::from_mont(F::inv(nn));
#pragma omp parallel for schedule(dynamic, 64)
        for (long long i = 0; i < (long long)n; i++) a[i] = J::times(a[i], (const uint8_t*)ninv.v, 32);
        for (u64 i = 1; i < n / 2; i++) std::swap(a[i], a[n - i]);
    }
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)n; i++) store_point<J>(a[i], out_jac, out, (u64)i);
    return 0;
}

// G.batchApplyKey (14268-14385, g?m_batchApplyKey[Mixed]): out[i] = in[i] * first * inc^i, first / inc Montgomery Fr.
template <class GF, class T> static int group_batch_apply_key(const uint8_t* in, int in_jac, u64 n, const uint8_t* first,
                                                              const uint8_t* inc, int out_jac, uint8_t* out) {
    typedef Jac<GF> J; typedef Fp<T> F;
    std::vector<F> sc(n);
    F t, ic; memcpy(t.v, first, 32); memcpy(ic.v, inc, 32);
    for (u64 i = 0; i < n; i++) { sc[i] = F::from_mont(t); t = F::mul(t, ic); }
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < (long long)n; i++)
        store_point<J>(J::times(load_point<J>(in, in_jac, (u64)i), (const uint8_t*)sc[i].v, 32), out_jac, out, (u64)i);
    return 0;
}

extern "C" {

int gfo_group_fft(int curve, int group, const uint8_t* in, int in_jacobian, u64 n, int inverse, int out_jacobian, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        return curve == C_BN254 ? group_fft<GF, BnFr>(in, in_jacobian, n, inverse, out_jacobian, out, roots_bn)
                                : group_fft<GF, BlsFr>(in, in_jacobian, n, inverse, out_jacobian, out, roots_bls);
    })
}

int gfo_group_batch_apply_key(int curve, int group, const uint8_t* in, int in_jacobian, u64 n, const uint8_t* first,
                              const uint8_t* inc, int out_jacobian, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        return curve == C_BN254 ? group_batch_apply_key<GF, BnFr>(in, in_jacobian, n, first, inc, out_jacobian, out)
                                : group_batch_apply_key<GF, BlsFr>(in, in_jacobian, n, first, inc, out_jacobian, out);
    })
}

}  // extern "C"
