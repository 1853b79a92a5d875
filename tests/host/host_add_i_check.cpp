// Host-side check that XYZZ::add_i (the full addition of the device reduction kernels, ec.cuh) returns the same bytes as
// XYZZ::add on all four groups: random sums, q = infinity, acc = infinity, P + P and P + (-P) with q in another
// projective representative.  The formulas are checked on arbitrary field elements: add and add_i evaluate the same
// expressions whether or not the inputs lie on the curve.  Built and run by tests/test_host_add_i.py.
#include <cstdio>
#include <cstring>
#include "../../snarkjs_b200/csrc/ec.cuh"
using namespace sb;

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

// uniform-ish canonical element: random limbs below 2^bitlen(p) (< 2p), then one conditional subtraction
template <class P> static void rand_fe(Fp<P>& a) {
    constexpr int N = P::N;
    int top = 0; for (uint32_t t = P::p(N - 1); t; t >>= 1) top++;
    for (int i = 0; i < N; i++) a.v[i] = (uint32_t)rnd();
    a.v[N - 1] &= (1u << top) - 1;
    a = Fp<P>::add(a, Fp<P>::zero());
}
template <class P> static void rand_fe(Fp2<P>& a) { rand_fe(a.a); rand_fe(a.b); }

template <class F> static XYZZ<F> rand_pt() { XYZZ<F> p; rand_fe(p.x); rand_fe(p.y); rand_fe(p.zz); rand_fe(p.zzz); return p; }
// the same point as p in another representative: (l^2 x, l^3 y, l^2 zz, l^3 zzz)
template <class F> static XYZZ<F> rescale(const XYZZ<F>& p) {
    F l; rand_fe(l);
    const F l2 = F::mul(l, l), l3 = F::mul(l2, l);
    XYZZ<F> r; r.x = F::mul(p.x, l2); r.y = F::mul(p.y, l3); r.zz = F::mul(p.zz, l2); r.zzz = F::mul(p.zzz, l3);
    return r;
}
template <class F> static bool same(const XYZZ<F>& a, const XYZZ<F>& b) { return memcmp(&a, &b, sizeof a) == 0; }

template <class F> static int check_group(const char* name) {
    int bad = 0;
    auto cmp = [&](const XYZZ<F>& acc, const XYZZ<F>& q, const char* what, int it) {
        XYZZ<F> a = acc, b = acc;
        a.add(q); b.add_i(q);
        if (!same(a, b)) { bad++; if (bad < 4) printf("%s add_i != add (%s, it=%d)\n", name, what, it); }
        return b;
    };
    for (int it = 0; it < 2000; it++) {
        const XYZZ<F> p = rand_pt<F>(), q = rand_pt<F>();
        cmp(p, q, "random", it);
        cmp(p, XYZZ<F>::inf(), "q = inf", it);
        XYZZ<F> qi = q; qi.zz = F::zero();            // infinity is zz == 0, whatever the other coordinates hold
        cmp(p, qi, "q = inf, nonzero x/y/zzz", it);
        if (!same(cmp(XYZZ<F>::inf(), q, "acc = inf", it), q)) { bad++; if (bad < 4) printf("%s inf + q != q (it=%d)\n", name, it); }
        const XYZZ<F> r = rescale(p);
        const XYZZ<F> d = cmp(p, r, "P + P", it), d2 = XYZZ<F>::dbl(p);
        if (!same(d, d2)) { bad++; if (bad < 4) printf("%s P + P != dbl(P) (it=%d)\n", name, it); }
        XYZZ<F> n = r; n.y = F::neg(n.y);
        if (!cmp(p, n, "P + (-P)", it).is_inf()) { bad++; if (bad < 4) printf("%s P + (-P) != inf (it=%d)\n", name, it); }
        if (it < 50) {   // a running sum, as the fold and axis-sum kernels form it
            XYZZ<F> a = XYZZ<F>::inf(), b = XYZZ<F>::inf();
            for (int k = 0; k < 16; k++) { const XYZZ<F> t = rand_pt<F>(); a.add(t); b.add_i(t); }
            if (!same(a, b)) { bad++; if (bad < 4) printf("%s running sum differs (it=%d)\n", name, it); }
        }
    }
    printf("%s: %s\n", name, bad ? "FAIL" : "ok");
    return bad;
}

int main() {
    int bad = 0;
    bad += check_group<Fp<BnFq>>("BN254 G1");
    bad += check_group<Fp2<BnFq>>("BN254 G2");
    bad += check_group<Fp<BlsFq>>("BLS12-381 G1");
    bad += check_group<Fp2<BlsFq>>("BLS12-381 G2");
    printf(bad ? "ADD_I CHECK FAILED\n" : "ADD_I CHECK PASSED\n");
    return bad ? 1 : 0;
}
