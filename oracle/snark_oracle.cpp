// ============================================================================
// oracle/snark_oracle.cpp — CPU restatement of the snarkjs hot path.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
// (snarkjs_b200/csrc) never links or calls anything in oracle/.
//
// The reference (iden3/snarkjs 0.7.6) has no native code: its arithmetic lives in the
// npm dependencies ffjavascript@0.3.1 -> wasmcurves@0.2.2 (WASM generated at run time),
// absent from node_modules but bundled verbatim into snarkjs' build/snarkjs.js.
// Each function below cites the bundle lines (first copy, 1-17660) it restates.
// There is no JS/WASM runtime in the build container, so the reference cannot be run
// here; parity is pinned instead against the reference-produced bytes embedded in the
// committed fixtures (tests/golden/, see tests/golden/make_golden.py):
//   * Fr NTT  : PLONK/fflonk zkey [coef n | evals 4n] blocks (32/1024/8192-pt),
//   * G1 MSM  : PLONK header commitments Qm..S3 and fflonk C0 (8/2048-pt),
//   * G1/G2 MSM: powersOfTau15_final.ptau Lagrange sections 12/13 vs sections 2/3.
//
// Build: g++ -O3 -march=native -fopenmp -shared -fPIC (oracle/Makefile).
// ============================================================================
#include <cstdint>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <algorithm>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint32_t u32;
typedef uint64_t u64;

// ---------------------------------------------------------------------------
// Field parameters.  n32-limb little-endian integers, Montgomery R = 2^(32*n32)
// (build/snarkjs.js:2873-2874).  np32 = -p^-1 mod 2^32 (build/snarkjs.js:3092).
// ---------------------------------------------------------------------------
template <int N> struct FParams {
    u32 p[N];
    u32 np32;
    u32 one[N];   // R mod p
    u32 r2[N];    // R^2 mod p
};

template <int N> static inline int int_gte(const u32* a, const u32* b) {
    for (int i = N - 1; i >= 0; i--) {
        if (a[i] > b[i]) return 1;
        if (a[i] < b[i]) return 0;
    }
    return 1;
}
template <int N> static inline u32 int_add(const u32* a, const u32* b, u32* r) {
    u64 c = 0;
    for (int i = 0; i < N; i++) { c += (u64)a[i] + b[i]; r[i] = (u32)c; c >>= 32; }
    return (u32)c;
}
template <int N> static inline u32 int_sub(const u32* a, const u32* b, u32* r) {
    u64 bw = 0;
    for (int i = 0; i < N; i++) {
        u64 t = (u64)a[i] - b[i] - bw;
        r[i] = (u32)t; bw = (t >> 32) & 1;
    }
    return (u32)bw;
}
template <int N> static inline int int_is_zero(const u32* a) {
    u32 o = 0; for (int i = 0; i < N; i++) o |= a[i]; return o == 0;
}

// Tag structs: one static parameter block per field.
struct BnFq  { static const int N = 8;  static FParams<8>  P; };
struct BnFr  { static const int N = 8;  static FParams<8>  P; };
struct BlsFq { static const int N = 12; static FParams<12> P; };
struct BlsFr { static const int N = 8;  static FParams<8>  P; };
FParams<8> BnFq::P; FParams<8> BnFr::P; FParams<12> BlsFq::P; FParams<8> BlsFr::P;

// ---------------------------------------------------------------------------
// Fp<T>: prime field element in Montgomery form, always fully reduced to [0,p).
// ---------------------------------------------------------------------------
template <class T> struct Fp {
    static const int N = T::N;
    u32 v[T::N];

    static Fp zero() { Fp r; memset(r.v, 0, sizeof r.v); return r; }
    static Fp one()  { Fp r; memcpy(r.v, T::P.one, sizeof r.v); return r; }
    bool is_zero() const { return int_is_zero<N>(v); }
    bool operator==(const Fp& o) const { return memcmp(v, o.v, sizeof v) == 0; }
    bool is_one() const { return memcmp(v, T::P.one, sizeof v) == 0; }

    // f1m_add  build/snarkjs.js:2902-2920  (add, subtract p on carry or >= p)
    static Fp add(const Fp& a, const Fp& b) {
        Fp r; u32 c = int_add<N>(a.v, b.v, r.v);
        if (c || int_gte<N>(r.v, T::P.p)) int_sub<N>(r.v, T::P.p, r.v);
        return r;
    }
    // f1m_sub  build/snarkjs.js:2922-2936  (subtract, add p back on borrow)
    static Fp sub(const Fp& a, const Fp& b) {
        Fp r; u32 bw = int_sub<N>(a.v, b.v, r.v);
        if (bw) int_add<N>(r.v, T::P.p, r.v);
        return r;
    }
    static Fp neg(const Fp& a) {
        if (a.is_zero()) return a;
        Fp r; int_sub<N>(T::P.p, a.v, r.v); return r;
    }
    // f1m_mul  build/snarkjs.js:3072-3273 — product-scanning Montgomery multiply over
    // 32-bit limbs with two 64-bit column accumulators (c0 = low-word sums, c1 = carries),
    // m[k] = (column * np32) mod 2^32, final conditional subtract => canonical result.
    static Fp mul(const Fp& x, const Fp& y) {
        const u32* q = T::P.p; const u64 np32 = T::P.np32;
        u64 m[N]; u64 c0 = 0, c1 = 0; Fp r;
        for (int k = 0; k < 2 * N - 1; k++) {
            int ilo = std::max(0, k - N + 1);
            for (int i = ilo; i <= k && i < N; i++) {
                c0 = (c0 & 0xFFFFFFFFull) + (u64)x.v[i] * y.v[k - i];
                c1 += c0 >> 32;
            }
            for (int i = std::max(1, k - N + 1); i <= k && i < N; i++) {
                c0 = (c0 & 0xFFFFFFFFull) + (u64)q[i] * m[k - i];
                c1 += c0 >> 32;
            }
            if (k < N) {
                m[k] = ((c0 & 0xFFFFFFFFull) * np32) & 0xFFFFFFFFull;
                c0 = (c0 & 0xFFFFFFFFull) + (u64)q[0] * m[k];
                c1 += c0 >> 32;
            } else {
                r.v[k - N] = (u32)c0;
            }
            c0 = c1; c1 = c0 >> 32;   // [c0,c1] = [c1,c0]; c1 = c0 >> 32
        }
        r.v[N - 1] = (u32)c0;
        if ((u32)c1) int_sub<N>(r.v, q, r.v);
        else if (int_gte<N>(r.v, q)) int_sub<N>(r.v, q, r.v);
        return r;
    }
    static Fp sqr(const Fp& a) { return mul(a, a); }   // f1m_square 3276 (same result)
    // f1m_toMontgomery 3586: x * R^2 ; f1m_fromMontgomery 3595: x * 1
    static Fp to_mont(const Fp& a) { Fp r2; memcpy(r2.v, T::P.r2, sizeof r2.v); return mul(a, r2); }
    static Fp from_mont(const Fp& a) { Fp o = zero(); o.v[0] = 1; return mul(a, o); }
    // exponentiation by a plain little-endian integer (WasmField1.exp)
    static Fp pow(const Fp& b, const u32* e, int nw) {
        Fp r = one();
        for (int i = nw * 32 - 1; i >= 0; i--) {
            r = sqr(r);
            if ((e[i >> 5] >> (i & 31)) & 1) r = mul(r, b);
        }
        return r;
    }
    // f1m_inverse 3609 (reference: fromMontgomery, int inverseMod, toMontgomery);
    // restated with Fermat: a^(p-2).  Same canonical value.
    static Fp inv(const Fp& a) {
        u32 e[N]; u32 two[N]; memset(two, 0, sizeof two); two[0] = 2;
        int_sub<N>(T::P.p, two, e);
        return pow(a, e, N);
    }
    static Fp dbl(const Fp& a) { return add(a, a); }
};

// Parameter derivation from the modulus alone.
template <class T> static void init_field(const char* hex_be) {
    const int N = T::N;
    u32* p = T::P.p; memset(p, 0, 4 * N);
    int len = (int)strlen(hex_be);
    for (int i = 0; i < len; i++) {
        char ch = hex_be[len - 1 - i];
        u32 d = (ch >= '0' && ch <= '9') ? ch - '0' : (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : ch - 'A' + 10;
        p[i / 8] |= d << (4 * (i % 8));
    }
    // np32 = -p^-1 mod 2^32 (Newton on the low word)
    u32 inv = 1; for (int i = 0; i < 6; i++) inv *= 2 - p[0] * inv;
    T::P.np32 = (u32)(0u - inv);
    // R mod p, R^2 mod p by repeated modular doubling of 1
    u32 t[N]; memset(t, 0, sizeof t); t[0] = 1;
    for (int i = 0; i < 64 * N; i++) {
        u32 c = int_add<N>(t, t, t);
        if (c || int_gte<N>(t, p)) int_sub<N>(t, p, t);
        if (i == 32 * N - 1) memcpy(T::P.one, t, sizeof t);
    }
    memcpy(T::P.r2, t, sizeof t);
}

// ---------------------------------------------------------------------------
// Fp2<T> = Fp[u]/(u^2+1)   (build_f2m, build/snarkjs.js:4028; mul 4157; square 4216)
// byte order c0 || c1.
// ---------------------------------------------------------------------------
template <class T> struct Fp2 {
    typedef Fp<T> B;
    B a, b;   // a + b u
    static Fp2 zero() { Fp2 r; r.a = B::zero(); r.b = B::zero(); return r; }
    static Fp2 one()  { Fp2 r; r.a = B::one();  r.b = B::zero(); return r; }
    bool is_zero() const { return a.is_zero() && b.is_zero(); }
    bool is_one() const { return a.is_one() && b.is_zero(); }
    bool operator==(const Fp2& o) const { return a == o.a && b == o.b; }
    static Fp2 add(const Fp2& x, const Fp2& y) { Fp2 r; r.a = B::add(x.a, y.a); r.b = B::add(x.b, y.b); return r; }
    static Fp2 sub(const Fp2& x, const Fp2& y) { Fp2 r; r.a = B::sub(x.a, y.a); r.b = B::sub(x.b, y.b); return r; }
    static Fp2 neg(const Fp2& x) { Fp2 r; r.a = B::neg(x.a); r.b = B::neg(x.b); return r; }
    static Fp2 dbl(const Fp2& x) { return add(x, x); }
    // f2m_mul 4157: A=x0*y0, B=x1*y1, C=(x0+x1)(y0+y1); r0 = A + nr*B (nr=-1), r1 = C-A-B
    static Fp2 mul(const Fp2& x, const Fp2& y) {
        B A = B::mul(x.a, y.a), Bb = B::mul(x.b, y.b);
        B C = B::mul(B::add(x.a, x.b), B::add(y.a, y.b));
        Fp2 r; r.a = B::sub(A, Bb); r.b = B::sub(B::sub(C, A), Bb); return r;
    }
    // f2m_square 4216: AB = x0*x1; r0 = (x0+x1)(x0 + nr*x1) - AB - nr*AB ; r1 = 2AB
    static Fp2 sqr(const Fp2& x) {
        B AB = B::mul(x.a, x.b);
        Fp2 r; r.a = B::mul(B::add(x.a, x.b), B::sub(x.a, x.b)); r.b = B::add(AB, AB); return r;
    }
    // f2m_inverse: (a - bu)/(a^2 + b^2)
    static Fp2 inv(const Fp2& x) {
        B t = B::inv(B::add(B::sqr(x.a), B::sqr(x.b)));
        Fp2 r; r.a = B::mul(x.a, t); r.b = B::neg(B::mul(x.b, t)); return r;
    }
};

// ---------------------------------------------------------------------------
// Short-Weierstrass a=0 curve in Jacobian coordinates over F
// (build_curve_jacobian_a0, build/snarkjs.js:5944-7430).
// zero <=> Z == 0; affine zero = (0,0).
// ---------------------------------------------------------------------------
template <class F> struct Jac {
    F x, y, z;
    struct Aff { F x, y; bool is_zero() const { return x.is_zero() && y.is_zero(); } };

    static Jac zero() { Jac r; r.x = F::zero(); r.y = F::one(); r.z = F::zero(); return r; }   // 6039-6065
    bool is_zero() const { return z.is_zero(); }
    static Jac from_affine(const Aff& a) {
        if (a.is_zero()) return zero();
        Jac r; r.x = a.x; r.y = a.y; r.z = F::one(); return r;
    }
    // _double 6206-6274 (dbl-2009-l); the Z==1 shortcut (_doubleAffine) gives the same point.
    static Jac dbl(const Jac& p) {
        if (p.is_zero()) return p;
        F A = F::sqr(p.x), B = F::sqr(p.y), C = F::sqr(B);
        F D = F::sqr(F::add(p.x, B)); D = F::sub(D, A); D = F::sub(D, C); D = F::add(D, D);
        F E = F::add(F::add(A, A), A);
        F Ff = F::sqr(E);
        F G = F::mul(p.y, p.z);
        Jac r;
        r.x = F::sub(Ff, F::add(D, D));
        F eightC = F::add(C, C); eightC = F::add(eightC, eightC); eightC = F::add(eightC, eightC);
        r.y = F::sub(F::mul(F::sub(D, r.x), E), eightC);
        r.z = F::add(G, G);
        return r;
    }
    // _add 6456 (add-2007-bl) with the reference's special cases (zero operands, equal => double)
    static Jac add(const Jac& p, const Jac& q) {
        if (p.is_zero()) return q;
        if (q.is_zero()) return p;
        F Z1Z1 = F::sqr(p.z), Z2Z2 = F::sqr(q.z);
        F U1 = F::mul(p.x, Z2Z2), U2 = F::mul(q.x, Z1Z1);
        F S1 = F::mul(F::mul(p.y, q.z), Z2Z2), S2 = F::mul(F::mul(q.y, p.z), Z1Z1);
        if (U1 == U2 && S1 == S2) return dbl(p);
        F H = F::sub(U2, U1);
        F S2mS1 = F::sub(S2, S1);
        F I = F::sqr(F::add(H, H));
        F J = F::mul(H, I);
        F rr = F::add(S2mS1, S2mS1);
        F V = F::mul(U1, I);
        Jac r;
        r.x = F::sub(F::sub(F::sqr(rr), J), F::add(V, V));
        F S1J = F::mul(S1, J);
        r.y = F::sub(F::mul(rr, F::sub(V, r.x)), F::add(S1J, S1J));
        r.z = F::mul(F::sub(F::sub(F::sqr(F::add(p.z, q.z)), Z1Z1), Z2Z2), H);
        return r;
    }
    // _addMixed 6576-6678 (madd-2007-bl)
    static Jac add_mixed(const Jac& p, const Aff& q) {
        if (p.is_zero()) return from_affine(q);
        if (q.is_zero()) return p;
        F Z1Z1 = F::sqr(p.z);
        F U2 = F::mul(q.x, Z1Z1);
        F S2 = F::mul(F::mul(q.y, p.z), Z1Z1);
        if (p.x == U2 && p.y == S2) return dbl(p);
        F H = F::sub(U2, p.x);
        F S2mS1 = F::sub(S2, p.y);
        F HH = F::sqr(H);
        F I = F::add(HH, HH); I = F::add(I, I);
        F J = F::mul(H, I);
        F rr = F::add(S2mS1, S2mS1);
        F V = F::mul(p.x, I);
        Jac r;
        r.x = F::sub(F::sub(F::sqr(rr), J), F::add(V, V));
        F Y1J = F::mul(p.y, J);
        r.y = F::sub(F::mul(rr, F::sub(V, r.x)), F::add(Y1J, Y1J));
        r.z = F::sub(F::sub(F::sqr(F::add(p.z, H)), Z1Z1), HH);
        return r;
    }
    static Jac neg(const Jac& p) { Jac r = p; r.y = F::neg(p.y); return r; }
    // _toAffine 6892: zero -> (0,0) else (X/Z^2, Y/Z^3)
    static Aff to_affine(const Jac& p) {
        Aff a;
        if (p.is_zero()) { a.x = F::zero(); a.y = F::zero(); return a; }
        F zi = F::inv(p.z), zi2 = F::sqr(zi);
        a.x = F::mul(p.x, zi2); a.y = F::mul(p.y, F::mul(zi2, zi));
        return a;
    }
    // _timesScalar 5232 (reference uses NAF; plain double-and-add gives the same group element)
    static Jac times(const Jac& p, const uint8_t* s, int nbytes) {
        Jac r = zero();
        for (int i = nbytes * 8 - 1; i >= 0; i--) {
            r = dbl(r);
            if ((s[i >> 3] >> (i & 7)) & 1) r = add(r, p);
        }
        return r;
    }
};

// ---------------------------------------------------------------------------
// Pippenger multiexp (build_multiexp, build/snarkjs.js:5466-5918 + driver 14517-14669)
// ---------------------------------------------------------------------------
static const int pTSizes[32] = {   // 14517-14522
    1, 1, 1, 1, 2, 3, 4, 5, 6, 7, 7, 8, 9, 10, 11, 12,
    13, 13, 14, 15, 16, 16, 17, 17, 17, 17, 17, 17, 17, 17, 17, 17};

static inline int log2u(u64 v) { int r = 0; while (v >>= 1) r++; return r; }   // src/misc.js:53

// _getChunk 5471-5540: bits [startBit, startBit+chunkSize) of a little-endian scalar
static inline u32 get_chunk(const uint8_t* s, int scalarSize, int startBit, int chunkSize) {
    u32 v = 0;
    for (int b = 0; b < chunkSize; b++) {
        int bit = startBit + b;
        if ((bit >> 3) >= scalarSize) break;
        v |= (u32)((s[bit >> 3] >> (bit & 7)) & 1) << b;
    }
    return v;
}

// _reduceTable 5819-5907 (recursive halving); table[idx-1] holds bucket idx.
template <class F> static void reduce_table(Jac<F>* t, int p) {
    if (p == 1) return;
    int half = 1 << (p - 1);
    Jac<F>* acc = t + half - 1;
    for (int i = 0; i < half - 1; i++) {
        t[i] = Jac<F>::add(t[i], t[half + i]);
        *acc = Jac<F>::add(*acc, t[half + i]);
    }
    reduce_table<F>(t, p - 1);
    for (int i = 0; i < p - 1; i++) *acc = Jac<F>::dbl(*acc);
    t[0] = Jac<F>::add(t[0], *acc);
}

// g?m_multiexpAffine_chunk 5542-5695: one window of one point-chunk.
template <class F> static Jac<F> multiexp_window(const typename Jac<F>::Aff* bases, const uint8_t* scalars,
                                                 int sScalar, u64 n, int startBit, int chunkSize) {
    if (n == 0) return Jac<F>::zero();
    int nTable = 1 << chunkSize;
    std::vector<Jac<F>> table(nTable, Jac<F>::zero());
    for (u64 i = 0; i < n; i++) {
        u32 idx = get_chunk(scalars + i * sScalar, sScalar, startBit, chunkSize);
        if (idx) table[idx - 1] = Jac<F>::add_mixed(table[idx - 1], bases[i]);
    }
    reduce_table<F>(table.data(), chunkSize);
    return table[0];
}

// _multiExpChunk 14527-14603 + _multiExp 14605-14661.  `concurrency` plays tm.concurrency.
template <class F> static Jac<F> multiexp_affine(const typename Jac<F>::Aff* bases, const uint8_t* scalars,
                                                 int sScalar, u64 nPoints, int concurrency) {
    if (nPoints == 0) return Jac<F>::zero();
    const u64 MAX_CHUNK = 1ull << 22, MIN_CHUNK = 1ull << 10;
    int bitChunk0 = pTSizes[log2u(nPoints)];
    int nChunks0 = (sScalar * 8 - 1) / bitChunk0 + 1;
    u64 chunkSize = (u64)((double)nPoints / ((double)concurrency / nChunks0));
    if (chunkSize > MAX_CHUNK) chunkSize = MAX_CHUNK;
    if (chunkSize < MIN_CHUNK) chunkSize = MIN_CHUNK;
    struct Task { u64 off, n; int w, bits, start; };
    std::vector<Task> tasks; std::vector<u64> chunk_first;
    std::vector<int> chunk_bits;
    for (u64 i = 0; i < nPoints; i += chunkSize) {
        u64 n = std::min(nPoints - i, chunkSize);
        int bc = pTSizes[log2u(n)];
        int nW = (sScalar * 8 - 1) / bc + 1;
        chunk_first.push_back(tasks.size()); chunk_bits.push_back(bc);
        for (int w = 0; w < nW; w++)
            tasks.push_back({i, n, w, std::min(sScalar * 8 - w * bc, bc), w * bc});
    }
    chunk_first.push_back(tasks.size());
    std::vector<Jac<F>> res(tasks.size());
#pragma omp parallel for schedule(dynamic, 1)
    for (long t = 0; t < (long)tasks.size(); t++) {
        const Task& k = tasks[t];
        res[t] = multiexp_window<F>(bases + k.off, scalars + k.off * sScalar, sScalar, k.n, k.start, k.bits);
    }
    Jac<F> total = Jac<F>::zero();
    for (int c = (int)chunk_bits.size() - 1; c >= 0; c--) {
        Jac<F> r = Jac<F>::zero();
        for (long t = (long)chunk_first[c + 1] - 1; t >= (long)chunk_first[c]; t--) {   // 14594-14600
            if (!r.is_zero()) for (int j = 0; j < chunk_bits[c]; j++) r = Jac<F>::dbl(r);
            r = Jac<F>::add(r, res[t]);
        }
        total = Jac<F>::add(total, r);   // 14655-14658
    }
    return total;
}

// ---------------------------------------------------------------------------
// Fr NTT (build_fft 7455-8798, driver _fft 14675-14918).  Radix-2 DIT: bit-reverse
// (buffReverseBits 12640-12654), log2 n butterfly stages (fftMix 8546-8666 /
// fftJoin 8089-8179 have the same butterfly: (u,v) -> (u + w v, u - w v), twiddle by
// running product), inverse = forward, then x[k] = X[(n-k) mod n] / n (fftFinal 8670-8772
// + reversed chunk order 14896-14905).
// Roots: nqr = first non-residue from 2; w[s] = nqr^((r-1)/2^s); w[i] = w[i+1]^2
// (12866-12889 / 7472-7495).
// ---------------------------------------------------------------------------
template <class T> struct Roots {
    int s; Fp<T> nqr, shift, w[64];
    void init() {
        typedef Fp<T> F; const int N = T::N;
        u32 one_i[N]; memset(one_i, 0, sizeof one_i); one_i[0] = 1;
        u32 pm1[N]; int_sub<N>(T::P.p, one_i, pm1);
        u32 half[N]; for (int i = 0; i < N; i++) half[i] = (pm1[i] >> 1) | (i + 1 < N ? pm1[i + 1] << 31 : 0);
        F negone = F::neg(F::one());
        F two = F::add(F::one(), F::one());
        nqr = two;
        while (!(F::pow(nqr, half, N) == negone)) nqr = F::add(nqr, F::one());
        shift = F::sqr(nqr);
        s = 0; u32 t[N]; memcpy(t, pm1, sizeof t);
        while (!(t[0] & 1)) { for (int i = 0; i < N; i++) t[i] = (t[i] >> 1) | (i + 1 < N ? t[i + 1] << 31 : 0); s++; }
        w[s] = F::pow(nqr, t, N);
        for (int i = s - 1; i >= 0; i--) w[i] = F::sqr(w[i + 1]);
    }
};
static Roots<BnFr> roots_bn; static Roots<BlsFr> roots_bls;

static inline u64 bitrev(u64 x, int bits) {
    u64 r = 0; for (int i = 0; i < bits; i++) { r = (r << 1) | (x & 1); x >>= 1; } return r;
}

template <class T> static int fft_inplace(Fp<T>* a, u64 n, int inverse, const Roots<T>& R) {
    typedef Fp<T> F;
    if (n == 0 || (n & (n - 1))) return -1;
    int bits = log2u(n);
    if (bits > R.s) return -2;
    for (u64 i = 0; i < n; i++) { u64 j = bitrev(i, bits); if (j > i) std::swap(a[i], a[j]); }
    for (int st = 1; st <= bits; st++) {
        u64 m = 1ull << st, mh = m >> 1;
        F wm = R.w[st];
        // per-stage twiddle table by running product (fftMix 8592-8661)
        std::vector<F> tw(mh); tw[0] = F::one();
        for (u64 j = 1; j < mh; j++) tw[j] = F::mul(tw[j - 1], wm);
#pragma omp parallel for schedule(static)
        for (long long k = 0; k < (long long)(n / 2); k++) {
            u64 blk = (u64)k / mh, j = (u64)k % mh;
            u64 i0 = blk * m + j, i1 = i0 + mh;
            F t = F::mul(tw[j], a[i1]);
            F u = a[i0];
            a[i0] = F::add(u, t);
            a[i1] = F::sub(u, t);
        }
    }
    if (inverse) {
        // n^-1 in Montgomery form
        F ninv = F::one(); F two = F::add(F::one(), F::one());
        F nn = F::one(); for (int i = 0; i < bits; i++) nn = F::mul(nn, two);
        ninv = F::inv(nn);
#pragma omp parallel for schedule(static)
        for (long long i = 0; i < (long long)n; i++) a[i] = F::mul(a[i], ninv);
        for (u64 i = 1; i < n / 2; i++) std::swap(a[i], a[n - i]);
    }
    return 0;
}

// ---------------------------------------------------------------------------
// extern "C" surface used by oracle/oracle.py (ctypes)
// ---------------------------------------------------------------------------
static bool g_init = false;
static void ensure_init() {
    if (g_init) return;
    init_field<BnFq>("30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47");
    init_field<BnFr>("30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001");
    init_field<BlsFq>("1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab");
    init_field<BlsFr>("73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001");
    roots_bn.init(); roots_bls.init();
    g_init = true;
}

enum { F_BN_FQ = 0, F_BN_FR = 1, F_BLS_FQ = 2, F_BLS_FR = 3 };
enum { C_BN254 = 0, C_BLS12_381 = 1 };

#define FIELD_DISPATCH(fid, ...)              \
    switch (fid) {                             \
    case F_BN_FQ:  { typedef BnFq  TT; __VA_ARGS__; } break; \
    case F_BN_FR:  { typedef BnFr  TT; __VA_ARGS__; } break; \
    case F_BLS_FQ: { typedef BlsFq TT; __VA_ARGS__; } break; \
    case F_BLS_FR: { typedef BlsFr TT; __VA_ARGS__; } break; \
    default: return -1; }

extern "C" {

int or_init() { ensure_init(); return 0; }
int or_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
void or_set_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int or_field_n8(int fid) { return (fid == F_BLS_FQ) ? 48 : 32; }

// op: 0 add, 1 sub, 2 mul, 3 neg(a), 4 inv(a), 5 toMont(a), 6 fromMont(a), 7 sqr(a)
int or_field_op(int fid, int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    ensure_init();
    FIELD_DISPATCH(fid, {
        typedef Fp<TT> F; F x, y, r; memcpy(x.v, a, sizeof x.v); if (b) memcpy(y.v, b, sizeof y.v);
        switch (op) {
        case 0: r = F::add(x, y); break;  case 1: r = F::sub(x, y); break;
        case 2: r = F::mul(x, y); break;  case 3: r = F::neg(x); break;
        case 4: r = F::inv(x); break;     case 5: r = F::to_mont(x); break;
        case 6: r = F::from_mont(x); break; case 7: r = F::sqr(x); break;
        default: return -1; }
        memcpy(out, r.v, sizeof r.v);
    })
    return 0;
}

// constants: what 0 = p, 1 = one (R mod p), 2 = R^2 mod p
int or_field_const(int fid, int what, uint8_t* out) {
    ensure_init();
    FIELD_DISPATCH(fid, {
        const u32* s = what == 0 ? TT::P.p : what == 1 ? TT::P.one : TT::P.r2;
        memcpy(out, s, 4 * TT::N);
    })
    return 0;
}

// Fr roots: idx = -1 -> shift (nqr^2), -2 -> nqr, else w[idx]; returns s
int or_fr_root(int curve, int idx, uint8_t* out) {
    ensure_init();
    if (curve == C_BN254) {
        const Fp<BnFr>& r = idx == -1 ? roots_bn.shift : idx == -2 ? roots_bn.nqr : roots_bn.w[idx];
        memcpy(out, r.v, 32); return roots_bn.s;
    } else {
        const Fp<BlsFr>& r = idx == -1 ? roots_bls.shift : idx == -2 ? roots_bls.nqr : roots_bls.w[idx];
        memcpy(out, r.v, 32); return roots_bls.s;
    }
}

// frm_batchToMontgomery / frm_batchFromMontgomery (engine_batchconvert 12780-12830)
int or_batch_convert(int fid, int to_mont, const uint8_t* in, u64 n, uint8_t* out) {
    ensure_init();
    FIELD_DISPATCH(fid, {
        typedef Fp<TT> F; const F* a = (const F*)in; F* o = (F*)out;
        _Pragma("omp parallel for schedule(static)")
        for (long long i = 0; i < (long long)n; i++) o[i] = to_mont ? F::to_mont(a[i]) : F::from_mont(a[i]);
    })
    return 0;
}

// Fr.fft / Fr.ifft (15101-15107): out-of-place, natural order in and out
int or_fr_fft(int curve, const uint8_t* in, u64 n, int inverse, uint8_t* out) {
    ensure_init();
    if (out != in) memcpy(out, in, n * 32);
    if (curve == C_BN254) return fft_inplace<BnFr>((Fp<BnFr>*)out, n, inverse, roots_bn);
    return fft_inplace<BlsFr>((Fp<BlsFr>*)out, n, inverse, roots_bls);
}

// frm_batchApplyKey 9315-9379: t = first; out[i] = in[i]*t; t *= inc
// (driver 14268-14385 splits by chunks with first*inc^offset — same values)
int or_fr_batch_apply_key(int curve, const uint8_t* in, u64 n, const uint8_t* first, const uint8_t* inc, uint8_t* out) {
    ensure_init();
    int fid = curve == C_BN254 ? F_BN_FR : F_BLS_FR;
    FIELD_DISPATCH(fid, {
        typedef Fp<TT> F; const F* a = (const F*)in; F* o = (F*)out;
        F t, ic; memcpy(t.v, first, 32); memcpy(ic.v, inc, 32);
        for (u64 i = 0; i < n; i++) { o[i] = F::mul(a[i], t); t = F::mul(t, ic); }
    })
    return 0;
}

// qap_joinABC 9174-9233 (out = a*b - c) followed by frm_batchFromMontgomery
// (src/groth16_prove.js:320-374)
int or_qap_join_abc(int curve, const uint8_t* a, const uint8_t* b, const uint8_t* c, u64 n, uint8_t* out) {
    ensure_init();
    int fid = curve == C_BN254 ? F_BN_FR : F_BLS_FR;
    FIELD_DISPATCH(fid, {
        typedef Fp<TT> F; const F* A = (const F*)a; const F* B = (const F*)b; const F* C = (const F*)c; F* o = (F*)out;
        _Pragma("omp parallel for schedule(static)")
        for (long long i = 0; i < (long long)n; i++) o[i] = F::from_mont(F::sub(F::mul(A[i], B[i]), C[i]));
    })
    return 0;
}

// buildABC1 src/groth16_prove.js:147-187.  coeffs = zkey section 4 payload after the u32 count:
// nCoef x (u32 m, u32 c, u32 s, FE coef*R^2); witness plain LE.  Outputs Montgomery, domainSize each.
int or_build_abc(int curve, const uint8_t* coeffs, u64 nCoef, const uint8_t* witness, u64 nWitness, u64 domainSize,
                 uint8_t* outA, uint8_t* outB, uint8_t* outC) {
    ensure_init();
    int fid = curve == C_BN254 ? F_BN_FR : F_BLS_FR;
    FIELD_DISPATCH(fid, {
        typedef Fp<TT> F; F* A = (F*)outA; F* B = (F*)outB; F* C = (F*)outC; const F* W = (const F*)witness;
        for (u64 i = 0; i < domainSize; i++) { A[i] = F::zero(); B[i] = F::zero(); }
        const int sCoef = 12 + 32;
        for (u64 i = 0; i < nCoef; i++) {
            const uint8_t* e = coeffs + i * sCoef;
            u32 m, c, s; memcpy(&m, e, 4); memcpy(&c, e + 4, 4); memcpy(&s, e + 8, 4);
            if (m > 1 || c >= domainSize || s >= nWitness) return -3;
            F coef; memcpy(coef.v, e + 12, 32);
            F* O = m ? B : A;
            O[c] = F::add(O[c], F::mul(coef, W[s]));
        }
        _Pragma("omp parallel for schedule(static)")
        for (long long i = 0; i < (long long)domainSize; i++) C[i] = F::mul(A[i], B[i]);
    })
    return 0;
}

// Group dispatch: group 1 = G1, 2 = G2.
#define GROUP_DISPATCH(curve, group, ...)                                   \
    if (curve == C_BN254 && group == 1)      { typedef Fp<BnFq>   GF; __VA_ARGS__; } \
    else if (curve == C_BN254 && group == 2) { typedef Fp2<BnFq>  GF; __VA_ARGS__; } \
    else if (curve == C_BLS12_381 && group == 1) { typedef Fp<BlsFq>  GF; __VA_ARGS__; } \
    else if (curve == C_BLS12_381 && group == 2) { typedef Fp2<BlsFq> GF; __VA_ARGS__; } \
    else return -1;

// G.multiExpAffine (14666-14668).  out = Jacobian Montgomery (3 coordinates).
int or_multiexp_affine(int curve, int group, const uint8_t* bases, const uint8_t* scalars, int sScalar, u64 n,
                       int concurrency, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J;
        J r = multiexp_affine<GF>((const typename J::Aff*)bases, scalars, sScalar, n, concurrency > 0 ? concurrency : 1);
        memcpy(out, &r, sizeof r);
    })
    return 0;
}

// naive sum_i s_i * P_i by double-and-add (self-check of the Pippenger restatement)
int or_multiexp_naive(int curve, int group, const uint8_t* bases, const uint8_t* scalars, int sScalar, u64 n, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J; const typename J::Aff* B = (const typename J::Aff*)bases;
        J acc = J::zero();
        for (u64 i = 0; i < n; i++) acc = J::add(acc, J::times(J::from_affine(B[i]), scalars + i * sScalar, sScalar));
        memcpy(out, &acc, sizeof acc);
    })
    return 0;
}

// op: 0 add(a,b) jac+jac ; 1 double(a) ; 2 toAffine(a) -> affine ; 3 neg(a) ; 4 addMixed(a jac, b affine) ;
//     5 fromAffine(a affine) -> jac ; 6 eq(a,b) (returns 1/0 in out[0])
int or_group_op(int curve, int group, int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J; J p, q, r; typename J::Aff af;
        switch (op) {
        case 0: memcpy(&p, a, sizeof p); memcpy(&q, b, sizeof q); r = J::add(p, q); memcpy(out, &r, sizeof r); break;
        case 1: memcpy(&p, a, sizeof p); r = J::dbl(p); memcpy(out, &r, sizeof r); break;
        case 2: memcpy(&p, a, sizeof p); af = J::to_affine(p); memcpy(out, &af, sizeof af); break;
        case 3: memcpy(&p, a, sizeof p); r = J::neg(p); memcpy(out, &r, sizeof r); break;
        case 4: memcpy(&p, a, sizeof p); memcpy(&af, b, sizeof af); r = J::add_mixed(p, af); memcpy(out, &r, sizeof r); break;
        case 5: memcpy(&af, a, sizeof af); r = J::from_affine(af); memcpy(out, &r, sizeof r); break;
        case 6: {
            memcpy(&p, a, sizeof p); memcpy(&q, b, sizeof q);
            typename J::Aff x = J::to_affine(p), y = J::to_affine(q);
            out[0] = (x.x == y.x && x.y == y.y) ? 1 : 0; break; }
        default: return -1; }
    })
    return 0;
}

// G.timesScalar: a Jacobian, s plain LE scalar of nbytes.  (g?m_timesFr = fromMontgomery + this, 9426-9456)
int or_group_times(int curve, int group, const uint8_t* a, const uint8_t* s, int nbytes, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J; J p; memcpy(&p, a, sizeof p);
        J r = J::times(p, s, nbytes); memcpy(out, &r, sizeof r);
    })
    return 0;
}

// batchToAffine 6955: n Jacobian -> n affine
int or_batch_to_affine(int curve, int group, const uint8_t* in, u64 n, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J; const J* P = (const J*)in; typename J::Aff* O = (typename J::Aff*)out;
        _Pragma("omp parallel for schedule(static)")
        for (long long i = 0; i < (long long)n; i++) O[i] = J::to_affine(P[i]);
    })
    return 0;
}

// Deterministic synthetic bases for benchmarks/tests: P_0 = k0*G, P_{i+1} = P_i + D (D = kd*G), affine Montgomery.
// gen = affine generator bytes.  Every chunk of 4096 points restarts from (k0 + chunk)*G' to allow OpenMP.
int or_gen_points(int curve, int group, const uint8_t* gen_affine, u64 seed, u64 n, uint8_t* out) {
    ensure_init();
    GROUP_DISPATCH(curve, group, {
        typedef Jac<GF> J; typename J::Aff g; memcpy(&g, gen_affine, sizeof g);
        typename J::Aff* O = (typename J::Aff*)out;
        const u64 CH = 4096; long long nch = (long long)((n + CH - 1) / CH);
        u64 kd = seed * 2654435761ull + 12345; uint8_t kdb[8]; memcpy(kdb, &kd, 8);
        J D = J::times(J::from_affine(g), kdb, 8);
        typename J::Aff Da = J::to_affine(D);
        _Pragma("omp parallel for schedule(dynamic, 1)")
        for (long long c = 0; c < nch; c++) {
            u64 k0 = (seed ^ 0x9E3779B97F4A7C15ull) + (u64)c * 0xD1B54A32D192ED03ull; uint8_t kb[8]; memcpy(kb, &k0, 8);
            J p = J::times(J::from_affine(g), kb, 8);
            u64 lo = (u64)c * CH, hi = std::min(n, lo + CH);
            std::vector<J> tmp(hi - lo);
            for (u64 i = lo; i < hi; i++) { tmp[i - lo] = p; p = J::add_mixed(p, Da); }
            // batch inversion of Z (Montgomery trick)
            std::vector<GF> pref(hi - lo); GF acc = GF::one();
            for (u64 i = 0; i < hi - lo; i++) { pref[i] = acc; acc = GF::mul(acc, tmp[i].z); }
            GF inv = GF::inv(acc);
            for (long long i = (long long)(hi - lo) - 1; i >= 0; i--) {
                GF zi = GF::mul(inv, pref[i]); inv = GF::mul(inv, tmp[i].z);
                GF zi2 = GF::sqr(zi);
                O[lo + i].x = GF::mul(tmp[i].x, zi2); O[lo + i].y = GF::mul(tmp[i].y, GF::mul(zi2, zi));
            }
        }
    })
    return 0;
}

}  // extern "C"
