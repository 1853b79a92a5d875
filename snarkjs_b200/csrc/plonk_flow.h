// plonk_flow.h — the PLONK prover's control flow (src/plonk_prove.js:47-889): five rounds, the Keccak transcript and
// the handful of scalar computations between the bulk steps.  Pure host C++, templated on a Backend that owns the
// bulk data and runs the bulk steps:
//
//   * api_plonk.inl's CUDA backend (kernels of plonk.cuh, the NTT passes of ntt.cuh, the MSM pipeline of msm.cuh);
//   * tests/host/host_plonk.cpp's host backend (the same plonk.cuh element functions in plain loops, NTT / MSM through
//     the CPU oracle) — so this file and plonk.cuh are checked against the oracle without a GPU.
//
// Field elements are canonical Montgomery (Fp<PR>) except the witness, which is plain like the wtns file.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include "plonk.cuh"
#include "zkey.h"

namespace sb {

// ------------------------------------------------------------------------------------------------ Keccak-256
// (src/Keccak256Transcript.js:21 uses @noble/hashes keccak_256: Keccak-f[1600], rate 136, domain byte 0x01)
inline void keccak_f1600(uint64_t* a) {
    static const uint64_t RC[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull, 0x000000000000808Bull,
        0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008Aull, 0x0000000000000088ull, 0x0000000080008009ull,
        0x000000008000000Aull, 0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull, 0x8000000000008003ull, 0x8000000000008002ull,
        0x8000000000000080ull, 0x000000000000800Aull, 0x800000008000000Aull, 0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull,
        0x8000000080008008ull};
    static const int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};   // [x + 5y]
    auto rol = [](uint64_t x, int n) { return n ? (x << n) | (x >> (64 - n)) : x; };
    for (int round = 0; round < 24; round++) {
        uint64_t c[5], d[5], b[25];
        for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rol(c[(x + 1) % 5], 1);
        for (int i = 0; i < 25; i++) a[i] ^= d[i % 5];
        for (int x = 0; x < 5; x++) for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rol(a[x + 5 * y], ROT[x + 5 * y]);
        for (int x = 0; x < 5; x++) for (int y = 0; y < 5; y++) a[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
        a[0] ^= RC[round];
    }
}
inline void keccak256(const uint8_t* data, size_t len, uint8_t out[32]) {
    const size_t rate = 136;
    std::vector<uint8_t> msg(data, data + len);
    msg.push_back(0x01);
    while (msg.size() % rate) msg.push_back(0);
    msg.back() |= 0x80;
    uint64_t a[25] = {0};
    for (size_t off = 0; off < msg.size(); off += rate) {
        for (size_t i = 0; i < rate / 8; i++) { uint64_t w = 0; for (int k = 7; k >= 0; k--) w = (w << 8) | msg[off + 8 * i + k]; a[i] ^= w; }
        keccak_f1600(a);
    }
    for (int i = 0; i < 4; i++) for (int k = 0; k < 8; k++) out[8 * i + k] = (uint8_t)(a[i] >> (8 * k));
}

// ------------------------------------------------------------------------------------------------ transcript
template <class PQ, class PR> struct PlonkTranscript {
    typedef Fp<PQ> Q; typedef Fp<PR> F;
    std::vector<uint8_t> buf;
    void reset() { buf.clear(); }
    // G1.toRprUncompressed (build/snarkjs.js:13725-13735, 7122-7148): x | y plain big-endian; infinity is all zeros
    void add_point(const uint8_t* affine_mont) {
        for (int k = 0; k < 2; k++) {
            Q c; memcpy(&c, affine_mont + k * sizeof(Q), sizeof(Q)); c = Q::from_mont(c);
            const uint8_t* le = (const uint8_t*)&c;
            for (size_t i = 0; i < sizeof(Q); i++) buf.push_back(le[sizeof(Q) - 1 - i]);
        }
    }
    // Fr.toRprBE (build/snarkjs.js:13052-13060)
    void add_scalar(const F& s) {
        F c = F::from_mont(s); const uint8_t* le = (const uint8_t*)&c;
        for (size_t i = 0; i < sizeof(F); i++) buf.push_back(le[sizeof(F) - 1 - i]);
    }
    // Fr.e(Scalar.fromRprBE(keccak_256(buffer))) (Keccak256Transcript.js:67-70)
    F challenge() const {
        uint8_t h[32]; keccak256(buf.data(), buf.size(), h);
        uint32_t x[8];
        for (int i = 0; i < 8; i++) x[i] = (uint32_t)h[31 - 4 * i] | ((uint32_t)h[30 - 4 * i] << 8) | ((uint32_t)h[29 - 4 * i] << 16) | ((uint32_t)h[28 - 4 * i] << 24);
        for (;;) {   // x mod r: r > 2^253, so at most a few subtractions
            bool ge = true;
            for (int i = 7; i >= 0; i--) { if (x[i] != PR::p(i)) { ge = x[i] > PR::p(i); break; } }
            if (!ge) break;
            uint64_t borrow = 0;
            for (int i = 0; i < 8; i++) { uint64_t d = (uint64_t)x[i] - PR::p(i) - borrow; x[i] = (uint32_t)d; borrow = (d >> 32) & 1; }
        }
        F c; memcpy(&c, x, 32);
        return F::to_mont(c);
    }
};


template <class F> inline F fr_from_u64(uint64_t x) { F a = F::zero(); a.v[0] = (uint32_t)x; a.v[1] = (uint32_t)(x >> 32); return F::to_mont(a); }
template <class F> inline F fr_pow2k(F x, int k) { for (int i = 0; i < k; i++) x = F::sqr(x); return x; }   // x^(2^k)

// lo[e] = base^e (e < 2^h), hi[e] = base^(e 2^h) (e < nhi)
template <class F> inline void plonk_pow_tables(const F& base, int h, uint64_t nhi, std::vector<F>& lo, std::vector<F>& hi) {
    lo.resize((size_t)1 << h); hi.resize(nhi ? nhi : 1);
    F t = F::one();
    for (size_t e = 0; e < lo.size(); e++) { lo[e] = t; t = F::mul(t, base); }
    F step = t; t = F::one();
    for (size_t e = 0; e < hi.size(); e++) { hi[e] = t; t = F::mul(t, step); }
}
inline int plonk_pow_h(uint64_t count) { int bits = 0; while (((uint64_t)1 << bits) < count) bits++; return (bits + 1) / 2; }

// what the key looks like to the flow: sizes, header values (host) and the bulk arrays (backend memory)
template <class F> struct PlonkKeyView {
    uint32_t nVars = 0, nPublic = 0, n = 0, nAdditions = 0, nConstraints = 0; int power = 0;
    F k1, k2, wn, w4n;                            // wn = Fr.w[power], w4n = Fr.w[power + 2]
    F z1[4], z2[4], z3[4];                        // MulZ tables
    const uint8_t* hdr_pts = nullptr;             // Qm Ql Qr Qo Qc S1 S2 S3: affine Montgomery bytes (host)
    uint32_t aff_bytes = 64;
    const uint32_t* add_sig = nullptr; const F* add_fac = nullptr; const uint32_t* add_order = nullptr;
    std::vector<uint32_t> level_end;              // additions sorted by dependency level: level l is order[level_end[l-1] .. level_end[l])
    const uint32_t* map[3] = {nullptr, nullptr, nullptr};
    const F* q_coef[5] = {nullptr}; const F* q_ev[5] = {nullptr};     // QM QL QR QO QC
    const F* s_coef[3] = {nullptr}; const F* s_ev[3] = {nullptr};
    const F* lag = nullptr;                       // max(nPublic, 1) arrays of 4n evaluations
    PlonkPow<F> wpow, w4pow;                      // powers of wn (n of them) and of w4n (4n)
};
// MulZ constants (src/mul_z.js:21-47) from w2 = Fr.w[2]
template <class F> inline void plonk_mulz_tables(const F& w2, F z1[4], F z2[4], F z3[4]) {
    const F one = F::one(), two = F::add(one, one), four = F::add(two, two), eight = F::add(four, four);
    z1[0] = F::zero(); z1[1] = F::add(F::neg(one), w2); z1[2] = F::neg(two); z1[3] = F::sub(F::neg(one), w2);
    z2[0] = F::zero(); z2[1] = F::mul(F::neg(two), w2); z2[2] = four; z2[3] = F::mul(two, w2);
    z3[0] = F::zero(); z3[1] = F::add(two, F::mul(two, w2)); z3[2] = F::neg(eight); z3[3] = F::sub(two, F::mul(two, w2));
}

template <class F> struct PlonkWork {             // backend memory, F elements
    F *W = nullptr;                               // nVars + 1
    F *bufA = nullptr, *bufB = nullptr, *bufC = nullptr, *bufZ = nullptr, *num = nullptr, *den = nullptr, *ratio = nullptr, *sn = nullptr;   // n each
    F *cA = nullptr, *cB = nullptr, *cC = nullptr, *cZ = nullptr, *T1 = nullptr, *T2 = nullptr, *T3 = nullptr, *g = nullptr, *P = nullptr, *scal = nullptr;   // n + 8 each
    F *evA = nullptr, *evB = nullptr, *evC = nullptr, *evZ = nullptr, *T = nullptr, *Tz = nullptr, *s4a = nullptr, *s4b = nullptr;   // 4n each
};
static constexpr int PLONK_PAD = 8;

// Backend concept (B):
//   void upload(F* dst, const F* host, size_t n);  void download(F* host, const F* src, size_t n);
//   void zero(F* p, size_t n);  void copy(F* dst, const F* src, size_t n);
//   F* ntt(F* a, F* b, uint64_t n, bool inverse);                 // a is clobbered; returns a or b
//   int commit(const F* coef, uint64_t len, uint8_t* affine);     // MSM of fromMontgomery(coef) over PTau[0..len)
//   void additions(const PlonkKeyView<F>&, F* W);  void wires(const PlonkKeyView<F>&, const F* W, F* A, F* B, F* C);
//   void blind(F* p, uint64_t n, const F* bf, int cnt);
//   int z(const PlonkKeyView<F>&, const PlonkRound<F>&, PlonkWork<F>&);                 // -> w.bufZ; nonzero flag = error
//   void t(const PlonkKeyView<F>&, const PlonkRound<F>&, PlonkWork<F>&);                // -> w.T, w.Tz
//   int divzh(uint64_t n, const F* t, const F* tz, F* out);  void tsplit(uint64_t n, const F* t, const F& b10, const F& b11, F* T1, F* T2, F* T3);
//   void make_pow(const F& base, uint64_t count, PlonkPow<F>& out, int slot);           // tables in backend memory
//   F eval(const F* f, uint64_t len, const PlonkPow<F>& pw, F* g, F* P);                // sum f[k] x^k
//   void mark(int round);                                                               // end of round 1..5 (timing hook; may be a no-op)
//   int quotient(const F* f_or_null, const PlonkLinIn*, const PlonkLin<F>*, uint64_t n, uint64_t len, uint64_t m, const F& sub0,
//                const PlonkPow<F>& pw, const PlonkPow<F>& ipw, F* g, F* P, F* q_plain); // f / (X - b) -> plain scalars
//   int commit_plain(const F* scal_plain, uint64_t len, uint8_t* affine);
// Returns 0, a positive code for the reference's own errors (2 witness length, 3 copy constraints, 4 divisibility; err holds
// the reference's message) or the backend's negative code.
template <class PQ, class PR, class B>
int plonk_prove_flow(B& be, const PlonkKeyView<Fp<PR>>& k, PlonkWork<Fp<PR>>& w, const uint8_t* witness_plain, uint64_t n_witness,
                     const uint8_t* blinders_mont /*11 x 32*/, uint8_t* proof_out, std::string& err) {
    typedef Fp<PR> F;
    const uint64_t n = k.n;
    const uint32_t aff = k.aff_bytes;
    if (n_witness != (uint64_t)k.nVars - k.nAdditions) {                                             // plonk_prove.js:66-68
        err = "Invalid witness length. Circuit: " + std::to_string(k.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k.nAdditions);
        return 2;
    }
    PlonkRound<F> r;
    r.b[0] = F::zero();
    for (int i = 1; i <= 11; i++) memcpy(&r.b[i], blinders_mont + 32 * (i - 1), 32);
    r.k1 = k.k1; r.k2 = k.k2; r.wn = k.wn;
    for (int i = 0; i < 4; i++) { r.z1[i] = k.z1[i]; r.z2[i] = k.z2[i]; r.z3[i] = k.z3[i]; }
    r.beta = r.gamma = r.alpha = r.alpha2 = F::zero();

    uint8_t* pt_A = proof_out; uint8_t* pt_B = pt_A + aff; uint8_t* pt_C = pt_B + aff; uint8_t* pt_Z = pt_C + aff;
    uint8_t* pt_T1 = pt_Z + aff; uint8_t* pt_T2 = pt_T1 + aff; uint8_t* pt_T3 = pt_T2 + aff; uint8_t* pt_Wxi = pt_T3 + aff; uint8_t* pt_Wxiw = pt_Wxi + aff;
    uint8_t* ev_out = pt_Wxiw + aff;     // eval_a, eval_b, eval_c, eval_s1, eval_s2, eval_zw (Montgomery)

    // ---------------- round 1 (:244-313)
    be.upload(w.W, (const F*)witness_plain, n_witness);
    be.zero(w.W, 1);                                                                                 // :97-99
    be.zero(w.W + n_witness, (size_t)k.nAdditions + 1);                                              // BigBuffer starts zeroed (:100)
    be.additions(k, w.W);
    be.wires(k, w.W, w.bufA, w.bufB, w.bufC);
    {
        F* bufs[3] = {w.bufA, w.bufB, w.bufC}; F* cs[3] = {w.cA, w.cB, w.cC}; F* evs[3] = {w.evA, w.evB, w.evC};
        uint8_t* pts[3] = {pt_A, pt_B, pt_C};
        const int bi[3][2] = {{2, 1}, {4, 3}, {6, 5}};
        for (int j = 0; j < 3; j++) {
            be.copy(w.num, bufs[j], n);
            F* res = be.ntt(w.num, w.den, n, true);                                                  // Polynomial.fromEvaluations
            be.zero(cs[j] + n, PLONK_PAD); be.copy(cs[j], res, n);
            be.zero(w.s4a + n, 3 * n); be.copy(w.s4a, cs[j], n);
            res = be.ntt(w.s4a, w.s4b, 4 * n, false);                                                // Evaluations.fromPolynomial(.., 4)
            be.copy(evs[j], res, 4 * n);
            F bf[2] = {r.b[bi[j][0]], r.b[bi[j][1]]};
            be.blind(cs[j], n, bf, 2);
            int rc = be.commit(cs[j], n + 2, pts[j]); if (rc) return rc;
        }
    }
    be.mark(1);
    // ---------------- round 2 (:315-458)
    PlonkTranscript<PQ, PR> tr;
    std::vector<F> pubA(k.nPublic);
    if (k.nPublic) be.download(pubA.data(), w.bufA, k.nPublic);
    for (int i = 0; i < 8; i++) tr.add_point(k.hdr_pts + (size_t)i * aff);
    for (uint32_t i = 0; i < k.nPublic; i++) tr.add_scalar(pubA[i]);
    tr.add_point(pt_A); tr.add_point(pt_B); tr.add_point(pt_C);
    r.beta = tr.challenge();
    tr.reset(); tr.add_scalar(r.beta);
    r.gamma = tr.challenge();
    {
        int flag = be.z(k, r, w);
        if (flag) { err = "Copy constraints does not match"; return 3; }                            // :436-438
        be.copy(w.num, w.bufZ, n);
        F* res = be.ntt(w.num, w.den, n, true);
        be.zero(w.cZ + n, PLONK_PAD); be.copy(w.cZ, res, n);
        be.zero(w.s4a + n, 3 * n); be.copy(w.s4a, w.cZ, n);
        res = be.ntt(w.s4a, w.s4b, 4 * n, false);
        be.copy(w.evZ, res, 4 * n);
        F bf[3] = {r.b[9], r.b[8], r.b[7]};
        be.blind(w.cZ, n, bf, 3);
        int rc = be.commit(w.cZ, n + 3, pt_Z); if (rc) return rc;
    }
    be.mark(2);
    // ---------------- round 3 (:460-684)
    tr.reset(); tr.add_scalar(r.beta); tr.add_scalar(r.gamma); tr.add_point(pt_Z);
    r.alpha = tr.challenge();
    r.alpha2 = F::sqr(r.alpha);
    {
        be.t(k, r, w);
        F* ct = be.ntt(w.T, w.s4a, 4 * n, true);
        F* ctz = be.ntt(w.Tz, w.s4b, 4 * n, true);
        int flag = be.divzh(n, ct, ctz, w.evA);                                                      // evA is free after t()
        if (flag & 1) { err = "Polynomial is not divisible"; return 4; }
        if (flag & 2) { err = "T Polynomial is not well calculated"; return 4; }
        be.zero(w.T1 + n, PLONK_PAD); be.zero(w.T2 + n, PLONK_PAD); be.zero(w.T3 + n, PLONK_PAD);
        be.tsplit(n, w.evA, r.b[10], r.b[11], w.T1, w.T2, w.T3);
        int rc = be.commit(w.T1, n + 1, pt_T1); if (rc) return rc;
        rc = be.commit(w.T2, n + 1, pt_T2); if (rc) return rc;
        rc = be.commit(w.T3, n + 6, pt_T3); if (rc) return rc;
    }
    be.mark(3);
    // ---------------- round 4 (:686-708)
    tr.reset(); tr.add_scalar(r.alpha); tr.add_point(pt_T1); tr.add_point(pt_T2); tr.add_point(pt_T3);
    const F xi = tr.challenge();
    const F xiw = F::mul(xi, k.wn);
    PlonkPow<F> pxi, pxiw, ipxi, ipxiw;
    be.make_pow(xi, n + PLONK_PAD, pxi, 0);
    be.make_pow(xiw, n + PLONK_PAD, pxiw, 1);
    const F ea = be.eval(w.cA, n + 2, pxi, w.g, w.P), eb = be.eval(w.cB, n + 2, pxi, w.g, w.P), ec = be.eval(w.cC, n + 2, pxi, w.g, w.P);
    const F es1 = be.eval(k.s_coef[0], n, pxi, w.g, w.P), es2 = be.eval(k.s_coef[1], n, pxi, w.g, w.P);
    const F ezw = be.eval(w.cZ, n + 3, pxiw, w.g, w.P);
    { const F evs[6] = {ea, eb, ec, es1, es2, ezw}; memcpy(ev_out, evs, sizeof evs); }
    be.mark(4);
    // ---------------- round 5 (:710-888)
    tr.reset(); tr.add_scalar(xi); tr.add_scalar(ea); tr.add_scalar(eb); tr.add_scalar(ec); tr.add_scalar(es1); tr.add_scalar(es2); tr.add_scalar(ezw);
    PlonkLin<F> L;
    L.v[0] = F::zero(); L.v[1] = tr.challenge();
    for (int i = 2; i < 6; i++) L.v[i] = F::mul(L.v[i - 1], L.v[1]);
    {
        const F xin = fr_pow2k(xi, k.power), zh = F::sub(xin, F::one()), nf = fr_from_u64<F>(n);
        // Lagrange evaluations and PI (:781-806); public signals are the witness values 1..nPublic
        F eval_pi = F::zero(), wq = F::one(), l1 = F::zero();
        const uint32_t nl = k.nPublic > 1 ? k.nPublic : 1;
        for (uint32_t i = 1; i <= nl; i++) {
            F li = F::mul(F::mul(wq, zh), F::inv(F::mul(nf, F::sub(xi, wq))));
            if (i == 1) l1 = li;
            if (i <= k.nPublic) {
                F pub; memcpy(&pub, witness_plain + 32 * (size_t)i, 32); pub = F::to_mont(pub);
                eval_pi = F::sub(eval_pi, F::mul(pub, li));
            }
            wq = F::mul(wq, k.wn);
        }
        const F betaxi = F::mul(r.beta, xi);
        F e2 = F::mul(F::add(F::add(ea, betaxi), r.gamma), F::add(F::add(eb, F::mul(betaxi, k.k1)), r.gamma));
        e2 = F::mul(F::mul(e2, F::add(F::add(ec, F::mul(betaxi, k.k2)), r.gamma)), r.alpha);
        F e3 = F::mul(F::add(F::add(ea, F::mul(r.beta, es1)), r.gamma), F::add(F::add(eb, F::mul(r.beta, es2)), r.gamma));
        e3 = F::mul(F::mul(e3, ezw), r.alpha);
        const F e4 = F::mul(l1, r.alpha2);            // eval_l1 (:791-794) equals L[1]
        L.coef_ab = F::mul(ea, eb); L.ea = ea; L.eb = eb; L.ec = ec;
        L.e24 = F::add(e2, e4); L.e3beta = F::mul(e3, r.beta);
        L.zh = zh; L.xin = xin; L.xin2 = F::sqr(xin);
        L.r0 = F::sub(F::sub(eval_pi, F::mul(e3, F::add(ec, r.gamma))), e4);
        F ws = F::mul(L.v[1], ea);
        ws = F::add(ws, F::mul(L.v[2], eb)); ws = F::add(ws, F::mul(L.v[3], ec));
        ws = F::add(ws, F::mul(L.v[4], es1)); ws = F::add(ws, F::mul(L.v[5], es2));
        L.wsub = ws;
    }
    be.make_pow(F::inv(xi), n + PLONK_PAD, ipxi, 2);
    be.make_pow(F::inv(xiw), n + PLONK_PAD, ipxiw, 3);
    {
        PlonkLinIn in;
        in.QM = k.q_coef[0]; in.QL = k.q_coef[1]; in.QR = k.q_coef[2]; in.QO = k.q_coef[3]; in.QC = k.q_coef[4];
        in.S1 = k.s_coef[0]; in.S2 = k.s_coef[1]; in.S3 = k.s_coef[2];
        in.A = w.cA; in.B = w.cB; in.C = w.cC; in.Z = w.cZ; in.T1 = w.T1; in.T2 = w.T2; in.T3 = w.T3;
        int flag = be.quotient(nullptr, &in, &L, n, 0, n + 6, F::zero(), pxi, ipxi, w.g, w.P, w.scal);
        if (flag) { err = "Polynomial is not divisible"; return 4; }
        int rc = be.commit_plain(w.scal, n + 6, pt_Wxi); if (rc) return rc;
        flag = be.quotient(w.cZ, nullptr, nullptr, n, n + 3, n + 3, ezw, pxiw, ipxiw, w.g, w.P, w.scal);
        if (flag) { err = "Polynomial is not divisible"; return 4; }
        rc = be.commit_plain(w.scal, n + 3, pt_Wxiw); if (rc) return rc;
    }
    be.mark(5);
    return 0;
}

// dependency levels of the additions (an addition may use earlier additions, plonk_prove.js:203-211): order = stable sort by level
inline void plonk_addition_levels(const uint32_t* sig, uint32_t n_add, uint32_t n_wit, std::vector<uint32_t>& order, std::vector<uint32_t>& level_end) {
    std::vector<uint32_t> lvl(n_add, 0);
    uint32_t maxl = 0;
    for (uint32_t i = 0; i < n_add; i++) {
        uint32_t l = 0;
        for (int k = 0; k < 2; k++) { uint32_t s = sig[2 * i + k]; if (s >= n_wit && s - n_wit < i) l = l > lvl[s - n_wit] + 1 ? l : lvl[s - n_wit] + 1; }
        lvl[i] = l; if (l > maxl) maxl = l;
    }
    std::vector<uint32_t> cnt(maxl + 2, 0);
    for (uint32_t i = 0; i < n_add; i++) cnt[lvl[i] + 1]++;
    for (uint32_t l = 0; l <= maxl; l++) cnt[l + 1] += cnt[l];
    level_end.assign(cnt.begin() + 1, cnt.end());
    if (n_add == 0) level_end.clear();
    order.resize(n_add);
    std::vector<uint32_t> pos(cnt.begin(), cnt.end() - 1);
    for (uint32_t i = 0; i < n_add; i++) order[pos[lvl[i]]++] = i;
}

}  // namespace sb
