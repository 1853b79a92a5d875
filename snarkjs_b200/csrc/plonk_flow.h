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
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include "keccak.cuh"
#include "plonk.cuh"
#include "zkey.h"

namespace sb {

// ------------------------------------------------------------------------------------------------ Keccak-256
// (the permutation is keccak.cuh's, shared with the device verifiers)
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

// ---------------------------------------------------------------------------------------------- per-proof scalar steps
// The host-side parts of one proof that both the single flow and the batched flow run: blinders and key constants, the
// transcript of each round, and round 5's scalars.
template <class F> inline void plonk_round_init(const PlonkKeyView<F>& k, const uint8_t* blinders_mont /*11 x 32*/, PlonkRound<F>& r) {
    r.b[0] = F::zero();
    for (int i = 1; i <= 11; i++) memcpy(&r.b[i], blinders_mont + 32 * (i - 1), 32);
    r.k1 = k.k1; r.k2 = k.k2; r.wn = k.wn;
    for (int i = 0; i < 4; i++) { r.z1[i] = k.z1[i]; r.z2[i] = k.z2[i]; r.z3[i] = k.z3[i]; }
    r.beta = r.gamma = r.alpha = r.alpha2 = F::zero();
}
// plonk_prove.js:66-68; 0 or 2 with err set
template <class F> inline int plonk_witness_length(const PlonkKeyView<F>& k, uint64_t n_witness, std::string& err) {
    if (n_witness == (uint64_t)k.nVars - k.nAdditions) return 0;
    err = "Invalid witness length. Circuit: " + std::to_string(k.nVars) + ", witness: " + std::to_string(n_witness) + ", " + std::to_string(k.nAdditions);
    return 2;
}
// the reference's text for the flow's positive codes 3..6
inline const char* plonk_error_text(int code) {
    return code == 3 ? "Copy constraints does not match" : code == 4 ? "Polynomial is not divisible" : code == 5 ? "T Polynomial is not well calculated"
         : code == 6 ? "Evaluations.getEvaluation() out of bounds" : "";
}
// round 2 (:315-330): beta, gamma from the key's eight points, the public A values and the commitments A, B, C
template <class PQ, class PR> inline void plonk_beta_gamma(const PlonkKeyView<Fp<PR>>& k, const Fp<PR>* pubA, const uint8_t* pt_A, const uint8_t* pt_B,
                                                          const uint8_t* pt_C, PlonkRound<Fp<PR>>& r) {
    PlonkTranscript<PQ, PR> tr;
    for (int i = 0; i < 8; i++) tr.add_point(k.hdr_pts + (size_t)i * k.aff_bytes);
    for (uint32_t i = 0; i < k.nPublic; i++) tr.add_scalar(pubA[i]);
    tr.add_point(pt_A); tr.add_point(pt_B); tr.add_point(pt_C);
    r.beta = tr.challenge();
    tr.reset(); tr.add_scalar(r.beta);
    r.gamma = tr.challenge();
}
// round 3 (:460-470)
template <class PQ, class PR> inline void plonk_alpha(const uint8_t* pt_Z, PlonkRound<Fp<PR>>& r) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(r.beta); tr.add_scalar(r.gamma); tr.add_point(pt_Z);
    r.alpha = tr.challenge();
    r.alpha2 = Fp<PR>::sqr(r.alpha);
}
// round 4 (:686-690)
template <class PQ, class PR> inline Fp<PR> plonk_xi(const PlonkRound<Fp<PR>>& r, const uint8_t* pt_T1, const uint8_t* pt_T2, const uint8_t* pt_T3) {
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(r.alpha); tr.add_point(pt_T1); tr.add_point(pt_T2); tr.add_point(pt_T3);
    return tr.challenge();
}
// round 5 (:710-806): the challenge v, its powers and the scalars of computeR / computeWxi.  ev = eval_a, eval_b, eval_c,
// eval_s1, eval_s2, eval_zw; the public signals are the plain witness values 1..nPublic.
template <class PQ, class PR> inline void plonk_lin(const PlonkKeyView<Fp<PR>>& k, const PlonkRound<Fp<PR>>& r, const Fp<PR>& xi, const Fp<PR> ev[6],
                                                    const uint8_t* witness_plain, PlonkLin<Fp<PR>>& L) {
    typedef Fp<PR> F;
    const F ea = ev[0], eb = ev[1], ec = ev[2], es1 = ev[3], es2 = ev[4], ezw = ev[5];
    PlonkTranscript<PQ, PR> tr;
    tr.add_scalar(xi); tr.add_scalar(ea); tr.add_scalar(eb); tr.add_scalar(ec); tr.add_scalar(es1); tr.add_scalar(es2); tr.add_scalar(ezw);
    L.v[0] = F::zero(); L.v[1] = tr.challenge();
    for (int i = 2; i < 6; i++) L.v[i] = F::mul(L.v[i - 1], L.v[1]);
    const uint64_t n = k.n;
    const F xin = fr_pow2k(xi, k.power), zh = F::sub(xin, F::one()), nf = fr_from_u64<F>(n);
    // Lagrange evaluations and PI (:781-806)
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
// Returns 0, a positive code for the reference's own errors (2 witness length, 3 copy constraints, 4 divisibility, 6 a key
// without public signals; err holds the reference's message) or the backend's negative code.
template <class PQ, class PR, class B>
int plonk_prove_flow(B& be, const PlonkKeyView<Fp<PR>>& k, PlonkWork<Fp<PR>>& w, const uint8_t* witness_plain, uint64_t n_witness,
                     const uint8_t* blinders_mont /*11 x 32*/, uint8_t* proof_out, std::string& err) {
    typedef Fp<PR> F;
    const uint64_t n = k.n;
    const uint32_t aff = k.aff_bytes;
    if (plonk_witness_length(k, n_witness, err)) return 2;
    PlonkRound<F> r;
    plonk_round_init(k, blinders_mont, r);

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
    std::vector<F> pubA(k.nPublic);
    if (k.nPublic) be.download(pubA.data(), w.bufA, k.nPublic);
    plonk_beta_gamma<PQ, PR>(k, pubA.data(), pt_A, pt_B, pt_C, r);
    {
        int flag = be.z(k, r, w);
        if (flag) { err = plonk_error_text(3); return 3; }                                            // :436-438
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
    // e4 reads L1 from a buffer of nPublic Lagrange polynomials (:503-509), which throws on a key without public signals
    // (:613-617, evaluations.js:39-44)
    if (!k.nPublic) { err = plonk_error_text(6); return 6; }
    plonk_alpha<PQ, PR>(pt_Z, r);
    {
        be.t(k, r, w);
        F* ct = be.ntt(w.T, w.s4a, 4 * n, true);
        F* ctz = be.ntt(w.Tz, w.s4b, 4 * n, true);
        int flag = be.divzh(n, ct, ctz, w.evA);                                                      // evA is free after t()
        if (flag & 1) { err = plonk_error_text(4); return 4; }
        if (flag & 2) { err = plonk_error_text(5); return 4; }
        be.zero(w.T1 + n, PLONK_PAD); be.zero(w.T2 + n, PLONK_PAD); be.zero(w.T3 + n, PLONK_PAD);
        be.tsplit(n, w.evA, r.b[10], r.b[11], w.T1, w.T2, w.T3);
        int rc = be.commit(w.T1, n + 1, pt_T1); if (rc) return rc;
        rc = be.commit(w.T2, n + 1, pt_T2); if (rc) return rc;
        rc = be.commit(w.T3, n + 6, pt_T3); if (rc) return rc;
    }
    be.mark(3);
    // ---------------- round 4 (:686-708)
    const F xi = plonk_xi<PQ, PR>(r, pt_T1, pt_T2, pt_T3);
    const F xiw = F::mul(xi, k.wn);
    PlonkPow<F> pxi, pxiw, ipxi, ipxiw;
    be.make_pow(xi, n + PLONK_PAD, pxi, 0);
    be.make_pow(xiw, n + PLONK_PAD, pxiw, 1);
    const F ea = be.eval(w.cA, n + 2, pxi, w.g, w.P), eb = be.eval(w.cB, n + 2, pxi, w.g, w.P), ec = be.eval(w.cC, n + 2, pxi, w.g, w.P);
    const F es1 = be.eval(k.s_coef[0], n, pxi, w.g, w.P), es2 = be.eval(k.s_coef[1], n, pxi, w.g, w.P);
    const F ezw = be.eval(w.cZ, n + 3, pxiw, w.g, w.P);
    const F evs[6] = {ea, eb, ec, es1, es2, ezw};
    memcpy(ev_out, evs, sizeof evs);
    be.mark(4);
    // ---------------- round 5 (:710-888)
    PlonkLin<F> L;
    plonk_lin<PQ, PR>(k, r, xi, evs, witness_plain, L);
    be.make_pow(F::inv(xi), n + PLONK_PAD, ipxi, 2);
    be.make_pow(F::inv(xiw), n + PLONK_PAD, ipxiw, 3);
    {
        PlonkLinIn in;
        in.QM = k.q_coef[0]; in.QL = k.q_coef[1]; in.QR = k.q_coef[2]; in.QO = k.q_coef[3]; in.QC = k.q_coef[4];
        in.S1 = k.s_coef[0]; in.S2 = k.s_coef[1]; in.S3 = k.s_coef[2];
        in.A = w.cA; in.B = w.cB; in.C = w.cC; in.Z = w.cZ; in.T1 = w.T1; in.T2 = w.T2; in.T3 = w.T3;
        int flag = be.quotient(nullptr, &in, &L, n, 0, n + 6, F::zero(), pxi, ipxi, w.g, w.P, w.scal);
        if (flag) { err = plonk_error_text(4); return 4; }
        int rc = be.commit_plain(w.scal, n + 6, pt_Wxi); if (rc) return rc;
        flag = be.quotient(w.cZ, nullptr, nullptr, n, n + 3, n + 3, ezw, pxiw, ipxiw, w.g, w.P, w.scal);
        if (flag) { err = plonk_error_text(4); return 4; }
        rc = be.commit_plain(w.scal, n + 3, pt_Wxiw); if (rc) return rc;
    }
    be.mark(5);
    return 0;
}

// ---------------------------------------------------------------------------------------------- batched flow
// K proofs against one key in lockstep.  Every work array holds the K proofs back to back at a fixed stride (array-major),
// so a round's transforms are one strided NTT and its commitments one batch of MSM rows.  Coefficient arrays have the
// stride plonk_batch_p(n) = n + 6: every commitment runs over n + 6 points, and the zeros past a polynomial's length add
// nothing to it.
inline uint64_t plonk_batch_p(uint64_t n) { return n + 6; }
// elements of X and Y per proof: three 4n transforms, or the round-4 terms (6 rows of n + 6) / round-5 rows (2 of n + 6)
inline uint64_t plonk_batch_xy(uint64_t n) { return std::max<uint64_t>(12 * n, 6 * plonk_batch_p(n)); }
template <class F> struct PlonkBatchWork {        // backend memory, F elements; capacities for K proofs
    uint64_t sW = 0;                              // stride of W: nVars + 2
    F* W = nullptr;                               // K x sW witnesses (additions appended)
    F* wires = nullptr;                           // 3K x n: A of every proof, then B, then C (evaluations)
    F *num = nullptr, *den = nullptr, *ratio = nullptr, *Z = nullptr;   // K x n each
    F* cABC = nullptr;                            // 3K x P coefficients of A, B, C (blinded), group-major like wires
    F* cZ = nullptr;                              // K x P
    F* cT = nullptr;                              // 3K x P: T1 rows, T2 rows, T3 rows
    F* scal = nullptr;                            // 3K x P plain MSM scalars
    F* evZ = nullptr;                             // K x 4n
    F *X = nullptr, *Y = nullptr;                 // K x plonk_batch_xy(n) each: NTT data and scratch, then the rounds 4-5 terms
};

// Batch backend concept (BB), the steps over all K proofs at once:
//   void zero(F* p, size_t n);  void copy(F* dst, const F* src, size_t n);
//   void copy2d(F* dst, uint64_t dpitch, const F* src, uint64_t spitch, uint64_t width, uint64_t rows);   // pitches in elements
//   void upload2d(F* dst, uint64_t dpitch, const F* host, uint64_t width, uint64_t rows);   void zero2d(F* dst, uint64_t dpitch, uint64_t width, uint64_t rows);
//   void download2d(F* host, const F* src, uint64_t spitch, uint64_t width, uint64_t rows);
//   F* ntt(F* a, F* b, uint64_t count, uint64_t len, bool inverse);          // count transforms of len contiguous; returns a or b
//   void set_rounds(const PlonkRound<F>* r, uint32_t K);  void set_lin(const PlonkLin<F>* L, const F* ezw, uint32_t K);
//   void additions(const PlonkKeyView<F>&, F* W, uint64_t sW, uint32_t K);  void wires(const PlonkKeyView<F>&, const F* W, uint64_t sW, F* out, uint32_t K);
//   void blind(F* p, uint64_t stride, uint64_t n, uint32_t groups, uint32_t K, const PlonkBlindIdx&);
//   void z(const PlonkKeyView<F>&, const PlonkBatchWork<F>&, uint32_t K, int* flags);                        // -> w.Z
//   void t(const PlonkKeyView<F>&, const F* ev, const F* evZ, const F* wires, F* T /*T rows, Tz rows*/, uint32_t K);
//   void divzh(uint64_t n, const F* t, F* out, uint32_t K, int* flags);  void tsplit(uint64_t n, const F* t, F* cT, uint32_t K);
//   void make_pows(const F* bases /*slots x K*/, int slots, int slot0, uint32_t K, PlonkPowK<F>* out);
//   void evals(const PlonkKeyView<F>&, const PlonkBatchWork<F>&, const PlonkPowK<F>& pxi, const PlonkPowK<F>& pxiw, uint32_t K, F* out /*K x 6*/);
//   void quotients(const PlonkKeyView<F>&, const PlonkBatchWork<F>&, const PlonkPowK<F> pw[4], uint32_t K, int* flags);   // -> 2K rows of w.scal
//   int commit(const F* coef, uint32_t rows, F* scal, uint8_t* affine);  int commit_plain(const F* scal, uint32_t rows, uint8_t* affine);
// flags (host, K ints): what the proof's step found, as the single flow's flags.  status[q] = 0 or the first code 3..6 of
// proof q (plonk_error_text); a failing proof runs on with the others and its slot is zero-filled at the end.  Returns 0 or
// the backend's negative code.  The caller checks the witness length.
template <class PQ, class PR, class BB>
int plonk_prove_flow_batch(BB& be, const PlonkKeyView<Fp<PR>>& k, const PlonkBatchWork<Fp<PR>>& w, uint32_t K, const uint8_t* witnesses_plain,
                           uint64_t n_witness, const uint8_t* blinders_mont /*K x 11 x 32*/, uint8_t* proofs_out, int32_t* status) {
    typedef Fp<PR> F;
    const uint64_t n = k.n, n4 = 4 * n, P = plonk_batch_p(n), sW = w.sW;
    const uint32_t aff = k.aff_bytes;
    const size_t pb = 9 * (size_t)aff + 6 * 32;
    auto pt = [&](uint32_t q, int i) { return proofs_out + q * pb + (size_t)i * aff; };   // A B C Z T1 T2 T3 Wxi Wxiw
    std::vector<int> flags(K, 0);
    auto settle = [&](int bit_mask, int code) { for (uint32_t q = 0; q < K; q++) if ((flags[q] & bit_mask) && !status[q]) status[q] = code; };
    std::vector<uint8_t> pts((size_t)3 * K * aff);
    // commitment rows group-major (row j K + q) -> point first + j of proof q
    auto scatter = [&](uint32_t groups, int first) {
        for (uint32_t j = 0; j < groups; j++) for (uint32_t q = 0; q < K; q++) memcpy(pt(q, first + j), pts.data() + ((size_t)j * K + q) * aff, aff);
    };
    std::vector<PlonkRound<F>> r(K);
    for (uint32_t q = 0; q < K; q++) { plonk_round_init(k, blinders_mont + (size_t)q * 11 * 32, r[q]); status[q] = 0; }
    be.set_rounds(r.data(), K);

    // ---------------- round 1
    be.zero(w.W, (size_t)K * sW);                                                                    // W[0] = 0, additions start zeroed
    be.upload2d(w.W, sW, (const F*)witnesses_plain, n_witness, K);
    be.zero2d(w.W, sW, 1, K);
    be.additions(k, w.W, sW, K);
    be.wires(k, w.W, sW, w.wires, K);
    be.copy(w.X, w.wires, (size_t)3 * K * n);
    F* res = be.ntt(w.X, w.Y, 3ull * K, n, true);
    be.zero(w.cABC, (size_t)3 * K * P);
    be.copy2d(w.cABC, P, res, n, n, 3ull * K);
    be.zero(w.X, (size_t)3 * K * n4);
    be.copy2d(w.X, n4, w.cABC, P, n, 3ull * K);
    F* ev = be.ntt(w.X, w.Y, 3ull * K, n4, false);                                                  // A, B, C on the 4n domain
    F* fr = ev == w.X ? w.Y : w.X;
    { const PlonkBlindIdx bi = {2, {{2, 1, 0}, {4, 3, 0}, {6, 5, 0}}}; be.blind(w.cABC, P, n, 3, K, bi); }
    { int rc = be.commit(w.cABC, 3 * K, w.scal, pts.data()); if (rc) return rc; }
    scatter(3, 0);
    // ---------------- round 2
    {
        std::vector<F> pub((size_t)K * k.nPublic + 1);
        if (k.nPublic) be.download2d(pub.data(), w.wires, n, k.nPublic, K);
        for (uint32_t q = 0; q < K; q++) plonk_beta_gamma<PQ, PR>(k, pub.data() + (size_t)q * k.nPublic, pt(q, 0), pt(q, 1), pt(q, 2), r[q]);
    }
    be.set_rounds(r.data(), K);
    be.z(k, w, K, flags.data());
    settle(~0, 3);
    be.copy(fr, w.Z, (size_t)K * n);
    res = be.ntt(fr, fr + (size_t)K * n4, K, n, true);
    be.zero(w.cZ, (size_t)K * P);
    be.copy2d(w.cZ, P, res, n, n, K);
    be.zero(w.evZ, (size_t)K * n4);
    be.copy2d(w.evZ, n4, w.cZ, P, n, K);
    res = be.ntt(w.evZ, fr, K, n4, false);
    if (res != w.evZ) be.copy(w.evZ, res, (size_t)K * n4);
    { const PlonkBlindIdx bi = {3, {{9, 8, 7}, {0, 0, 0}, {0, 0, 0}}}; be.blind(w.cZ, P, n, 1, K, bi); }
    { int rc = be.commit(w.cZ, K, w.scal, pts.data()); if (rc) return rc; }
    scatter(1, 3);
    // ---------------- round 3
    if (!k.nPublic) {                                                                                // as the single flow: code 6
        for (uint32_t q = 0; q < K; q++) if (!status[q]) status[q] = 6;
        memset(proofs_out, 0, K * pb);
        return 0;
    }
    for (uint32_t q = 0; q < K; q++) plonk_alpha<PQ, PR>(pt(q, 3), r[q]);
    be.set_rounds(r.data(), K);
    be.t(k, ev, w.evZ, w.wires, fr, K);                                                              // T rows, then Tz rows
    res = be.ntt(fr, ev, 2ull * K, n4, true);
    F* oth = res == fr ? ev : fr;
    std::fill(flags.begin(), flags.end(), 0);
    be.divzh(n, res, oth, K, flags.data());
    settle(1, 4); settle(2, 5);
    be.zero(w.cT, (size_t)3 * K * P);
    be.tsplit(n, oth, w.cT, K);
    { int rc = be.commit(w.cT, 3 * K, w.scal, pts.data()); if (rc) return rc; }
    scatter(3, 4);
    // ---------------- round 4
    std::vector<F> xs((size_t)2 * K), evs((size_t)6 * K);
    for (uint32_t q = 0; q < K; q++) { xs[q] = plonk_xi<PQ, PR>(r[q], pt(q, 4), pt(q, 5), pt(q, 6)); xs[K + q] = F::mul(xs[q], k.wn); }
    PlonkPowK<F> pw[4];
    be.make_pows(xs.data(), 2, 0, K, pw);
    be.evals(k, w, pw[0], pw[1], K, evs.data());
    for (uint32_t q = 0; q < K; q++) memcpy(pt(q, 9), evs.data() + 6 * (size_t)q, 6 * sizeof(F));
    // ---------------- round 5
    std::vector<PlonkLin<F>> L(K);
    std::vector<F> ezw(K), ixs((size_t)2 * K);
    for (uint32_t q = 0; q < K; q++) {
        plonk_lin<PQ, PR>(k, r[q], xs[q], evs.data() + 6 * (size_t)q, witnesses_plain + (size_t)q * n_witness * 32, L[q]);
        ezw[q] = evs[6 * (size_t)q + 5];
        ixs[q] = F::inv(xs[q]); ixs[K + q] = F::inv(xs[K + q]);
    }
    be.set_lin(L.data(), ezw.data(), K);
    be.make_pows(ixs.data(), 2, 2, K, pw + 2);
    std::fill(flags.begin(), flags.end(), 0);
    be.quotients(k, w, pw, K, flags.data());
    settle(~0, 4);
    { int rc = be.commit_plain(w.scal, 2 * K, pts.data()); if (rc) return rc; }
    scatter(2, 7);
    for (uint32_t q = 0; q < K; q++) if (status[q]) memset(proofs_out + q * pb, 0, pb);
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
