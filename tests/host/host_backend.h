// Host backend shared by host_plonk.cpp and host_fflonk.cpp: the Backend concept of plonk_flow.h implemented with plain
// loops over the plonk.cuh element functions; NTT / MSM are borrowed from the CPU oracle (function pointers filled by
// the caller from dlopen).  Test infrastructure only.  The independent element loops carry OpenMP pragmas: bench.py's
// reference arm compiles this with -fopenmp as the multi-threaded CPU port of plonk prove / fflonk prove.
#pragma once
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <dlfcn.h>
#include <vector>
#include <string>
#include "../../snarkjs_b200/csrc/plonk_flow.h"
using namespace sb;

typedef int (*or_fft_t)(int, const uint8_t*, uint64_t, int, uint8_t*);
typedef int (*or_msm_t)(int, int, const uint8_t*, const uint8_t*, int, uint64_t, int, uint8_t*);
typedef int (*or_gop_t)(int, int, int, const uint8_t*, const uint8_t*, uint8_t*);
typedef int (*or_root_t)(int, int, uint8_t*);

template <class F> struct HostBackend {
    or_fft_t fft; or_msm_t msm; or_gop_t gop;
    int curve; uint32_t n8q;
    const uint8_t* ptau;
    std::vector<std::vector<F>> pow_store;
    std::string err;

    void mark(int) {}
    void upload(F* dst, const F* host, size_t n) { memcpy(dst, host, n * sizeof(F)); }
    void download(F* host, const F* src, size_t n) { memcpy(host, src, n * sizeof(F)); }
    void zero(F* p, size_t n) { memset(p, 0, n * sizeof(F)); }
    void copy(F* dst, const F* src, size_t n) { memmove(dst, src, n * sizeof(F)); }
    F* ntt(F* a, F* b, uint64_t n, bool inverse) { fft(curve, (const uint8_t*)a, n, inverse ? 1 : 0, (uint8_t*)b); return b; }
    int commit_plain(const F* scal, uint64_t len, uint8_t* affine) {
        std::vector<uint8_t> jac(3 * n8q), aff(3 * n8q);
        if (msm(curve, 1, ptau, (const uint8_t*)scal, 32, len, 4, jac.data())) return -9;
        if (gop(curve, 1, 2, jac.data(), nullptr, aff.data())) return -9;
        memcpy(affine, aff.data(), 2 * n8q);
        return 0;
    }
    int commit(const F* coef, uint64_t len, uint8_t* affine) {
        std::vector<F> s(len);
        _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < len; i++) s[i] = F::from_mont(coef[i]);
        return commit_plain(s.data(), len, affine);
    }
    void additions(const PlonkKeyView<F>& k, F* W) {
        uint32_t lo = 0;
        for (uint32_t hi : k.level_end) { for (uint32_t j = lo; j < hi; j++) pl_addition<F>(k.add_order[j], k.add_sig, k.add_fac, W, k.nVars - k.nAdditions, k.nVars); lo = hi; }
    }
    void wires(const PlonkKeyView<F>& k, const F* W, F* A, F* B, F* C) {
        F* out[3] = {A, B, C};
        for (int j = 0; j < 3; j++) { _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < k.n; i++) pl_wire<F>(i, k.map[j], W, k.nVars, k.nConstraints, out[j]); }
    }
    void blind(F* p, uint64_t n, const F* bf, int cnt) { pl_blind<F>(p, n, bf, cnt); }
    int z(const PlonkKeyView<F>& k, const PlonkRound<F>& r, PlonkWork<F>& w) {
        const uint64_t n = k.n;
        _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < n; i++) pl_z_terms<F>(i, w.bufA, w.bufB, w.bufC, k.s_ev[0], k.s_ev[1], k.s_ev[2], k.wpow, r, w.num, w.den);
        _Pragma("omp parallel for schedule(static)") for (uint64_t lo = 0; lo < n; lo += 16) pl_ratio_chunk<F>(w.den, w.num, w.ratio, lo, lo + 16 < n ? lo + 16 : n);
        F acc = F::one();
        for (uint64_t i = 0; i < n; i++) { w.bufZ[i] = acc; acc = F::mul(acc, w.ratio[i]); }     // exclusive product scan
        return (F::mul(w.bufZ[n - 1], w.ratio[n - 1]) == F::one()) ? 0 : 4;
    }
    void t(const PlonkKeyView<F>& k, const PlonkRound<F>& r, PlonkWork<F>& w) {
        PlonkTIn in;
        in.A = w.evA; in.B = w.evB; in.C = w.evC; in.Z = w.evZ;
        in.QM = k.q_ev[0]; in.QL = k.q_ev[1]; in.QR = k.q_ev[2]; in.QO = k.q_ev[3]; in.QC = k.q_ev[4];
        in.S1 = k.s_ev[0]; in.S2 = k.s_ev[1]; in.S3 = k.s_ev[2]; in.LAG = k.lag; in.pubA = w.bufA; in.n_public = k.nPublic;
        _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < 4ull * k.n; i++) pl_t_eval<F>(i, 4ull * k.n, in, k.w4pow, r, w.T, w.Tz);
    }
    int divzh(uint64_t n, const F* t, const F* tz, F* out) { int f = 0; _Pragma("omp parallel for schedule(static) reduction(|:f)") for (uint64_t i = 0; i < n; i++) f |= pl_divzh<F>(i, n, t, tz, out); return f; }
    void tsplit(uint64_t n, const F* t, const F& b10, const F& b11, F* T1, F* T2, F* T3) { _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < n + 6; i++) pl_tsplit<F>(i, n, t, b10, b11, T1, T2, T3); }
    void make_pow(const F& base, uint64_t count, PlonkPow<F>& out, int) {
        int h = plonk_pow_h(count);
        std::vector<F> lo, hi; plonk_pow_tables<F>(base, h, (count >> h) + 1, lo, hi);
        pow_store.push_back(lo); out.lo = pow_store.back().data();
        pow_store.push_back(hi); out.hi = pow_store.back().data(); out.h = h;
    }
    F eval(const F* f, uint64_t len, const PlonkPow<F>& pw, F*, F*) {
        // field addition is exact: any grouping of the sum gives the same element, so the chunks may run in parallel
        const uint64_t CH = 64; std::vector<F> part(CH, F::zero());
        _Pragma("omp parallel for schedule(static)") for (uint64_t c = 0; c < CH; c++) {
            F s = F::zero(); const uint64_t lo = len * c / CH, hi = len * (c + 1) / CH;
            for (uint64_t i = lo; i < hi; i++) s = F::add(s, F::mul(f[i], pl_pow(pw, i)));
            part[c] = s;
        }
        F s = F::zero();
        for (uint64_t c = 0; c < CH; c++) s = F::add(s, part[c]);
        return s;
    }
    int quotient(const F* f, const PlonkLinIn* lin, const PlonkLin<F>* L, uint64_t n, uint64_t len, uint64_t m, const F& sub0,
                 const PlonkPow<F>& pw, const PlonkPow<F>& ipw, F* g, F* P, F* q_plain) {
        _Pragma("omp parallel for schedule(static)") for (uint64_t i = 0; i < m; i++) {
            F x;
            if (lin) x = pl_wxi_coef<F>(i, n, *lin, *L);
            else { x = i < len ? f[i] : F::zero(); if (i == 0) x = F::sub(x, sub0); }
            g[i] = F::mul(x, pl_pow(pw, i));
        }
        F acc = F::zero();
        for (uint64_t i = 0; i < m; i++) { acc = F::add(acc, g[i]); P[i] = acc; }                    // inclusive sum scan
        _Pragma("omp parallel for schedule(static)") for (uint64_t j = 0; j < m; j++) q_plain[j] = F::from_mont(pl_quot_coef<F>(j, m, P, ipw));
        return P[m - 1].is_zero() ? 0 : 1;
    }
};

// The key arrays of a parsed PLONK / fflonk key (zkey.h's PlonkLayout), copied out of the container the way the device
// loaders upload them, with the view's pointers set to them
template <class F> struct HostKeyArrays {
    std::vector<uint32_t> sig, order, maps[3];
    std::vector<F> fac, q_coef[5], q_ev[5], s_coef[3], s_ev[3], lag;
    static const F* copy(std::vector<F>& v, const Span& s) { v.resize(s.len / sizeof(F)); if (s.len) memcpy(v.data(), s.p, s.len); return v.data(); }
    template <class View> void fill(const PlonkHeader& z, const PlonkLayout& lay, View& k) {
        const uint64_t n = z.n;
        sig.assign(2 * (size_t)z.nAdditions + 2, 0); fac.assign(2 * (size_t)z.nAdditions + 2, F::zero());
        for (uint32_t i = 0; i < z.nAdditions; i++) { memcpy(&sig[2 * i], lay.additions.p + 72 * (size_t)i, 8); memcpy(&fac[2 * i], lay.additions.p + 72 * (size_t)i + 8, 64); }
        plonk_addition_levels(sig.data(), z.nAdditions, z.nVars - z.nAdditions, order, k.level_end);
        k.add_sig = sig.data(); k.add_fac = fac.data(); k.add_order = order.data();
        for (int j = 0; j < 3; j++) { maps[j].assign(z.nConstraints + 1, 0); if (lay.maps[j].len) memcpy(maps[j].data(), lay.maps[j].p, lay.maps[j].len); k.map[j] = maps[j].data(); }
        for (int j = 0; j < 5; j++) { k.q_coef[j] = copy(q_coef[j], lay.q_coef[j]); k.q_ev[j] = copy(q_ev[j], lay.q_ev[j]); }
        for (int j = 0; j < 3; j++) { k.s_coef[j] = copy(s_coef[j], lay.s_coef[j]); k.s_ev[j] = copy(s_ev[j], lay.s_ev[j]); }
        lag.assign((size_t)(z.nPublic > 1 ? z.nPublic : 1) * 4 * n, F::zero());                // polynomials the key leaves out stay zero
        for (size_t j = 0; j < lay.lag.size(); j++) memcpy(lag.data() + j * 4 * n, lay.lag[j].p, lay.lag[j].len);
        k.lag = lag.data();
    }
};
