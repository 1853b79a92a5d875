// zkey.h — the .zkey and .wtns containers: every check on caller-supplied key and witness bytes, and where each array
// the provers upload sits inside them.  Pure host C++ (no CUDA runtime): api.cu's loaders run it before they allocate
// anything, and tests/host builds it with g++ for the host flows and the mutation fuzzer.
//
// binfile container: @iden3/binfileutils readBinFile (build/snarkjs.js:17468-17498).  Groth16: src/zkey_utils.js:229-259;
// PLONK: src/zkey_utils.js:261-299 and src/plonk_constants.js:1-15 (written by src/plonk_setup.js:99-480); fflonk:
// src/zkey_utils.js:301-339 and src/fflonk_constants.js:27-44; wtns: src/wtns_utils.js:62-72.
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>
#include "../../include/snarkb200.h"
#include "fp.cuh"

namespace sb {

struct Span { const uint8_t* p = nullptr; uint64_t len = 0; };
inline Span sub_span(const Span& s, uint64_t off, uint64_t len) { return Span{s.p + off, len}; }   // off + len <= s.len

// section id -> payload.  exact: the container ends where its last section ends (Groth16 zkeys and wtns files, as the
// reference requires); PLONK and fflonk keys may carry trailing bytes.  No id may appear twice.
typedef std::map<uint32_t, Span> Sections;
inline int binfile_sections(const uint8_t* d, uint64_t len, const char* magic, uint32_t max_version, bool exact, Sections& secs, std::string& err) {
    if (len < 12 || memcmp(d, magic, 4) != 0) { err = std::string(magic) + ": Invalid File format"; return -1; }
    uint32_t ver, nsec; memcpy(&ver, d + 4, 4); memcpy(&nsec, d + 8, 4);
    if (ver > max_version) { err = "Version not supported"; return -1; }
    uint64_t pos = 12;
    bool fits = true;
    for (uint32_t i = 0; i < nsec && fits; i++) {
        if (len - pos < 12) { fits = false; break; }
        uint32_t id; uint64_t sl; memcpy(&id, d + pos, 4); memcpy(&sl, d + pos + 4, 8); pos += 12;
        if (sl > len - pos) { fits = false; break; }   // (not pos + sl > len: sl comes from the file and may wrap)
        if (!secs.emplace(id, Span{d + pos, sl}).second) { err = "Section Duplicated " + std::to_string(id); return -1; }
        pos += sl;
    }
    if (!fits || (exact && pos != len)) { err = "Invalid file size"; return -1; }
    return 0;
}

// the n8 little-endian bytes at p are the base (or scalar) field modulus of the curve
inline bool modulus_matches(const uint8_t* p, uint32_t n8, int curve, bool scalar_field) {
    uint32_t limbs[12] = {0};
    if (curve == SB_BN254) { if (n8 != 32) return false; for (int i = 0; i < 8; i++) limbs[i] = scalar_field ? BnFr::p(i) : BnFq::p(i); }
    else if (scalar_field) { if (n8 != 32) return false; for (int i = 0; i < 8; i++) limbs[i] = BlsFr::p(i); }
    else { if (n8 != 48) return false; for (int i = 0; i < 12; i++) limbs[i] = BlsFq::p(i); }
    return memcmp(p, limbs, n8) == 0;
}

// ------------------------------------------------------------------------------------------------ Groth16
// Header values point into the caller's bytes; the CSR arrays are built here.  The loader still checks the moduli
// against its curve and the domain against the 2-adicity of Fr.
struct Groth16Zkey {
    uint32_t n8q = 0, n8r = 0, nVars = 0, nPublic = 0, domainSize = 0; int power = 0;
    const uint8_t *q = nullptr, *r = nullptr;
    const uint8_t *alpha1 = nullptr, *beta1 = nullptr, *beta2 = nullptr, *gamma2 = nullptr, *delta1 = nullptr, *delta2 = nullptr;
    Span A, B1, B2, C, H;                  // sections 5-9: nVars, nVars, nVars (G2), nVars - nPublic - 1 and domainSize points
    // section 4 as CSR over the rows m * domainSize + c (matrix m, constraint c): src/zkey_utils.js:110-118,
    // groth16_prove.js:147-187.  Row i holds entries [rowptr[i], rowptr[i+1]) of sig (signal ids) and coef (32 bytes each).
    std::vector<uint64_t> rowptr; std::vector<uint32_t> sig; std::vector<uint8_t> coef;
};
inline int groth16_parse_zkey(const uint8_t* d, uint64_t len, Groth16Zkey& z, std::string& err) {
    Sections secs;
    if (binfile_sections(d, len, "zkey", 2, true, secs, err)) return -1;
    for (uint32_t id : {1u, 2u, 4u, 5u, 6u, 7u, 8u, 9u}) if (!secs.count(id)) { err = "Missing section " + std::to_string(id); return -1; }
    const Span s1 = secs[1], h = secs[2], s4 = secs[4];
    if (s1.len < 4) { err = "zkey: short read"; return -1; }
    uint32_t proto; memcpy(&proto, s1.p, 4);
    if (proto != 1) { err = "zkey file is not groth16"; return -1; }
    // no supported curve has other field sizes, so no context would match
    const char* other_curve = "zkey curve does not match the context curve";
    if (h.len < 4) { err = "zkey header too short"; return -1; }
    memcpy(&z.n8q, h.p, 4);
    if (z.n8q != 32 && z.n8q != 48) { err = other_curve; return -1; }
    const uint64_t sG1 = 2 * z.n8q, sG2 = 4 * z.n8q, n8r = 32;
    if (h.len < 4 + z.n8q + 4 + n8r + 12 + 3 * sG1 + 3 * sG2) { err = "zkey header too short"; return -1; }
    memcpy(&z.n8r, h.p + 4 + z.n8q, 4);
    if (z.n8r != n8r) { err = other_curve; return -1; }
    z.q = h.p + 4; z.r = h.p + 8 + z.n8q;
    const uint8_t* p = z.r + n8r;
    memcpy(&z.nVars, p, 4); memcpy(&z.nPublic, p + 4, 4); memcpy(&z.domainSize, p + 8, 4); p += 12;
    z.alpha1 = p; p += sG1; z.beta1 = p; p += sG1; z.beta2 = p; p += sG2; z.gamma2 = p; p += sG2; z.delta1 = p; p += sG1; z.delta2 = p;
    const uint64_t n = z.domainSize, nv = z.nVars;
    if (n == 0 || (n & (n - 1))) { err = "domain size is not a power of two"; return -1; }
    while (((uint64_t)1 << z.power) < n) z.power++;
    if (nv < (uint64_t)z.nPublic + 1) { err = "invalid zkey header"; return -1; }
    z.A = secs[5]; z.B1 = secs[6]; z.B2 = secs[7]; z.C = secs[8]; z.H = secs[9];
    if (z.A.len != nv * sG1 || z.B1.len != nv * sG1 || z.B2.len != nv * sG2 || z.C.len != (nv - z.nPublic - 1) * sG1 || z.H.len != n * sG1) {
        err = "zkey section size mismatch"; return -1;
    }
    if (s4.len < 4) { err = "zkey: short read"; return -1; }
    uint32_t ncoef; memcpy(&ncoef, s4.p, 4);
    const uint64_t sCoef = 12 + n8r;
    if (s4.len != 4 + ncoef * sCoef) { err = "zkey coefficient section size mismatch"; return -1; }
    const uint8_t* cf = s4.p + 4;
    z.rowptr.assign(2 * n + 1, 0);
    for (uint64_t i = 0; i < ncoef; i++) {
        uint32_t m, cc, s; memcpy(&m, cf + i * sCoef, 4); memcpy(&cc, cf + i * sCoef + 4, 4); memcpy(&s, cf + i * sCoef + 8, 4);
        if (m > 1 || cc >= n || s >= nv) { err = "zkey coefficient out of range"; return -1; }
        z.rowptr[m * n + cc + 1]++;
    }
    for (uint64_t i = 0; i < 2 * n; i++) z.rowptr[i + 1] += z.rowptr[i];
    std::vector<uint64_t> cursor(z.rowptr.begin(), z.rowptr.end() - 1);
    z.sig.resize(ncoef); z.coef.resize((size_t)ncoef * 32);
    for (uint64_t i = 0; i < ncoef; i++) {
        uint32_t m, cc; memcpy(&m, cf + i * sCoef, 4); memcpy(&cc, cf + i * sCoef + 4, 4);
        const uint64_t at = cursor[m * n + cc]++;
        memcpy(&z.sig[at], cf + i * sCoef + 8, 4); memcpy(&z.coef[at * 32], cf + i * sCoef + 12, 32);
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ wtns
struct Wtns { uint32_t n8 = 0, nWitness = 0; const uint8_t* q = nullptr; Span values; };   // the loader checks q against its curve
inline int wtns_parse(const uint8_t* d, uint64_t len, Wtns& w, std::string& err) {
    Sections secs;
    if (binfile_sections(d, len, "wtns", 2, true, secs, err)) return -1;
    if (!secs.count(1) || !secs.count(2)) { err = "Missing section"; return -1; }
    const Span h = secs[1];
    if (h.len < 4) { err = "wtns header too short"; return -1; }
    memcpy(&w.n8, h.p, 4);
    if (h.len < 8 + (uint64_t)w.n8) { err = "wtns header too short"; return -1; }
    w.q = h.p + 4;
    memcpy(&w.nWitness, h.p + 4 + w.n8, 4);
    w.values = secs[2];
    if (w.values.len != (uint64_t)w.nWitness * w.n8) { err = "Invalid witness section size"; return -1; }
    return 0;
}

// ------------------------------------------------------------------------------------------------ PLONK and fflonk
// Header values of both formats; pointers into section 2 (header).
struct PlonkHeader {
    uint32_t n8q = 0, n8r = 0, nVars = 0, nPublic = 0, n = 0, nAdditions = 0, nConstraints = 0; int power = 0;
    Span header;
    const uint8_t *q = nullptr, *r = nullptr, *k1 = nullptr, *k2 = nullptr, *X_2 = nullptr;
};
// Where the arrays the PLONK and fflonk provers upload sit in the key.
struct PlonkLayout {
    Span additions;                        // nAdditions records (s1 u32, s2 u32, f1, f2): 72 bytes each
    Span maps[3];                          // nConstraints signal ids each
    Span q_coef[5], q_ev[5];               // selectors in section order: n coefficients, 4n evaluations each
    Span s_coef[3], s_ev[3];               // sigmas
    std::vector<Span> lag;                 // 4n evaluations of each Lagrange polynomial present, at most max(nPublic, 1)
    Span ptau;                             // n + 6 (PLONK) or 9n + 18 (fflonk) affine G1 points
    Span c0;                               // fflonk: C0's 8n coefficients
};

// The parse result: header values, the key's sections below id 16 (PLONK) or 20 (fflonk) by id, and the layout.  Its
// pointers point into the caller's bytes.
struct PlonkZkey : PlonkHeader { const uint8_t* hdr_pts = nullptr; Span sec[16]; PlonkLayout lay; };                  // hdr_pts: Qm Ql Qr Qo Qc S1 S2 S3
struct FflonkZkey : PlonkHeader { const uint8_t *w3 = nullptr, *w4 = nullptr, *w8 = nullptr, *wr = nullptr, *C0 = nullptr; Span sec[20]; PlonkLayout lay; };

// What the two formats share: the container, sections 1-2 up to k1 / k2 (the header then holds n_fr more scalars and n_q
// more base-field elements), and the counts' consistency (nConstraints + cons_slack <= n).
inline int plonk_family_header(const uint8_t* d, uint64_t len, uint32_t protocol, const char* not_this, uint32_t n_fr, uint32_t n_q,
                               uint32_t cons_slack, Sections& secs, PlonkHeader& z, std::string& err) {
    if (binfile_sections(d, len, "zkey", 2, false, secs, err)) return -1;
    if (!secs.count(1) || secs[1].len < 4 || !secs.count(2)) { err = "zkey: missing header"; return -1; }
    uint32_t proto; memcpy(&proto, secs[1].p, 4);
    if (proto != protocol) { err = not_this; return -1; }
    z.header = secs[2];
    const uint8_t* h = z.header.p; const uint64_t hl = z.header.len;
    if (hl < 8) { err = "zkey: short header"; return -1; }
    memcpy(&z.n8q, h, 4);
    if (z.n8q != 32 && z.n8q != 48) { err = "zkey: unsupported base field size"; return -1; }
    z.q = h + 4;
    if (hl < 8 + (uint64_t)z.n8q) { err = "zkey: short header"; return -1; }
    memcpy(&z.n8r, h + 4 + z.n8q, 4);
    if (z.n8r != 32) { err = "zkey: unsupported scalar field size"; return -1; }
    z.r = h + 8 + z.n8q;
    const uint64_t o = 8 + (uint64_t)z.n8q + z.n8r;
    if (hl < o + 20 + 32 * (uint64_t)n_fr + (uint64_t)n_q * z.n8q) { err = "zkey: short header"; return -1; }
    memcpy(&z.nVars, h + o, 4); memcpy(&z.nPublic, h + o + 4, 4); memcpy(&z.n, h + o + 8, 4); memcpy(&z.nAdditions, h + o + 12, 4); memcpy(&z.nConstraints, h + o + 16, 4);
    z.k1 = h + o + 20; z.k2 = z.k1 + 32;
    if (z.n < 8 || (z.n & (z.n - 1))) { err = "zkey: domain size is not a power of two"; return -1; }
    z.power = 0; while ((1u << z.power) < z.n) z.power++;
    if (z.nAdditions > z.nVars || (uint64_t)z.nConstraints + cons_slack > z.n || z.nPublic > z.nConstraints ||
        (uint64_t)z.nPublic + 1 > (uint64_t)z.nVars - z.nAdditions)   /* the public signals are witness[1..nPublic] */ { err = "zkey: inconsistent header"; return -1; }
    return 0;
}

// The sections below id nsec into sec[id]; sections 3..last must hold at least want[id] bytes (lag_id's may hold exactly
// nPublic Lagrange polynomials instead of max(nPublic, 1)).  Then the spans both formats place alike: additions, wire maps
// and selectors.
inline int plonk_family_sections(const Sections& secs, const PlonkHeader& z, const uint64_t* want, int last, int lag_id,
                                 Span* sec, uint32_t nsec, PlonkLayout& lay, std::string& err) {
    const uint64_t sd = (uint64_t)z.n * 32;
    for (const auto& kv : secs) if (kv.first < nsec) sec[kv.first] = kv.second;
    for (int id = 3; id <= last; id++) {
        if (!secs.count(id) && want[id]) { err = "zkey: missing section " + std::to_string(id); return -1; }
        const uint64_t need = id == lag_id ? z.nPublic * 5 * sd : want[id];
        if (sec[id].len < need) { err = "zkey: section " + std::to_string(id) + " too short"; return -1; }
    }
    lay.additions = sub_span(sec[3], 0, (uint64_t)z.nAdditions * 72);
    for (int j = 0; j < 3; j++) lay.maps[j] = sub_span(sec[4 + j], 0, (uint64_t)z.nConstraints * 4);
    for (int j = 0; j < 5; j++) { lay.q_coef[j] = sub_span(sec[7 + j], 0, sd); lay.q_ev[j] = sub_span(sec[7 + j], sd, 4 * sd); }
    return 0;
}

// PLONK (protocol 2): the three sigmas one after the other in section 12, the Lagrange polynomials in 13, n + 6 PTau
// points in 14
inline int plonk_parse_zkey(const uint8_t* d, uint64_t len, PlonkZkey& z, std::string& err) {
    Sections secs;
    if (plonk_family_header(d, len, 2, "zkey file is not plonk", 2, 8 * 2 + 4, 0, secs, z, err)) return -1;   // plonk_prove.js:58-60
    z.hdr_pts = z.k2 + 32; z.X_2 = z.hdr_pts + 8 * 2 * z.n8q;
    const uint64_t n = z.n, sd = n * 32, npl = z.nPublic > 1 ? z.nPublic : 1, nc4 = (uint64_t)z.nConstraints * 4;
    const uint64_t want[15] = {0, 0, 0, (uint64_t)z.nAdditions * 72, nc4, nc4, nc4, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 15 * sd, npl * 5 * sd, (n + 6) * 2 * z.n8q};
    const Span* sec = z.sec; PlonkLayout& lay = z.lay;
    if (plonk_family_sections(secs, z, want, 14, 13, z.sec, 16, lay, err)) return -1;
    for (int j = 0; j < 3; j++) { lay.s_coef[j] = sub_span(sec[12], 5 * sd * j, sd); lay.s_ev[j] = sub_span(sec[12], 5 * sd * j + sd, 4 * sd); }
    for (uint64_t j = 0; j < npl && j < sec[13].len / (5 * sd); j++) lay.lag.push_back(sub_span(sec[13], 5 * sd * j + sd, 4 * sd));
    lay.ptau = sub_span(sec[14], 0, want[14]);
    return 0;
}

// fflonk (protocol 10): one section per sigma (12-14), the Lagrange polynomials in 15, 9n + 18 PTau points in 16, C0 in 17
inline int fflonk_parse_zkey(const uint8_t* d, uint64_t len, FflonkZkey& z, std::string& err) {
    Sections secs;
    if (plonk_family_header(d, len, 10, "zkey file is not fflonk", 6, 4 + 2, 2, secs, z, err)) return -1;   // fflonk_prove.js:71-73
    z.w3 = z.k2 + 32; z.w4 = z.w3 + 32; z.w8 = z.w4 + 32; z.wr = z.w8 + 32; z.X_2 = z.wr + 32; z.C0 = z.X_2 + 4 * z.n8q;
    const uint64_t n = z.n, sd = n * 32, npl = z.nPublic > 1 ? z.nPublic : 1, nc4 = (uint64_t)z.nConstraints * 4;
    const uint64_t want[18] = {0, 0, 0, (uint64_t)z.nAdditions * 72, nc4, nc4, nc4, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 5 * sd, 5 * sd,
                               npl * 5 * sd, (9 * n + 18) * 2 * z.n8q, 8 * sd};
    const Span* sec = z.sec; PlonkLayout& lay = z.lay;
    if (plonk_family_sections(secs, z, want, 17, -1, z.sec, 20, lay, err)) return -1;
    for (int j = 0; j < 3; j++) { lay.s_coef[j] = sub_span(sec[12 + j], 0, sd); lay.s_ev[j] = sub_span(sec[12 + j], sd, 4 * sd); }
    for (uint64_t j = 0; j < npl; j++) lay.lag.push_back(sub_span(sec[15], 5 * sd * j + sd, 4 * sd));
    lay.ptau = sub_span(sec[16], 0, want[16]);
    lay.c0 = sub_span(sec[17], 0, want[17]);
    return 0;
}

}  // namespace sb
