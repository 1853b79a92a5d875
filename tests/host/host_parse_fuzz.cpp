// Mutation fuzzing of the container parsers of zkey.h (plonk_parse_zkey, fflonk_parse_zkey, groth16_parse_zkey,
// wtns_parse) and of the host-side load logic that consumes their output (plonk_addition_levels), built with
// -fsanitize=address,undefined by tests/test_host_templates.py.  Every mutated container must either be rejected with a
// message or be accepted with every span and CSR entry the parser returned staying inside the buffer; the sanitizers turn
// an out-of-bounds read or an overflowed size into a crash.  The buffer handed to the parser is an exact-size heap block,
// so reading one byte past the file is detected.   usage: host_parse_fuzz plonk|fflonk|groth16|wtns <file> <iterations>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include "../../snarkjs_b200/csrc/fflonk_flow.h"
using namespace sb;

static uint64_t st = 0x243F6A8885A308D3ull;
static uint64_t rnd() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; }
static volatile uint64_t sink;
static void touch(const uint8_t* p, uint64_t len) { uint64_t s = 0; for (uint64_t i = 0; i < len; i += 97) s += p[i]; if (len) s += p[len - 1]; sink += s; }

static void touch(const Span& s) { touch(s.p, s.len); }

// every span the parser returned, with host reads in place of the loaders' uploads
static void consume(const PlonkHeader& z, const PlonkLayout& lay) {
    touch(z.header); touch(z.q, z.n8q); touch(z.r, z.n8r); touch(z.k1, 32); touch(z.k2, 32);
    const uint32_t na = z.nAdditions;
    std::vector<uint32_t> sig(2 * (size_t)na + 2), order, level_end;
    for (uint32_t i = 0; i < na; i++) { memcpy(&sig[2 * (size_t)i], lay.additions.p + 72 * (size_t)i, 8); touch(lay.additions.p + 72 * (size_t)i + 8, 64); }
    plonk_addition_levels(sig.data(), na, z.nVars - na, order, level_end);
    uint64_t tot = 0; for (uint32_t e : level_end) tot = e;
    if (na && tot != na) { fprintf(stderr, "addition levels do not cover all additions\n"); abort(); }
    for (uint32_t o : order) if (o >= na) { fprintf(stderr, "addition order out of range\n"); abort(); }
    for (const Span& s : lay.maps) touch(s);
    for (int j = 0; j < 5; j++) { touch(lay.q_coef[j]); touch(lay.q_ev[j]); }
    for (int j = 0; j < 3; j++) { touch(lay.s_coef[j]); touch(lay.s_ev[j]); }
    for (const Span& s : lay.lag) touch(s);
    touch(lay.ptau); touch(lay.c0);
}
static void consume(const Groth16Zkey& z) {
    touch(z.q, z.n8q); touch(z.r, z.n8r);
    for (const uint8_t* p : {z.alpha1, z.beta1, z.delta1}) touch(p, 2 * (uint64_t)z.n8q);
    for (const uint8_t* p : {z.beta2, z.gamma2, z.delta2}) touch(p, 4 * (uint64_t)z.n8q);
    for (const Span& s : {z.A, z.B1, z.B2, z.C, z.H}) touch(s);
    if (z.rowptr.size() != 2 * (uint64_t)z.domainSize + 1 || z.rowptr.back() != z.sig.size() || z.coef.size() != 32 * z.sig.size()) { fprintf(stderr, "CSR shape\n"); abort(); }
    for (size_t i = 0; i + 1 < z.rowptr.size(); i++) if (z.rowptr[i] > z.rowptr[i + 1]) { fprintf(stderr, "CSR row pointers not monotone\n"); abort(); }
    for (uint32_t s : z.sig) if (s >= z.nVars) { fprintf(stderr, "CSR signal out of range\n"); abort(); }
    touch(z.coef.data(), z.coef.size());
}

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    const std::string proto = argv[1];
    if (proto != "plonk" && proto != "fflonk" && proto != "groth16" && proto != "wtns") return 2;
    std::ifstream f(argv[2], std::ios::binary);
    std::vector<uint8_t> good((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const long iters = atol(argv[3]);
    if (good.size() < 64) { fprintf(stderr, "cannot read %s\n", argv[2]); return 2; }
    long accepted = 0, rejected = 0;
    for (long it = 0; it <= iters; it++) {
        uint64_t len = good.size();
        const int mode = it == 0 ? -1 : (int)(rnd() % 6);
        if (mode == 0) len = rnd() % (good.size() + 1);                       // truncation
        uint8_t* buf = (uint8_t*)malloc(len ? len : 1);                         // exact size: ASan sees any overrun
        memcpy(buf, good.data(), len);
        if (len >= 64) {
            if (mode == 1) for (int k = 0; k < 1 + (int)(rnd() % 4); k++) buf[rnd() % std::min<uint64_t>(len, 2048)] ^= (uint8_t)(1u << (rnd() % 8));   // bit flips in the headers / section table
            if (mode == 2) { uint64_t p = rnd() % std::min<uint64_t>(len - 8, 4096); uint64_t v = rnd() % 3 == 0 ? ~0ull - (rnd() % 64) : (rnd() % 2 ? rnd() : rnd() % (2 * len)); memcpy(buf + p, &v, 8); }   // a wild 64-bit field
            if (mode == 3) { uint64_t p = rnd() % std::min<uint64_t>(len - 4, 4096); uint32_t v = rnd() % 2 ? (uint32_t)rnd() : (uint32_t)(rnd() % 64); memcpy(buf + p, &v, 4); }       // a wild 32-bit field (counts, sizes)
            if (mode == 4) for (int k = 0; k < 16; k++) { uint64_t p = rnd() % (len - 4); uint32_t v = (uint32_t)rnd(); memcpy(buf + p, &v, 4); }                                      // garbage anywhere (signal ids, maps)
            if (mode == 5) { uint64_t p = 12 + rnd() % std::min<uint64_t>(len - 12, 600); memset(buf + p, rnd() % 2 ? 0xff : 0, std::min<uint64_t>(12, len - p)); }                   // a smashed section header
        }
        std::string err; int rc;
        if (proto == "plonk") { PlonkZkey z; rc = plonk_parse_zkey(buf, len, z, err); if (!rc) { consume(z, z.lay); touch(z.hdr_pts, 16 * (uint64_t)z.n8q); touch(z.X_2, 4 * (uint64_t)z.n8q); } }
        else if (proto == "fflonk") {
            FflonkZkey z; rc = fflonk_parse_zkey(buf, len, z, err);
            if (!rc) { consume(z, z.lay); for (const uint8_t* p : {z.w3, z.w4, z.w8, z.wr}) touch(p, 32); touch(z.X_2, 4 * (uint64_t)z.n8q); touch(z.C0, 2 * (uint64_t)z.n8q); fflonk_c0_is_interleave(z); }
        }
        else if (proto == "groth16") { Groth16Zkey z; rc = groth16_parse_zkey(buf, len, z, err); if (!rc) consume(z); }
        else { Wtns w; rc = wtns_parse(buf, len, w, err); if (!rc) { touch(w.q, w.n8); touch(w.values); } }
        free(buf);
        if (rc) { if (err.empty()) { fprintf(stderr, "rejected without a message (iteration %ld)\n", it); return 1; } rejected++; }
        else accepted++;
        if (it == 0 && rc) { fprintf(stderr, "the unmodified key was rejected: %s\n", err.c_str()); return 1; }
    }
    printf("FUZZ OK %s: %ld accepted, %ld rejected\n", argv[1], accepted, rejected);
    return 0;
}
