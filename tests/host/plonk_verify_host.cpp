// plonk_verify_host.cpp — the per-proof code of the device PLONK / fflonk verifiers (csrc/verify_plonk.cuh: Keccak, checks,
// transcript, PI, scalars, d4 and the pairing inputs) run on the CPU by the same template code, with fp.cuh's host multiply.
// The scalar multiplications the device does with gfft_mul are plain double-and-add here.
//   keccak IN OUT:  IN = blocks of (uint32 len, len bytes); OUT = the 32-byte digests
//   verify IN OUT:  IN = records of (int32 proto 0 PLONK / 1 fflonk, int32 curve 0 BN254 / 1 BLS12-381, uint32 n_public,
//                   uint32 power, vk bytes, G1 generator, G2 generator, Fr.w[power] (Montgomery), n_public plain signals,
//                   one proof); OUT = per record int32 status, the scalar struct (Montgomery Fr values in declaration order)
//                   and, when the status is 0, p1 || p2 affine (Montgomery, all zero = infinity)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../snarkjs_b200/csrc/verify_plonk.cuh"
using namespace sb;

static void rd(FILE* f, void* p, size_t n) { if (n && fread(p, 1, n, f) != n) { fprintf(stderr, "short input\n"); exit(1); } }

template <class F> static XYZZ<F> mul(const XYZZ<F>& p, const FrPlain& k) {
    XYZZ<F> r = XYZZ<F>::inf();
    for (int i = 255; i >= 0; i--) {
        r = XYZZ<F>::dbl(r);
        if ((k.v[i >> 5] >> (i & 31)) & 1) r.add(p);
    }
    return r;
}
template <class F> static void put_affine(FILE* out, const XYZZ<F>& p) {
    F x = F::zero(), y = F::zero();
    if (!p.is_inf()) { const F t = F::inv(p.zzz), u = F::mul(p.zz, t); x = F::mul(p.x, F::sqr(u)); y = F::mul(p.y, t); }
    fwrite(&x, sizeof x, 1, out); fwrite(&y, sizeof y, 1, out);
}

template <class P, class V> static void verify(FILE* in, FILE* out, uint32_t n_public, uint32_t power) {
    typedef Fp<P> F;
    const size_t n8 = sizeof(F);
    const size_t vk_len = V::NT == PvPlonk::NT ? 20 * n8 + 64 : 6 * n8 + 224;
    std::vector<uint8_t> vk(vk_len), g1(2 * n8), g2(4 * n8), wp(32), pub(32 * (size_t)n_public), prf(pv_proof_bytes<P, V>());
    rd(in, vk.data(), vk.size()); rd(in, g1.data(), g1.size()); rd(in, g2.data(), g2.size()); rd(in, wp.data(), 32);
    rd(in, pub.data(), pub.size()); rd(in, prf.data(), prf.size());
    PvKey<P> key;
    if (!pv_key_host<P, V>(vk.data(), n_public, power, g1.data(), g2.data(), wp.data(), key)) { fprintf(stderr, "vk not valid\n"); exit(3); }
    typename V::template Vs<P> o;
    memset(&o, 0, sizeof o);
    const int32_t st = V::template scalars<P>(key, prf.data(), (const FrPlain*)pub.data(), o);
    fwrite(&st, 4, 1, out);
    fwrite(&o, sizeof o, 1, out);
    if (st) return;
    std::vector<XYZZ<F>> t(V::NT);
    for (int j = 0; j < V::NT; j++) {
        const int b = V::base(j);
        const F* src = b == PV_GEN ? key.g1 : b >= PV_PRF ? (const F*)prf.data() + 2 * (b - PV_PRF) : key.pt + 2 * b;
        t[j] = mul(pv_affine(src[0], src[1]), fr_plain<P>(o.s[j]));
    }
    if constexpr (V::NT == PvPlonk::NT) plonk_d4<P>(prf.data(), t.data(), fr_plain<P>(o.s[17]), [](const XYZZ<F>& p, const FrPlain& s) { return mul(p, s); });
    XYZZ<F> p1, p2;
    pv_inputs<P, V>(key, prf.data(), t.data(), p1, p2);
    put_affine(out, p1); put_affine(out, p2);
}

int main(int argc, char** argv) {
    if (argc != 4) { fprintf(stderr, "usage: %s keccak|verify in.bin out.bin\n", argv[0]); return 1; }
    FILE* in = fopen(argv[2], "rb"); FILE* out = fopen(argv[3], "wb");
    if (!in || !out) { perror("open"); return 1; }
    if (!strcmp(argv[1], "keccak")) {
        uint32_t len;
        while (fread(&len, 4, 1, in) == 1) {
            std::vector<uint8_t> m(len);
            rd(in, m.data(), len);
            Keccak256 h; h.reset();
            for (uint8_t b : m) h.byte(b);
            uint8_t d[32]; h.finish(d);
            fwrite(d, 1, 32, out);
        }
    } else {
        struct { int32_t proto, curve; uint32_t n_public, power; } h;
        while (fread(&h, sizeof h, 1, in) == 1) {
            if (h.proto == 0 && h.curve == 0) verify<BnFq, PvPlonk>(in, out, h.n_public, h.power);
            else if (h.proto == 0 && h.curve == 1) verify<BlsFq, PvPlonk>(in, out, h.n_public, h.power);
            else if (h.proto == 1 && h.curve == 0) verify<BnFq, PvFflonk>(in, out, h.n_public, h.power);
            else { fprintf(stderr, "proto %d is not defined on curve %d\n", h.proto, h.curve); return 2; }
        }
    }
    fclose(out);
    return 0;
}
