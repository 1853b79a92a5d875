// pairing_eval_host.cpp — the records of sb_pairing_eval (csrc/pairing.cuh, pair_eval_record) computed on the CPU by the same
// template code, with fp.cuh's host multiply.  Input file: blocks of (int32 curve, int32 op, uint64 n, n input records);
// output file: the n output records of every block, back to back.  Curve 0 = BN254, 1 = BLS12-381.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../snarkjs_b200/csrc/pairing.cuh"

template <class P> static bool run(FILE* in, FILE* out, int op, uint64_t n) {
    int wi, wo;
    if (!sb::pair_eval_shape(op, &wi, &wo)) return false;
    std::vector<sb::Fp<P>> a(wi), r(wo);
    for (uint64_t k = 0; k < n; k++) {
        if (fread(a.data(), sizeof(sb::Fp<P>), wi, in) != (size_t)wi) { fprintf(stderr, "short input\n"); exit(1); }
        sb::pair_eval_record<P>(op, a.data(), r.data());
        fwrite(r.data(), sizeof(sb::Fp<P>), wo, out);
    }
    return true;
}

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 1; }
    FILE* in = fopen(argv[1], "rb"); FILE* out = fopen(argv[2], "wb");
    if (!in || !out) { perror("open"); return 1; }
    struct { int32_t curve, op; uint64_t n; } h;
    while (fread(&h, sizeof h, 1, in) == 1) {
        const bool ok = h.curve == 0 ? run<sb::BnFq>(in, out, h.op, h.n) : h.curve == 1 ? run<sb::BlsFq>(in, out, h.op, h.n) : false;
        if (!ok) { fprintf(stderr, "op %d is not defined on curve %d\n", h.op, h.curve); return 2; }
    }
    fclose(out);
    return 0;
}
