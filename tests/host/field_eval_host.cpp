// CPU driver of sb_field_eval's per-record dispatch (snarkjs_b200/csrc/field_eval.cuh) compiled with g++: the same
// fp.cuh / ec.cuh template code the kernel runs, with the PTX carry chains emulated (-DSB_HOST_EMULATE_PTX) or with the
// host multiply.  Built and run by tests/test_host_field_edges.py.
//   field_eval_host IN OUT: IN is a sequence of blocks {int32 field, int32 op, uint64 n, n input records}; OUT receives the
//   n output records of each block, in order.
#include <cstdio>
#include <vector>
#include "../../snarkjs_b200/csrc/field_eval.cuh"
using namespace sb;

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s IN OUT\n", argv[0]); return 2; }
    FILE* in = fopen(argv[1], "rb");
    FILE* out = fopen(argv[2], "wb");
    if (!in || !out) { fprintf(stderr, "cannot open %s or %s\n", argv[1], argv[2]); return 2; }
    int32_t hdr[2];
    uint64_t n;
    while (fread(hdr, 4, 2, in) == 2) {
        if (fread(&n, 8, 1, in) != 1) { fprintf(stderr, "truncated block header\n"); return 2; }
        const int wi = field_eval_words(hdr[0], hdr[1], false), wo = field_eval_words(hdr[0], hdr[1], true);
        if (!wi) { fprintf(stderr, "op %d is not defined on field %d\n", hdr[1], hdr[0]); return 2; }
        std::vector<uint32_t> a((size_t)n * wi), r((size_t)n * wo);
        if (fread(a.data(), 4, a.size(), in) != a.size()) { fprintf(stderr, "truncated block\n"); return 2; }
        for (uint64_t i = 0; i < n; i++) field_eval_record(hdr[0], hdr[1], a.data() + i * wi, r.data() + i * wo);
        fwrite(r.data(), 4, r.size(), out);
    }
    fclose(out);
    fclose(in);
    return 0;
}
