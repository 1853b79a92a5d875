// field_eval.cu — sb_field_eval's kernel: one thread per record, one instantiation per valid (field, op) pair, so each
// primitive is compiled with the constant-folded dispatch of field_eval.cuh around it and nothing else.
#include "field_eval.cuh"
#include "field_entry.h"
namespace sb {

template <int FIELD, int OP>
__global__ void k_field_eval(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t n) {
    constexpr int wi = field_eval_words(FIELD, OP, false), wo = field_eval_words(FIELD, OP, true);
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    field_eval_record(FIELD, OP, in + i * wi, out + i * wo);
}

template <int FIELD, int OP = 0>
static int launch_op(int op, const void* in, void* out, uint64_t n, cudaStream_t stream) {
    if constexpr (OP == FE_NOPS) {
        return -1;
    } else {
        if (op != OP) return launch_op<FIELD, OP + 1>(op, in, out, n, stream);
        if constexpr (field_eval_words(FIELD, OP, false) == 0) return -1;
        else {
            k_field_eval<FIELD, OP><<<(unsigned)((n + 127) / 128), 128, 0, stream>>>((const uint32_t*)in, (uint32_t*)out, n);
            return (int)cudaGetLastError();
        }
    }
}

int field_eval_shape(int field, int op, int* in_words, int* out_words) {
    *in_words = field_eval_words(field, op, false);
    *out_words = field_eval_words(field, op, true);
    return *in_words ? 0 : -1;
}

int field_eval(int field, int op, const void* in, void* out, uint64_t n, cudaStream_t stream) {
    if (!field_eval_words(field, op, false)) return -1;
    if (!n) return 0;
    switch (field) {
    case FE_BN_FQ: return launch_op<FE_BN_FQ>(op, in, out, n, stream);
    case FE_BN_FR: return launch_op<FE_BN_FR>(op, in, out, n, stream);
    case FE_BLS_FQ: return launch_op<FE_BLS_FQ>(op, in, out, n, stream);
    case FE_BLS_FR: return launch_op<FE_BLS_FR>(op, in, out, n, stream);
    case FE_BN_FQ2: return launch_op<FE_BN_FQ2>(op, in, out, n, stream);
    case FE_BLS_FQ2: return launch_op<FE_BLS_FQ2>(op, in, out, n, stream);
    default: return -1;
    }
}

}  // namespace sb
