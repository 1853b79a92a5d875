// field_entry.h — untyped entry points of the field-primitive test kernel (field_eval.cu, field_eval.cuh).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
namespace sb {
// 32-bit words per input / output record of (field, op); -1 if sb_field_eval does not define the pair
int field_eval_shape(int field, int op, int* in_words, int* out_words);
// n records of (field, op): in / out are device pointers
int field_eval(int field, int op, const void* in, void* out, uint64_t n, cudaStream_t stream);
}
