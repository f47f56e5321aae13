// Warp-level tensor-core MMA (mma.sync.m16n8k16, sm_80+): fp16 operands in registers, fp32 accumulators.
#pragma once
#include <stdint.h>
#include <cuda_fp16.h>

namespace o2345 {

// c[16 x 8] += a[16 x 16] . b[16 x 8] (A row-major fragment, B column-major fragment)
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// two floats rounded to one packed half2 operand register (x in the low half)
__device__ __forceinline__ uint32_t pack2(float x, float y) {
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace o2345
