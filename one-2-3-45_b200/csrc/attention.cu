// Fused multi-head self-attention for the UNet's spatial transformers (SURVEY.md row A4): softmax(Q K^T * scale) V in one
// kernel, scores never leave the SM.  Replaces reference ldm/modules/attention.py:170-193, which materialises the
// [(b h), N, N] score tensor (134 MB per layer at N = 1024) three times; the three-kernel route (batched GEMM -> softmax
// -> batched GEMM) runs 4096 one-k-block CTAs for QK^T alone.
//
// Head dims are 40 / 80 / 160 and sequences 16..1024 tokens: far too small per (batch, head) to fill a 128-row GEMM tile
// pipeline, so this kernel uses warp-level mma.sync.m16n8k16 (fp16 in, fp32 accumulate) in the FlashAttention-2
// arrangement: one CTA = 4 warps = 64 queries of one (b, h); K / V stream through a two-stage cp.async ring of 64-key tiles (both row-major;
// the P V operand comes out of ldmatrix.trans); online softmax in fp32 registers with exp2; the S
// accumulator fragments are re-used in place as the A fragments of the P V product.  The arithmetic is softmax-bound
// (N^2 exps per head), not tensor-bound, at these sizes.
#include <cuda_fp16.h>

#include <cmath>

#include "common.cuh"
#include "mma_sync.cuh"

namespace o2345 {
namespace {

// 2^x on the SFU (ex2.approx: 2 ulp; the probabilities are rounded to fp16 for the P V product right after)
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int KT = 64;  // keys per tile

// D: head dim, DP: its padding to a multiple of 16, NW: warps per CTA = 16 queries each (8 warps share one K / V stream for
// 128 queries: half the shared-memory fills per query of the 4-warp version, used for long sequences)
template <int D, int DP, int NW>
__global__ void __launch_bounds__(32 * NW)
attention_kernel(const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v, int N, int H, int ld,
                 __half* __restrict__ out, int ldo, float scale_log2) {
  pdl_wait();
  pdl_trigger();
  constexpr int QT = 16 * NW, NT = 32 * NW;
  constexpr int LDQ = DP + 8, KS = DP / 16, NO = DP / 8;
  constexpr int STAGE = 2 * KT * LDQ;      // halves per K + V stage
  extern __shared__ __align__(16) __half smem_h[];
  __half* sQ = smem_h;
  __half* sKV = sQ + QT * LDQ;             // two stages of [K tile | V tile], both row-major [key][d]; the P V operand is read with ldmatrix.trans
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / H, h = bh % H;
  const int q0 = blockIdx.x * QT;
  const int64_t base = (int64_t)b * N * ld + (int64_t)h * D;
  constexpr int CH = D / 8;  // 16-byte chunks per row

  // K / V tiles stream through a two-stage cp.async ring: tile i + 1 is in flight while tile i is multiplied (round 1 loaded
  // each tile synchronously between two __syncthreads: the kernel sat at ~1/7 of its issue-bound time waiting for L2).
  // Rows past N: K garbage is masked after the product; V must be finite (0 * NaN), so its copy zero-fills (src-size 0).
  auto load_tile = [&](int stage, int k0) {
    __half* dK = sKV + stage * STAGE;
    __half* dV = dK + KT * LDQ;
    for (int i = tid; i < KT * CH; i += NT) {
      const int r = i / CH, c = i % CH;
      const bool in = k0 + r < N;
      const int64_t off = base + (int64_t)(in ? k0 + r : 0) * ld + 8 * c;
      const uint32_t ak = (uint32_t)__cvta_generic_to_shared(dK + r * LDQ + 8 * c), av = (uint32_t)__cvta_generic_to_shared(dV + r * LDQ + 8 * c);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ak), "l"(k + off) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(av), "l"(v + off), "r"(in ? 16 : 0) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  // zero Q's and both stages' padding columns d..DP-1 (the copies only touch the first d columns), then Q
  for (int i = tid; i < (QT * LDQ + 2 * STAGE) / 8; i += NT) reinterpret_cast<uint4*>(sQ)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  load_tile(0, 0);
  for (int i = tid; i < QT * CH; i += NT) {
    int r = i / CH, c = i % CH;
    if (q0 + r < N) *reinterpret_cast<uint4*>(sQ + r * LDQ + 8 * c) = *reinterpret_cast<const uint4*>(q + base + (int64_t)(q0 + r) * ld + 8 * c);
  }
  __syncthreads();
  uint32_t qa[KS][4];
#pragma unroll
  for (int kk = 0; kk < KS; ++kk) {
    const __half* p0 = sQ + (16 * warp + g) * LDQ + 16 * kk + 2 * t;
    qa[kk][0] = *reinterpret_cast<const uint32_t*>(p0);
    qa[kk][1] = *reinterpret_cast<const uint32_t*>(p0 + 8 * LDQ);
    qa[kk][2] = *reinterpret_cast<const uint32_t*>(p0 + 8);
    qa[kk][3] = *reinterpret_cast<const uint32_t*>(p0 + 8 * LDQ + 8);
  }
  float o[NO][4];
#pragma unroll
  for (int n = 0; n < NO; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m0 = -1e30f, m1 = -1e30f;
  float ls[4] = {0.f, 0.f, 0.f, 0.f};     // running row sums (rows g, g + 8), accumulated by the tensor cores

  int it = 0;
  for (int k0 = 0; k0 < N; k0 += KT, ++it) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");   // tile `it` has landed (it is the only group in flight here)
    __syncthreads();                                        // ... for every thread, and tile it - 1 is fully consumed
    if (k0 + KT < N) load_tile((it + 1) & 1, k0 + KT);      // overwrites the stage tile it - 1 used
    const __half* sK = sKV + (it & 1) * STAGE;
    const __half* sV = sK + KT * LDQ;
    // ---- S = Q K^T for this warp's 16 queries x 64 keys
    float s[KT / 8][4];
#pragma unroll
    for (int j = 0; j < KT / 8; j += 2) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      s[j + 1][0] = s[j + 1][1] = s[j + 1][2] = s[j + 1][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        // one ldmatrix.x4 = the B fragments of two MMAs: matrices (keys 8j.., d 16kk..), (8j.., 16kk+8..), (8j+8.., 16kk..),
        // (8j+8.., 16kk+8..); lane l supplies the row address of matrix l / 8, row l % 8
        uint32_t b0, b1, b2, b3;
        const uint32_t addr = (uint32_t)__cvta_generic_to_shared(sK + (8 * j + 8 * (lane >> 4) + (lane & 7)) * LDQ + 16 * kk + 8 * ((lane >> 3) & 1));
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "r"(addr));
        mma16816(s[j], qa[kk], b0, b1);
        mma16816(s[j + 1], qa[kk], b2, b3);
      }
    }
    // ---- online softmax (rows g and g+8 of this warp's tile).  The running maximum is kept on the RAW scores; the scale
    // (softmax scale x log2 e, > 0) is folded into the exponent: p = 2^(s * c - m * c) is one FFMA + one ex2 per score (round 2
    // first scaled every score, then subtracted: two instructions more per score in the loop that bounds this kernel).  Keys
    // past N only exist in the last tile: the masking compare / select runs there only.
    if (k0 + KT > N) {
#pragma unroll
      for (int j = 0; j < KT / 8; ++j) {
        const int key = k0 + 8 * j + 2 * t;
        if (key >= N) s[j][0] = -1e30f, s[j][2] = -1e30f;
        if (key + 1 >= N) s[j][1] = -1e30f, s[j][3] = -1e30f;
      }
    }
    float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)), mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)), mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float a0 = ex2((m0 - mn0) * scale_log2), a1 = ex2((m1 - mn1) * scale_log2);
    m0 = mn0, m1 = mn1;
    const float ms0 = -mn0 * scale_log2, ms1 = -mn1 * scale_log2;
#pragma unroll
    for (int n = 0; n < NO; ++n) o[n][0] *= a0, o[n][1] *= a0, o[n][2] *= a1, o[n][3] *= a1;
    ls[0] *= a0, ls[1] *= a0, ls[2] *= a1, ls[3] *= a1;
    // ---- P = 2^(s c - m c), rounded to fp16 into the A fragments of the next product (the S fragments' positions ARE those
    // fragments' positions); O += P V, and the row sums l += P 1 on the tensor cores too (a B fragment of ones: four MMAs
    // per tile instead of 32 FADDs per lane and the final cross-lane reduction, and the denominator sums the same rounded
    // probabilities the numerator uses).  (ex2.approx.f16x2 on packed pairs was tried: it compiles to two MUFU.EX2.F16, no saving.)
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk) {
      const uint32_t pa[4] = {pack2(ex2(fmaf(s[2 * kk][0], scale_log2, ms0)), ex2(fmaf(s[2 * kk][1], scale_log2, ms0))),
                              pack2(ex2(fmaf(s[2 * kk][2], scale_log2, ms1)), ex2(fmaf(s[2 * kk][3], scale_log2, ms1))),
                              pack2(ex2(fmaf(s[2 * kk + 1][0], scale_log2, ms0)), ex2(fmaf(s[2 * kk + 1][1], scale_log2, ms0))),
                              pack2(ex2(fmaf(s[2 * kk + 1][2], scale_log2, ms1)), ex2(fmaf(s[2 * kk + 1][3], scale_log2, ms1)))};
      mma16816(ls, pa, 0x3C003C00u, 0x3C003C00u);
#pragma unroll
      for (int n = 0; n < NO; ++n) {
        // B fragment of P V: keys 16 kk .. +15 (k) x head dims 8 n .. +7 (n) out of the row-major V tile
        uint32_t b0, b1;
        const uint32_t addr = (uint32_t)__cvta_generic_to_shared(sV + (16 * kk + (lane & 15)) * LDQ + 8 * n);
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(addr));
        mma16816(o[n], pa, b0, b1);
      }
    }
  }
  const float l0 = ls[0], l1 = ls[2];   // every column of the ones product holds the row sum: no cross-lane reduction needed
  float i0 = 1.f / l0, i1 = 1.f / l1;
  int row0 = q0 + 16 * warp + g, row1 = row0 + 8;
#pragma unroll
  for (int n = 0; n < NO; ++n) {
    int col = 8 * n + 2 * t;
    if (col < D) {
      if (row0 < N) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * N + row0) * ldo + h * D + col) = pack2(o[n][0] * i0, o[n][1] * i0);
      if (row1 < N) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * N + row1) * ldo + h * D + col) = pack2(o[n][2] * i1, o[n][3] * i1);
    }
  }
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int o2345_attention_f16(const void* q, const void* k, const void* v, int B, int N, int H, int d, int ld, void* out,
                                   int ldo, float scale, o2345_stream_t stream) {
  O2345_CHECK_ARG(q && k && v && out, "null pointer");
  O2345_CHECK_ARG(B > 0 && N > 0 && H > 0 && (ld % 8) == 0 && (ldo % 2) == 0, "bad sizes");
  O2345_CHECK_ARG(d == 40 || d == 64 || d == 80 || d == 160, "head dim must be 40, 64, 80 or 160");
  O2345_CHECK_ARG(((uintptr_t)q % 16) == 0 && ((uintptr_t)k % 16) == 0 && ((uintptr_t)v % 16) == 0, "q/k/v must be 16-byte aligned");
  // the running maximum is taken on the raw scores, with the scale folded into the exponent: right only for scale > 0
  O2345_CHECK_ARG(scale > 0.f && std::isfinite(scale), "scale must be positive and finite");
  const int nw = N >= 512 ? 8 : 4;               // 128 queries per CTA on long sequences
  dim3 grid(cdiv(N, 16 * nw), B * H);
  float sl2 = scale * 1.4426950408889634f;
  cudaStream_t st = (cudaStream_t)stream;
  const __half *qh = (const __half*)q, *kh = (const __half*)k, *vh = (const __half*)v;
  auto smem = [&](int dp) { return (size_t)((16 * nw + 4 * KT) * (dp + 8)) * sizeof(__half); };   // Q + two stages of K and V
  static PerDeviceOnce attr;
  if (attr.need()) {
    O2345_CUDA(cudaFuncSetAttribute(attention_kernel<160, 160, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((64 + 4 * KT) * 168 * 2)));
    O2345_CUDA(cudaFuncSetAttribute(attention_kernel<160, 160, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((128 + 4 * KT) * 168 * 2)));
    O2345_CUDA(cudaFuncSetAttribute(attention_kernel<80, 80, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((64 + 4 * KT) * 88 * 2)));
    O2345_CUDA(cudaFuncSetAttribute(attention_kernel<80, 80, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((128 + 4 * KT) * 88 * 2)));
    O2345_CUDA(cudaFuncSetAttribute(attention_kernel<64, 64, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((128 + 4 * KT) * 72 * 2)));
  }
#define O2345_ATT(D_, DP_)                                                                                                        \
  do {                                                                                                                            \
    if (nw == 8)                                                                                                                  \
      O2345_CUDA(launch_pdl(attention_kernel<D_, DP_, 8>, dim3(grid), dim3(256), smem(DP_), st, qh, kh, vh, N, H, ld, (__half*)out, \
                            ldo, sl2));                                                                                           \
    else                                                                                                                          \
      O2345_CUDA(launch_pdl(attention_kernel<D_, DP_, 4>, dim3(grid), dim3(128), smem(DP_), st, qh, kh, vh, N, H, ld, (__half*)out, \
                            ldo, sl2));                                                                                           \
  } while (0)
  if (d == 40) O2345_ATT(40, 48);
  else if (d == 64) O2345_ATT(64, 64);
  else if (d == 80) O2345_ATT(80, 80);
  else if (d == 160) O2345_ATT(160, 160);
  else { set_error("o2345_attention_f16: head dim %d not built (40 / 64 / 80 / 160)", d); return O2345_EUNSUPPORTED; }
#undef O2345_ATT
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
