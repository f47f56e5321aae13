// fp16 GEMM on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers), operands fed by TMA.
// Path A of SURVEY.md section 8 (rows A2-A4, A6, A8): every Linear / 1x1 conv / 3x3 conv of the Zero123 UNet, the VAE and
// the CLIP tower, and the QK^T / PV products of the unfused attention fallback, go through this file.
//
//   C[M,N] = epilogue( alpha * A[M,K] . B[N,K]^T + bias[N] + rowbias[row / rpg, N] ) (+ residual[M,N])   fp16 in, fp32 acc
//
// A and B are both K-major (row-major activations [rows, K]; nn.Linear / flattened conv weights [N, K]).
//
// ONE kernel template, gemm_tc_kernel<BN, STAGES, MODE>: a CTA computes a 128 x BN tile.
// Warp roles (384 threads = three warpgroups, one CTA per SM):
//   warpgroup 0   one thread is the TMA producer: cp.async.bulk.tensor (SWIZZLE_128B) into a STAGES-deep shared-memory ring
//                 guarded by full / empty mbarriers;
//   warpgroups 1-2  each issues wgmma.mma_async m64nBNk16 on its 64 rows of the tile, four per stage, one stage in flight
//                 while the previous one is released; once the K loop is done the (now idle) operand ring receives the fp32
//                 accumulator tile, and the same EIGHT warps run the epilogue: warp w owns 32 rows and one of two column
//                 ranges of the tile; alpha / bias / activation / GEGLU gate -> fp16 -> a shared-memory transpose ->
//                 coalesced row stores with the residual added.
// MODE selects the epilogue at compile time:
//   0 staged, no activation   1 staged, GEGLU gate   2 staged, SiLU / GELU / QuickGELU (runtime switch per tile)
//   3 generic (fp32 output, batched, unaligned N) and SPLIT-K.
// Split-K (tiles alone cannot fill 132 SMs): the `splits` CTAs of a tile are launched as ONE thread-block cluster
// (1, 1, splits), so the hardware co-schedules them.  Each stores its partial accumulator into its own fp32 plane of the
// workspace, a cluster barrier (release / acquire) publishes the planes, and every split then sums the planes and applies
// the epilogue to ITS share of the tile.  No atomics, no tickets, no zero-initialised scratch, no second kernel.
// Every mbarrier wait is bounded in TIME (4 s): a protocol bug or a lost arrival records which barrier of which CTA of
// which problem stalled in a host-visible buffer (o2345_last_trap) and traps, instead of spinning for tens of minutes.
#include <cuda.h>
#include <stdlib.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace o2345 {
namespace {

constexpr int BM = 128, BK = 64;
constexpr int EPI_WARPS = 8;
constexpr int EPI_THREADS = 32 * EPI_WARPS;
constexpr int GEMM_THREADS = 128 + EPI_THREADS;
constexpr uint64_t WAIT_LIMIT_NS = 4000000000ull;   // bounded waits: a protocol bug traps (with a record) instead of hanging the GPU
constexpr int MAX_CLUSTER = 8;                      // splits: one cluster per tile (8 = the portable cluster size)
constexpr int RES_PREFETCH = 8;                     // 16-byte residual pieces per lane fetched before the accumulator is read

enum { WAIT_EMPTY = 1, WAIT_FULL = 2 };   // which wait timed out (o2345_last_trap)

struct TrapRecord {
  unsigned long long magic;
  int tag, stage, bx, by, bz, rank, M, N, K, bn, mode, splits, conv;
};
constexpr unsigned long long TRAP_MAGIC = 0x6f32333435545250ull;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done;
}
__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // the eight MMA / epilogue warps only

// the accumulator tile in shared memory: fp32 [128][BN + 4] (the pad spreads the row-per-thread reads over the banks)
__host__ __device__ constexpr int acc_ld(int bn) { return bn + 4; }
// 32 consecutive accumulator columns of one row
__device__ __forceinline__ void acc_ld32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x), r[4 * i + 1] = __float_as_uint(v.y), r[4 * i + 2] = __float_as_uint(v.z), r[4 * i + 3] = __float_as_uint(v.w);
  }
}

struct GemmParams {
  int M, N, K;
  int64_t ldc;                 // elements between consecutive rows of C / residual
  int nh;                      // batched mode: blockIdx.z = b * nh + h
  int64_t stride_c_h, stride_c_b;  // element offsets of C (and residual) per inner / outer batch index
  const float* bias;           // [N] or nullptr
  const __half* rowbias;       // [groups, rowbias_ld] or nullptr: added before the activation, group = row / rows_per_group
  int64_t rowbias_ld;
  int rows_per_group;
  const __half* residual;      // [M, ldc] or nullptr, added after the activation
  void* C;
  int out_f32;                 // 0: fp16 output, 1: fp32 output
  int act;                     // 0 none, 1 SiLU, 2 GELU(erf), 4 QuickGELU x sigmoid(1.702 x), 3 GEGLU: columns come in chunks of 32 = 16 values + their 16 gates,
                               //    out[:, 16 j + e] = v_e * gelu(g_e); C has N / 2 columns
  float alpha;                 // scale applied to the accumulator before bias
  int batched;                 // 4-D tensor maps (K, rows, h, b)
  // implicit 3x3 convolution (stride 1, zero padding 1): A is the channel-last activation [B, H, W, C] seen through a
  // 4-D tensor map (C, W, H, B); an output tile of 128 consecutive pixels is a box (64 ch, tw, th, tb), and kernel tap
  // (ky, kx) is the same box shifted by (kx-1, ky-1) -- TMA's out-of-bounds zero fill IS the convolution padding.
  int conv, cC, cH, cW, cblocks;
  // tap geometry: ctaps taps in rows of ctx, tap j reads the box shifted by (j % ctx + cox, j / ctx + coy).  3 x 3 / pad 1: ctaps 9,
  // ctx 3, cox = coy = -1.  Nearest-neighbour 2x up-sampling followed by a 3 x 3 convolution is FOUR 2 x 2 convolutions of the
  // low-resolution input, one per output phase (a, b) = (row parity, column parity): ctaps 4, ctx 2, cox = b - 1, coy = a - 1,
  // weights pre-summed on the host (rows that collapse onto the same input pixel), and the tile's 128 low-resolution pixels
  // are written to output pixels (2 y + a, 2 x + b): up = 1, upa = a, upb = b.  No im2col buffer, 4 C instead of 9 C per output.
  int ctaps, ctx, cox, coy, up, upa, upb;
  // split-K: the splits of a tile form one cluster; CTA z stores its partial accumulator in plane z of ws [splits, M, N],
  // the cluster barrier publishes the planes, then every split sums and finishes its share of the tile.
  int splits;
  float* ws;
  int persist;                 // 1: a grid of at most one CTA per SM walks the tiles (staged epilogues only)
  long long* trace;            // diagnostic: CTA (0,0,0) stores clock64() stamps of its phases (o2345_debug_gemm_trace), else nullptr
  TrapRecord* diag;            // host-mapped record written before a bounded wait traps (may be nullptr)
  int bn, mode;                // for the trap record
};

__device__ __forceinline__ void stamp(const GemmParams& p, int slot) {
  if (p.trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) p.trace[slot] = clock64();
}
// wall-clock (globaltimer, ns) stamps of tile (0,0): comparable across the SMs the splits of a tile run on
__device__ __forceinline__ void stamp_ns(const GemmParams& p, int slot, bool any_z = false) {
  if (p.trace && blockIdx.x == 0 && blockIdx.y == 0 && (any_z || blockIdx.z == 0)) p.trace[slot] = (long long)global_ns();
}

// row of C that accumulator row `row` is written to (up-sampling phases scatter the low-resolution pixels over the 2x grid)
__device__ __forceinline__ int64_t out_row(const GemmParams& p, int row) {
  if (!p.up) return row;
  const int x = row % p.cW, t = row / p.cW, y = t % p.cH, b = t / p.cH;
  return ((int64_t)b * (2 * p.cH) + 2 * y + p.upa) * (2 * p.cW) + 2 * x + p.upb;
}

__device__ __noinline__ void wait_timed_out(const GemmParams& p, int tag, int stage) {
  if (p.diag) {
    TrapRecord* d = p.diag;
    d->tag = tag, d->stage = stage, d->bx = blockIdx.x, d->by = blockIdx.y, d->bz = blockIdx.z, d->rank = (int)cluster_ctarank();
    d->M = p.M, d->N = p.N, d->K = p.K, d->bn = p.bn, d->mode = p.mode, d->splits = p.splits, d->conv = p.conv;
    __threadfence_system();
    d->magic = TRAP_MAGIC;
    __threadfence_system();
  }
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, const GemmParams& p, int tag, int stage) {
  if (mbar_try(bar, parity)) return;
  const uint64_t t0 = global_ns();
  uint32_t spins = 0;
  while (!mbar_try(bar, parity))
    if (((++spins) & 255u) == 0 && global_ns() - t0 > WAIT_LIMIT_NS) wait_timed_out(p, tag, stage);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// GELU(erf) for the GEGLU gate of the staged epilogue, whose result is rounded to fp16 (2^-11 relative) right away: erf by
// Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7 absolute, ~3e-7 with ex2.approx), 14 instructions instead of erff's ~30 with
// range branches -- the GEGLU projections (8192 x 2560 x 320 ...) are bound by the epilogue's ALU work, not by the MMAs.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  const float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.f);
  return 0.5f * x * (1.f + copysignf(erf_abs, x));
}
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return x / (1.f + __expf(-x));
  if (act == 2) return gelu_erf(x);
  if (act == 4) return x / (1.f + __expf(-1.702f * x));   // QuickGELU (CLIP)
  return x;
}

__device__ __forceinline__ void store8(const GemmParams& p, int64_t off, const float (&v)[8]) {
  if (p.out_f32) {
    float* o = reinterpret_cast<float*>(p.C) + off;
    *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    __half2 h[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.C) + off) = *reinterpret_cast<uint4*>(h);
  }
}

// Generic epilogue (MODE 3, one pass): one thread's 32 consecutive accumulator columns [col0, col0 + 32) of output row
// `row` (crow = element offset of the row in C / residual), stored straight from registers.
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const uint32_t (&r)[32], int row, int64_t crow, int col0) {
  const __half* rb = p.rowbias ? p.rowbias + (int64_t)(row / p.rows_per_group) * p.rowbias_ld : nullptr;
  if (p.act == 3) {  // GEGLU: 16 values then their 16 gates; N is a multiple of 32 (checked on the host)
    if (col0 >= p.N) return;
    float v[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      float a = __uint_as_float(r[e]) * p.alpha, g = __uint_as_float(r[16 + e]) * p.alpha;
      if (p.bias) a += __ldg(p.bias + col0 + e), g += __ldg(p.bias + col0 + 16 + e);
      v[e] = a * gelu_erf(g);
    }
    const int64_t o = crow + (col0 >> 1);
    float lo[8], hi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) lo[e] = v[e], hi[e] = v[8 + e];
    store8(p, o, lo);
    store8(p, o + 8, hi);
    return;
  }
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int col = col0 + j;
    if (col >= p.N) break;
    float v[8];
    const bool full = col + 8 <= p.N;
    if (full && rb) {
      uint4 q = *reinterpret_cast<const uint4*>(rb + col);
      const __half* h = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = __half2float(h[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = (rb && col + e < p.N) ? __half2float(rb[col + e]) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float x = fmaf(__uint_as_float(r[j + e]), p.alpha, v[e]);
      if (p.bias && col + e < p.N) x += __ldg(p.bias + col + e);
      v[e] = apply_act(x, p.act);
    }
    if (full && (p.ldc & 7) == 0) {
      if (p.residual) {
        uint4 q = *reinterpret_cast<const uint4*>(p.residual + crow + col);
        const __half* h = reinterpret_cast<const __half*>(&q);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] += __half2float(h[e]);
      }
      store8(p, crow + col, v);
    } else {
      for (int e = 0; e < 8 && col + e < p.N; ++e) {
        float x = v[e];
        if (p.residual) x += __half2float(p.residual[crow + col + e]);
        if (p.out_f32) reinterpret_cast<float*>(p.C)[crow + col + e] = x;
        else reinterpret_cast<__half*>(p.C)[crow + col + e] = __float2half_rn(x);
      }
    }
  }
}

// split-K, every CTA: one thread's 32 accumulator columns of one row go to THIS split's private fp32 partial plane
// ws[split][M][N] with plain vector stores (round 1 and the first round-2 version added into one shared plane with
// red.global.add.f32: the L2 atomic units sustain only ~90 G elements/s, 35-60 us for a 2 M element output)
__device__ __forceinline__ void splitk_partial(const GemmParams& p, const uint32_t (&r)[32], int split, int row, int col0) {
  float* w = p.ws + ((int64_t)split * p.M + row) * p.N + col0;
  if ((p.N & 3) == 0) {
#pragma unroll
    for (int e = 0; e < 32; e += 4)
      if (col0 + e < p.N)
        __stcg(reinterpret_cast<float4*>(w + e), make_float4(__uint_as_float(r[e]), __uint_as_float(r[e + 1]),
                                                              __uint_as_float(r[e + 2]), __uint_as_float(r[e + 3])));
  } else {
#pragma unroll
    for (int e = 0; e < 32; ++e)
      if (col0 + e < p.N) __stcg(w + e, __uint_as_float(r[e]));
  }
}

// split-K, after the cluster barrier: split z of a tile applies out = act(alpha * sum_s ws[s] + bias + rowbias) + residual to ITS
// share (pieces [z, z + 1) * NP / splits) of the CTA's 128 x BN block.  te = 0..255 (the epilogue threads): one thread per
// (row, 8 columns) when N and ldc allow 16-byte accesses, else one per element.  The planes were written by other SMs: reads
// bypass L1.  Row-bias / residual loads are issued before the plane sums so that one round trip covers them all.
template <int BN>
__device__ __forceinline__ void splitk_finalize(const GemmParams& p, int m0, int n0, int z, int te) {
  const bool vec = (p.N % 8) == 0 && (p.ldc % 8) == 0 && (!p.rowbias || (p.rowbias_ld % 8) == 0);
  const int64_t plane = (int64_t)p.M * p.N;
  if (vec) {
    constexpr int PPR = BN / 8;
    constexpr int NP = BM * PPR;
    const int share = (NP + p.splits - 1) / p.splits;
    const int i1 = min(NP, (z + 1) * share);
    // a thread's pieces are EPI_THREADS apart: when that is a multiple of the pieces per row its columns never change and
    // the bias is fetched once
    constexpr bool FIXED_COLS = (EPI_THREADS % PPR) == 0;
    float bcol[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) bcol[e] = 0.f;
    if (FIXED_COLS && p.bias) {
      const int i0 = z * share + te, col = n0 + (i0 - (i0 / PPR) * PPR) * 8;
      if (col < p.N) {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col)), b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col + 4));
        bcol[0] = b0.x, bcol[1] = b0.y, bcol[2] = b0.z, bcol[3] = b0.w, bcol[4] = b1.x, bcol[5] = b1.y, bcol[6] = b1.z, bcol[7] = b1.w;
      }
    }
    for (int i = z * share + te; i < i1; i += EPI_THREADS) {
      const int rl = i / PPR, row = m0 + rl, col = n0 + (i - rl * PPR) * 8;
      if (row >= p.M || col >= p.N) continue;
      const int64_t woff = (int64_t)row * p.N + col, o = out_row(p, row) * p.ldc + col;
      uint4 qb = make_uint4(0u, 0u, 0u, 0u), qr = make_uint4(0u, 0u, 0u, 0u);
      if (p.rowbias) qb = *reinterpret_cast<const uint4*>(p.rowbias + (int64_t)(row / p.rows_per_group) * p.rowbias_ld + col);
      if (p.residual) qr = *reinterpret_cast<const uint4*>(p.residual + o);
      if (!FIXED_COLS && p.bias) {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col)), b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col + 4));
        bcol[0] = b0.x, bcol[1] = b0.y, bcol[2] = b0.z, bcol[3] = b0.w, bcol[4] = b1.x, bcol[5] = b1.y, bcol[6] = b1.z, bcol[7] = b1.w;
      }
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = 0.f;
      for (int s = 0; s < p.splits; s += 4) {
        float4 a[4], b[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const bool on = s + t < p.splits;
          const float4* w = reinterpret_cast<const float4*>(p.ws + (int64_t)(s + t) * plane + woff);
          a[t] = on ? __ldcg(w) : make_float4(0.f, 0.f, 0.f, 0.f);
          b[t] = on ? __ldcg(w + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          v[0] += a[t].x, v[1] += a[t].y, v[2] += a[t].z, v[3] += a[t].w;
          v[4] += b[t].x, v[5] += b[t].y, v[6] += b[t].z, v[7] += b[t].w;
        }
      }
      const __half* hb = reinterpret_cast<const __half*>(&qb);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float x = fmaf(v[e], p.alpha, p.rowbias ? __half2float(hb[e]) : 0.f) + bcol[e];
        v[e] = apply_act(x, p.act);
      }
      if (p.residual) {
        const __half* h = reinterpret_cast<const __half*>(&qr);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] += __half2float(h[e]);
      }
      store8(p, o, v);
    }
    return;
  }
  const int share = (BM * BN + p.splits - 1) / p.splits;
  const int i1 = min(BM * BN, (z + 1) * share);
  for (int i = z * share + te; i < i1; i += EPI_THREADS) {
    const int rl = i / BN, row = m0 + rl, col = n0 + (i - rl * BN);
    if (row >= p.M || col >= p.N) continue;
    float x = 0.f;
    for (int s = 0; s < p.splits; ++s) x += __ldcg(p.ws + (int64_t)s * plane + (int64_t)row * p.N + col);
    x *= p.alpha;
    if (p.rowbias) x += __half2float(p.rowbias[(int64_t)(row / p.rows_per_group) * p.rowbias_ld + col]);
    if (p.bias) x += __ldg(p.bias + col);
    x = apply_act(x, p.act);
    const int64_t o = out_row(p, row) * p.ldc + col;
    if (p.residual) x += __half2float(p.residual[o]);
    if (p.out_f32) reinterpret_cast<float*>(p.C)[o] = x;
    else reinterpret_cast<__half*>(p.C)[o] = __float2half_rn(x);
  }
}

constexpr int EPI_RB_GROUPS = 8;                 // row-bias groups (images) one 128-row tile may span when staged in smem
__host__ __device__ constexpr int epi_smem_bytes(int bn) { return bn * 4 + EPI_RB_GROUPS * bn * 2; }
// the two column ranges of the eight epilogue warps split the tile at a multiple of 32 (a GEGLU chunk never straddles them)
__host__ __device__ constexpr int col_split(int bn) { return ((bn / 2 + 31) / 32) * 32; }

// Called by the eight epilogue warps while the main loop runs: the tile's bias and row-group-bias slices go to shared
// memory, so that the epilogue proper never waits on a first-touch global load.
template <int BN>
__device__ __forceinline__ void epilogue_preload(const GemmParams& p, int m0, int n0, float* sbias, __half* srb, int te) {
  for (int i = te; i < BN; i += EPI_THREADS) sbias[i] = (p.bias && n0 + i < p.N) ? __ldg(p.bias + n0 + i) : 0.f;
  if (p.rowbias) {
    const int g0 = m0 / p.rows_per_group;
    const int last = (m0 + BM - 1 < p.M ? m0 + BM - 1 : p.M - 1) / p.rows_per_group;
    const int ng = last - g0 + 1;
    if (ng >= 1 && ng <= EPI_RB_GROUPS)
      for (int i = te; i < ng * BN; i += EPI_THREADS) {
        const int gi = i / BN, c = i - gi * BN;
        srb[i] = (n0 + c < p.N) ? p.rowbias[(int64_t)(g0 + gi) * p.rowbias_ld + n0 + c] : __float2half(0.f);
      }
  }
  epi_bar();
}

template <int ACT>
__device__ __forceinline__ float act_fn(float x) {
  if (ACT == 1) return __fdividef(x, 1.f + __expf(-x));
  if (ACT == 2) return gelu_erf(x);
  if (ACT == 4) return __fdividef(x, 1.f + __expf(-1.702f * x));
  return x;
}

// Phase 1 of the staged epilogue for one thread (= one accumulator row) over tile columns [c_lo, c_hi): accumulator tile ->
// alpha / bias / row-group bias / activation (ACT 3: GEGLU gate) -> fp16 -> this row of the warp's shared-memory slab.
// rb: this row's row-group bias indexed by TILE column (nullptr: none); rb_smem: it is the shared-memory copy (no N tail).
template <int ACT>
__device__ __forceinline__ void stage_rows(const GemmParams& p, const float* acc_row, uint8_t* mine, int n0, int c_lo, int c_hi,
                                           const float* sbias, const __half* rb, bool rb_smem) {
#pragma unroll 1
  for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
    if (n0 + c0 >= p.N) break;                     // warp-uniform
    uint32_t r[32];
    acc_ld32(acc_row + c0, r);
    if (ACT == 3) {
      __half2 h[8];
#pragma unroll
      for (int e = 0; e < 16; e += 2) {
        float a0 = fmaf(__uint_as_float(r[e]), p.alpha, sbias[c0 + e]), a1 = fmaf(__uint_as_float(r[e + 1]), p.alpha, sbias[c0 + e + 1]);
        float g0 = fmaf(__uint_as_float(r[16 + e]), p.alpha, sbias[c0 + 16 + e]);
        float g1 = fmaf(__uint_as_float(r[17 + e]), p.alpha, sbias[c0 + 17 + e]);
        h[e >> 1] = __floats2half2_rn(a0 * gelu_erf_fast(g0), a1 * gelu_erf_fast(g1));
      }
      uint4* d = reinterpret_cast<uint4*>(mine + (c0 - c_lo));   // (c0 - c_lo) / 2 output columns x 2 bytes
      d[0] = reinterpret_cast<uint4*>(h)[0], d[1] = reinterpret_cast<uint4*>(h)[1];
    } else {
#pragma unroll
      for (int j = 0; j < 32; j += 8) {
        float v[8];
        const float4 b0 = *reinterpret_cast<const float4*>(sbias + c0 + j), b1 = *reinterpret_cast<const float4*>(sbias + c0 + j + 4);
        v[0] = b0.x, v[1] = b0.y, v[2] = b0.z, v[3] = b0.w, v[4] = b1.x, v[5] = b1.y, v[6] = b1.z, v[7] = b1.w;
        if (rb && (rb_smem || n0 + c0 + j + 8 <= p.N)) {
          uint4 q = *reinterpret_cast<const uint4*>(rb + c0 + j);
          const __half* hq = reinterpret_cast<const __half*>(&q);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] += __half2float(hq[e]);
        }
        __half2 h[4];
#pragma unroll
        for (int e = 0; e < 8; e += 2) {
          float x0 = fmaf(__uint_as_float(r[j + e]), p.alpha, v[e]), x1 = fmaf(__uint_as_float(r[j + e + 1]), p.alpha, v[e + 1]);
          h[e >> 1] = __floats2half2_rn(act_fn<ACT>(x0), act_fn<ACT>(x1));
        }
        *reinterpret_cast<uint4*>(mine + (c0 - c_lo + j) * 2) = *reinterpret_cast<uint4*>(h);
      }
    }
  }
}

// Output geometry of one epilogue warp in the staged modes: 32 rows x tile columns [c_lo, c_hi) become `outc` fp16 columns
// (GEGLU halves them) = `ppr` 16-byte pieces per row, `total` pieces per warp, lane l owns pieces l, l + 32, ...
struct WarpOut {
  int outc, stride, ppr, total, ocol0, nout;
};
template <int MODE>
__device__ __forceinline__ WarpOut warp_out(const GemmParams& p, int n0, int c_lo, int c_hi) {
  constexpr bool geglu = MODE == 1;
  WarpOut g;
  g.outc = geglu ? (c_hi - c_lo) >> 1 : (c_hi - c_lo);
  g.stride = g.outc * 2 + 16;                      // +16: 16-byte pieces of consecutive rows rotate banks
  g.ppr = g.outc >> 3;
  g.total = 32 * g.ppr;
  g.ocol0 = geglu ? (n0 + c_lo) >> 1 : n0 + c_lo;  // first column of C this warp writes
  g.nout = geglu ? p.N >> 1 : p.N;
  return g;
}

// The first RES_PREFETCH residual pieces of this lane, fetched while the main loop runs.
__device__ __forceinline__ void prefetch_residual(const GemmParams& p, const WarpOut& g, int lane, int row0,
                                                  uint4 (&resq)[RES_PREFETCH]) {
#pragma unroll
  for (int u = 0; u < RES_PREFETCH; ++u) {
    resq[u] = make_uint4(0u, 0u, 0u, 0u);
    const int pp = lane + 32 * u;
    if (p.residual && pp < g.total) {
      const int rl = pp / g.ppr, ci = pp - rl * g.ppr;
      const int grow = row0 + rl, col = g.ocol0 + ci * 8;
      if (grow < p.M && col < g.nout) resq[u] = *reinterpret_cast<const uint4*>(p.residual + out_row(p, grow) * p.ldc + col);
    }
  }
}

__device__ __forceinline__ uint4 add_h8(uint4 v, uint4 q) {
  __half2* a = reinterpret_cast<__half2*>(&v);
  const __half2* b = reinterpret_cast<const __half2*>(&q);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 fa = __half22float2(a[e]), fb = __half22float2(b[e]);
    a[e] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
  }
  return v;
}

// Staged epilogue of ONE warp: 32 accumulator rows x tile columns [c_lo, c_hi), fp16 output.
//   phase 1   thread = row of the accumulator tile: alpha / bias / row-group bias / activation / GEGLU gate, rounded to
//             fp16 (where autocast rounds the layer output) into this warp's slab;
//   phase 2   the warp walks the slab in 16-byte pieces along rows, adds the residual (prefetched for the first
//             RES_PREFETCH pieces of a lane) and writes whole rows: every global access is a run of full 32-byte sectors.
// (r1 trace: with one 16-byte store per lane to 32 different rows the epilogue took 46 000 cycles per tile.)
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_staged(const GemmParams& p, const WarpOut& g, const float* acc_row, uint8_t* slab, int lane,
                                                int m0, int row0, int n0, int c_lo, int c_hi, const float* sbias, const __half* srb,
                                                const uint4 (&resq)[RES_PREFETCH]) {
  const int row = row0 + lane;
  // row-group bias of this thread's row: from the smem copy when the tile spans few groups, else straight from global
  const __half* rb = nullptr;
  bool rb_smem = false;
  if (MODE != 1 && p.rowbias) {
    const int rr = row < p.M ? row : p.M - 1;
    const int g0 = m0 / p.rows_per_group, last = (m0 + BM - 1 < p.M ? m0 + BM - 1 : p.M - 1) / p.rows_per_group;
    rb_smem = last - g0 + 1 <= EPI_RB_GROUPS;
    rb = rb_smem ? srb + (rr / p.rows_per_group - g0) * BN : p.rowbias + (int64_t)(rr / p.rows_per_group) * p.rowbias_ld + n0;
  }
  uint8_t* mine = slab + lane * g.stride;
  if (MODE == 0) {
    stage_rows<0>(p, acc_row, mine, n0, c_lo, c_hi, sbias, rb, rb_smem);
  } else if (MODE == 1) {
    stage_rows<3>(p, acc_row, mine, n0, c_lo, c_hi, sbias, rb, rb_smem);
  } else {   // the activation switch is hoisted out of the element loops: one branch per tile
    switch (p.act) {
      case 1: stage_rows<1>(p, acc_row, mine, n0, c_lo, c_hi, sbias, rb, rb_smem); break;
      case 2: stage_rows<2>(p, acc_row, mine, n0, c_lo, c_hi, sbias, rb, rb_smem); break;
      default: stage_rows<4>(p, acc_row, mine, n0, c_lo, c_hi, sbias, rb, rb_smem); break;
    }
  }
  __syncwarp();
  __half* C = reinterpret_cast<__half*>(p.C);
  // N is a multiple of 8 on this path (host check): no partial pieces
#pragma unroll
  for (int u = 0; u < RES_PREFETCH; ++u) {
    const int pp = lane + 32 * u;
    if (pp < g.total) {
      const int rl = pp / g.ppr, ci = pp - rl * g.ppr;
      const int grow = row0 + rl, col = g.ocol0 + ci * 8;
      if (grow < p.M && col < g.nout) {
        uint4 v = *reinterpret_cast<const uint4*>(slab + rl * g.stride + ci * 16);
        if (p.residual) v = add_h8(v, resq[u]);
        *reinterpret_cast<uint4*>(C + out_row(p, grow) * p.ldc + col) = v;
      }
    }
  }
  constexpr int UN = 4;
  for (int base = lane + 32 * RES_PREFETCH; base < g.total; base += 32 * UN) {
    uint4 v[UN], q[UN];
    int64_t o[UN];
    bool ok[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int pp = base + 32 * u;
      const int rl = pp / g.ppr, ci = pp - rl * g.ppr;
      const int grow = row0 + rl, col = g.ocol0 + ci * 8;
      ok[u] = pp < g.total && grow < p.M && col < g.nout;
      o[u] = out_row(p, grow) * p.ldc + col;
      if (ok[u]) {
        v[u] = *reinterpret_cast<const uint4*>(slab + rl * g.stride + ci * 16);
        if (p.residual) q[u] = *reinterpret_cast<const uint4*>(p.residual + o[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      if (!ok[u]) continue;
      if (p.residual) v[u] = add_h8(v[u], q[u]);
      *reinterpret_cast<uint4*>(C + o[u]) = v[u];
    }
  }
}

__host__ __device__ constexpr int epi_slab_bytes(int bn) { return EPI_WARPS * 32 * (col_split(bn) * 2 + 16); }
constexpr int smem_bytes(int bn, int stages) {
  return stages * (BM * BK * 2 + bn * BK * 2) + epi_slab_bytes(bn) + 2 * stages * 8 + 16 + epi_smem_bytes(bn) + 1024;
}

// Where the producer's next k-block comes from.  The producer is one thread that waits for a free stage and then issues its
// loads, so every instruction between the two adds to the latency of refilling the ring.  Integer divisions by runtime sizes
// cost ~100 cycles of dependent instructions each.  So the tile's pixel origin and batch indices are computed once per
// tile, and the conv's (tap, channel block) is stepped along with kb instead of divided out of it.
struct ProducerPos {
  int x, y, b;       // conv: tile origin in the activation (x, y, image); batched: (head, batch) in (y, b)
  int tap, tx, ty;   // conv: tap of the next k-block and its column / row in the tap grid
  int cb;            // conv: channel block of the next k-block
};
__device__ __forceinline__ ProducerPos producer_start(const GemmParams& p, int m0, int bz, int kb0) {
  ProducerPos q;
  q.x = q.y = q.b = q.tap = q.tx = q.ty = q.cb = 0;
  if (p.conv) {
    const int r = m0 / p.cW;
    q.x = m0 - r * p.cW, q.y = r % p.cH, q.b = r / p.cH;
    q.tap = kb0 / p.cblocks, q.cb = kb0 - q.tap * p.cblocks;
    q.ty = q.tap / p.ctx, q.tx = q.tap - q.ty * p.ctx;
  } else if (p.batched) {
    q.y = bz % p.nh, q.b = bz / p.nh;
  }
  return q;
}
__device__ __forceinline__ void producer_step(const GemmParams& p, ProducerPos& q) {
  if (p.conv && ++q.cb == p.cblocks) {
    q.cb = 0, ++q.tap;
    if (++q.tx == p.ctx) q.tx = 0, ++q.ty;
  }
}

// One stage of the TMA producer: the 128 rows of A and the BN rows of B for k-block kb of the tile at (m0, n0); q is kb's position.
template <int BN>
__device__ __forceinline__ void produce_stage(const GemmParams& p, const CUtensorMap* tmA, const CUtensorMap* tmB, uint8_t* a_dst,
                                              uint8_t* b_dst, uint64_t* full_bar, int kb, int m0, int n0, const ProducerPos& q) {
  mbar_expect_tx(full_bar, BM * BK * 2 + BN * BK * 2);
  if (p.conv) {
    const int c0 = q.cb * BK;
    tma_load_4d(a_dst, tmA, full_bar, c0, q.x + q.tx + p.cox, q.y + q.ty + p.coy, q.b);
    tma_load_2d(b_dst, tmB, full_bar, q.tap * p.cC + c0, n0);
  } else if (p.batched) {
    tma_load_4d(a_dst, tmA, full_bar, kb * BK, m0, q.y, q.b);
    tma_load_4d(b_dst, tmB, full_bar, kb * BK, n0, q.y, q.b);
  } else {
    tma_load_2d(a_dst, tmA, full_bar, kb * BK, m0);
    tma_load_2d(b_dst, tmB, full_bar, kb * BK, n0);
  }
}

// A warpgroup's m64nBN accumulator fragment -> rows [row0, row0 + 64) of the shared-memory accumulator tile
template <int BN>
__device__ __forceinline__ void acc_store(float* acc, const float (&d)[BN / 2], int row0, int t) {
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(acc + r * acc_ld(BN) + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc + (r + 8) * acc_ld(BN) + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// ------------------------------------------------------------------------------------------------ the kernel
template <int BN, int STAGES, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by SWIZZLE_128B
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
  static_assert(B_BYTES % 1024 == 0, "stage bases must stay 1024-byte aligned for SWIZZLE_128B");
  static_assert(BN % 32 == 0 && BN >= 64 && BN <= 256, "tile width: a multiple of 32 (GEGLU chunks, 32-column epilogue reads)");
  static_assert(BM * acc_ld(BN) * 4 <= STAGES * (A_BYTES + B_BYTES), "the accumulator tile must fit in the operand ring");
  constexpr int CSPLIT = col_split(BN);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint8_t* slabs = sB + STAGES * B_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(slabs + epi_slab_bytes(BN));
  uint64_t* empty = full + STAGES;
  float* sbias = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(empty + STAGES) + 15) & ~(uintptr_t)15);
  __half* srb = reinterpret_cast<__half*>(sbias + BN);
  float* acc = reinterpret_cast<float*>(smem);                // the operand ring, once the K loop is done

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) stamp(p, 0), stamp_ns(p, 16);
  const int bz = blockIdx.z;
  const int nk = p.conv ? p.ctaps * p.cblocks : (p.K + BK - 1) / BK;
  // split-K: blockIdx.z owns k-blocks [kb0, kb1) and stores its partial tile into its plane of the fp32 workspace
  const bool split = MODE == 3 && p.splits > 1;
  int kb0 = 0, kb1 = nk;
  if (split) {
    kb0 = (int)((int64_t)nk * bz / p.splits);
    kb1 = (int)((int64_t)nk * (bz + 1) / p.splits);
  }

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < STAGES; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 2);   // empty: one arrival per MMA warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();      // everything above touched no global memory: it overlaps the tail of the previous kernel
  pdl_trigger();
  if (threadIdx.x == 0) stamp(p, 1);

  // Tiles of this CTA: one (blockIdx.x, blockIdx.y), or -- persistent launch (p.persist, staged epilogues only) -- tiles
  // blockIdx.x, blockIdx.x + gridDim.x, ... of the column-major tile order.  The ring's stage / phase counters run on across
  // tiles, so the producer fills the next tile's first stages as soon as the epilogue has handed the ring back.
  const int tiles_m = (p.M + BM - 1) / BM, tiles = tiles_m * ((p.N + BN - 1) / BN);
  const bool persist = MODE != 3 && p.persist;
  uint32_t cnt = 0;   // k-blocks consumed so far by this CTA
  for (int t = persist ? blockIdx.x : blockIdx.y * tiles_m + blockIdx.x; t < tiles; t += persist ? gridDim.x : tiles) {
  const int m0 = (t % tiles_m) * BM, n0 = (t / tiles_m) * BN;
  if (warp < 4) {
    if (threadIdx.x == 0) {  // ---------------- TMA producer
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the epilogue's generic accesses to the ring come first
      ProducerPos q = producer_start(p, m0, bz, kb0);
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t c = cnt + (kb - kb0);
        const int s = c % STAGES;
        const uint32_t ph = (c / STAGES) & 1;
        mbar_wait(empty + s, ph ^ 1, p, WAIT_EMPTY, s);
        produce_stage<BN>(p, &tmA, &tmB, sA + s * A_BYTES, sB + s * B_BYTES, full + s, kb, m0, n0, q);
        producer_step(p, q);
        if (kb == kb0) stamp(p, 2);
      }
      stamp(p, 3);
    }
    __syncwarp();
  } else {  // ------------------------ warpgroups 1 and 2: MMAs on rows [64 wg, 64 wg + 64), then the epilogue
    const int wg = (warp >> 2) - 1, e = warp - 4, quarter = e & 3, te = threadIdx.x - 128;
    const int c_lo = e < 4 ? 0 : CSPLIT, c_hi = e < 4 ? CSPLIT : BN;   // this warp's tile columns
    const int row0 = m0 + quarter * 32;
    if (MODE != 3) epilogue_preload<BN>(p, m0, n0, sbias, srb, te);
    {
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t c = cnt + (kb - kb0);
        const int s = c % STAGES;
        const uint32_t ph = (c / STAGES) & 1;
        mbar_wait(full + s, ph, p, WAIT_FULL, s);
        if (kb == kb0 && te == 0) stamp(p, 4);
        const uint32_t a0 = smem_u32(sA + s * A_BYTES) + wg * (64 * 128), b0 = smem_u32(sB + s * B_BYTES);
        wg::fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)   // advancing 16 fp16 along K inside the 128-byte swizzle atom = +32 bytes on the start address
          wg::mma_f16<BN>(d, wg::desc_sw128(a0 + k * 32), wg::desc_sw128(b0 + k * 32), 1);
        wg::commit();
        wg::wait<1>();                      // the previous stage's MMAs are done: hand that stage back to the producer
        if (kb > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(empty + (c - 1) % STAGES);
      }
      wg::wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty + (cnt + kb1 - kb0 - 1) % STAGES);
      if (te == 0) stamp(p, 5);
      epi_bar();                            // both warpgroups are done reading the ring: it becomes the accumulator tile
      acc_store<BN>(acc, d, 64 * wg, threadIdx.x & 127);
    }
    epi_bar();
    if (te == 0) stamp(p, 6);
    const float* acc_row = acc + (quarter * 32 + lane) * acc_ld(BN);
    if (MODE != 3) {
      const WarpOut g = warp_out<MODE>(p, n0, c_lo, c_hi);
      uint4 resq[RES_PREFETCH];
      prefetch_residual(p, g, lane, row0, resq);
      epilogue_staged<BN, MODE>(p, g, acc_row, slabs + e * 32 * (CSPLIT * 2 + 16), lane, m0, row0, n0, c_lo, c_hi, sbias, srb, resq);
    } else {
      const int row = row0 + lane;
      if (split) {
        if (te == 0) stamp_ns(p, 17);
#pragma unroll 1
        for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
          uint32_t r[32];
          acc_ld32(acc_row + c0, r);
          if (row < p.M) splitk_partial(p, r, bz, row, n0 + c0);
        }
        if (te == 0) stamp_ns(p, 18);
      } else {
        const int64_t crow = (p.batched ? (int64_t)(bz % p.nh) * p.stride_c_h + (int64_t)(bz / p.nh) * p.stride_c_b : 0) +
                             out_row(p, row < p.M ? row : 0) * p.ldc;
#pragma unroll 1
        for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
          uint32_t r[32];
          acc_ld32(acc_row + c0, r);
          if (row < p.M) epilogue_chunk(p, r, row, crow, n0 + c0);
        }
      }
    }
    if (te == 0) stamp(p, 7);
  }
  cnt += kb1 - kb0;
  __syncthreads();   // the epilogue is done with the accumulator tile, slabs and bias slices: the ring is free for the next tile
  }
  if (split) {
    // the `splits` CTAs of a tile form ONE cluster (co-scheduled by the hardware): this barrier -- release / acquire at
    // cluster scope -- publishes every split's partial plane to its siblings
    cluster_sync_all();
    if (warp >= 4) {   // every split finalizes its share of the 128 x BN block: sum of the planes + epilogue
      if (threadIdx.x == 128) stamp_ns(p, 21, true);
      splitk_finalize<BN>(p, blockIdx.x * BM, blockIdx.y * BN, bz, threadIdx.x - 128);
      if (threadIdx.x == 128) stamp_ns(p, 22, true);
    }
  }
  if (threadIdx.x == 0) stamp(p, 8);
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// [nb, nh, rows, K] fp16 view with row stride ld and batch strides sh / sb (elements); box = 64 x box_rows (x 1 x 1)
int make_map(CUtensorMap* m, const void* ptr, int64_t rows, int64_t K, int64_t ld, int nh, int nb, int64_t sh, int64_t sb,
             int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return O2345_ECUDA; }
  cuuint64_t dims[4] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)(nh > 0 ? nh : 1), (cuuint64_t)(nb > 0 ? nb : 1)};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)sh * 2, (cuuint64_t)sb * 2};
  cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  int rank = nh > 0 ? 4 : 2;
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with %d (rows=%lld K=%lld ld=%lld)", (int)r, (long long)rows, (long long)K, (long long)ld); return O2345_ECUDA; }
  return O2345_OK;
}

// Host-mapped trap record (one per process): allocated on the first launch that is not inside a stream capture.
TrapRecord* g_diag = nullptr;
bool g_diag_tried = false;
TrapRecord* diag_buffer(cudaStream_t st) {
  if (!g_diag_tried) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
      cudaGetLastError();
      return g_diag;
    }
    g_diag_tried = true;
    void* h = nullptr;
    if (cudaHostAlloc(&h, sizeof(TrapRecord), cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) {
      memset(h, 0, sizeof(TrapRecord));
      g_diag = reinterpret_cast<TrapRecord*>(h);
    } else {
      cudaGetLastError();
    }
  }
  return g_diag;
}

struct Config {
  int bn, splits;
  int persist;   // 1: persistent launch (at most one CTA per SM walks the tiles)
};

// tuning / sweep hook: O2345_GEMM_FORCE="ctas,bn,splits" (0 = keep the heuristic's choice for that field; ctas is 1, one CTA
// per tile); also settable through o2345_debug_gemm_force (tools/gemm_sweep.py)
int g_force[3] = {-1, 0, 0};
int g_persist = 0;             // 0: heuristic, 1: persistent launch wherever available, 2: never (o2345_debug_gemm_persist)
int g_persist_min_tiles = 0;   // heuristic threshold override (0: default)
void read_force_env() {
  if (g_force[0] >= 0) return;
  g_force[0] = g_force[1] = g_force[2] = 0;
  const char* e = getenv("O2345_GEMM_FORCE");
  if (e) sscanf(e, "%d,%d,%d", &g_force[0], &g_force[1], &g_force[2]);
}

// Tile width and k-splits for a problem of M x N with nk k-blocks of 64: the candidate with the lowest predicted time under a
// small cost model (its constants are starting values, not yet fitted on an H100 with tools/gemm_sweep.py):
//   * a launch costs ~5 us of fixed latency (launch, prologue, first TMA round trip, tear-down) + ~3 us of epilogue per
//     160 columns of tile and wave of CTAs;
//   * the main loop is bound by operand delivery or by the tensor pipe (a 128 x BN x 64 k-block is 4 BN cycles of wgmma at
//     ~2 048 fp16 FMA per clock and SM): an SM ingests ~40 B/clk, the whole L2 -> SM fabric ~6 300 B/clk -- so few fat tiles
//     starve (few SMs pull), many thin tiles re-read A (fabric), and long-K problems with few tiles want split-K;
//   * split-K adds ~4 us + ~1 us per split and 128 tile columns (partial planes through L2, cluster barrier, finalize).
float g_model[7] = {40.f, 0.5f, 6300.f, 5.f, 3.f, 4.f, 1.f};   // bw_sm, alpha, cap, fixed, epi, so0, so1 (tools: o2345_debug_gemm_model)
float predict_us(int M, int N, int nk, int bn, int splits) {
  const float bw_sm = g_model[0], alpha = g_model[1], cap = g_model[2], fixed = g_model[3], epi = g_model[4], so0 = g_model[5],
              so1 = g_model[6], cyc_per_us = 1750.f;
  const int tiles = cdiv(M, BM) * cdiv(N, bn);
  const int n = tiles * splits;
  const int kb = cdiv(nk, splits);
  const float bytes_cta = (float)kb * (float)(BM * BK * 2 + bn * BK * 2);
  const int sms = sm_count();
  const int rounds = cdiv(n, sms);
  float f = (float)(n - sms) / (float)sms;
  f = f < 0.f ? 0.f : (f > 1.f ? 1.f : f);
  const float t_sm = (float)rounds * bytes_cta / (bw_sm * (1.f + alpha * f));
  const float t_fabric = (float)n * bytes_cta / cap;
  const float t_mma = (float)rounds * (float)kb * 4.f * (float)bn;
  float t = t_sm > t_fabric ? t_sm : t_fabric;
  if (t_mma > t) t = t_mma;
  float us = fixed + t / cyc_per_us + epi * (float)bn / 160.f * (float)cdiv(n, sms);
  if (splits > 1) us += so0 + so1 * (float)splits * (float)bn / 128.f;
  return us;
}

Config pick_config(const GemmParams& p, int nk, bool can_split, int64_t ws_floats) {
  read_force_env();
  Config c;
  const int M = p.M, N = p.N;
  c.persist = 0;
  if (p.batched) {
    c.bn = N <= 64 ? 64 : 128, c.splits = 1;
    return c;
  }
  static const int kBn[4] = {64, 128, 160, 256};
  static const int kSplits[6] = {1, 2, 3, 4, 6, 8};
  const bool split_ok = can_split && p.act != 3 && p.ws && 2 * (int64_t)M * N <= ws_floats;
  const int max_planes = split_ok ? (int)(ws_floats / ((int64_t)M * N)) : 1;
  float best = 1e30f;
  c.bn = 128, c.splits = 1;
  for (int bi = 0; bi < 4; ++bi) {
    const int bn = kBn[bi];
    if (bn > 64 && N <= 64) continue;
    if (g_force[1] > 0 && bn != g_force[1]) continue;
    for (int si = 0; si < 6; ++si) {
      const int sp = kSplits[si];
      if (g_force[2] > 0 && sp != (g_force[2] > nk ? nk : g_force[2])) continue;
      if (sp > 1 && (!split_ok || sp > max_planes || sp > MAX_CLUSTER || nk / sp < 3)) continue;
      const float us = predict_us(M, N, nk, bn, sp);
      if (us < best) best = us, c.bn = bn, c.splits = sp;
    }
  }
  if (best > 1e29f) {   // a forced configuration that is not available: fall back to the nearest valid one
    c.bn = (g_force[1] == 64 || g_force[1] == 128 || g_force[1] == 160 || g_force[1] == 256) ? g_force[1] : 128;
    c.splits = 1;
  }
  // Many waves of tiles: one CTA per SM walks them, so that launch, prologue and the wave tail are paid once per SM
  const int tiles = cdiv(M, BM) * cdiv(N, c.bn);
  const int min_tiles = g_persist_min_tiles > 0 ? g_persist_min_tiles : 4 * sm_count();
  c.persist = c.splits == 1 && (g_persist == 1 || (g_persist == 0 && tiles >= min_tiles));
  return c;
}

// which compile-time epilogue: staged fp16 output needs whole 16-byte pieces and one pass (no split-K, no head batches)
int pick_mode(const GemmParams& p, const Config& c) {
  const int nout = p.act == 3 ? p.N / 2 : p.N;
  const bool staged = !p.out_f32 && c.splits <= 1 && !p.batched && (nout % 8) == 0 && (p.ldc % 8) == 0 && ((uintptr_t)p.C % 16) == 0 &&
                      (!p.residual || ((uintptr_t)p.residual % 16) == 0);
  if (!staged) return 3;
  return p.act == 0 ? 0 : (p.act == 3 ? 1 : 2);
}

long long* g_trace = nullptr;

template <int BN, int STAGES, int MODE>
int launch(const CUtensorMap& a, const CUtensorMap& b, GemmParams p, int batch, int persist, cudaStream_t st) {
  constexpr int SMEM = smem_bytes(BN, STAGES);
  static_assert(SMEM <= 227 * 1024, "one CTA per SM");
  static PerDeviceOnce attr;
  if (attr.need())
    O2345_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, STAGES, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  p.bn = BN, p.mode = MODE;
  p.diag = diag_buffer(st);
  const int splits = (MODE == 3 && batch == 0 && p.splits > 1) ? p.splits : 1;
  p.splits = splits;
  dim3 grid(cdiv(p.M, BM), cdiv(p.N, BN), batch > 0 ? batch : splits);
  p.persist = MODE != 3 && batch == 0 && splits == 1 && persist;
  if (p.persist) {
    const int tiles = (int)grid.x * (int)grid.y;
    grid = dim3(tiles < sm_count() ? tiles : sm_count(), 1, 1);
  }
  O2345_CUDA(launch_pdl_cluster(gemm_tc_kernel<BN, STAGES, MODE>, grid, dim3(GEMM_THREADS), (size_t)SMEM, st, 1, splits, a, b, p));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

template <int BN, int STAGES>
int launch_mode(int mode, const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, int batch, int persist, cudaStream_t st) {
  switch (mode) {
    case 0: return launch<BN, STAGES, 0>(a, b, p, batch, persist, st);
    case 1: return launch<BN, STAGES, 1>(a, b, p, batch, persist, st);
    case 2: return launch<BN, STAGES, 2>(a, b, p, batch, persist, st);
    default: return launch<BN, STAGES, 3>(a, b, p, batch, persist, st);
  }
}

// ring depth per tile width: as many stages as fit next to the epilogue slabs in 227 KB (one CTA per SM)
int dispatch(const Config& c, int mode, const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, int batch, cudaStream_t st) {
  if (c.bn == 64) return launch_mode<64, 6>(mode, a, b, p, batch, c.persist, st);
  if (c.bn == 128) return launch_mode<128, 5>(mode, a, b, p, batch, c.persist, st);
  if (c.bn == 160) return launch_mode<160, 4>(mode, a, b, p, batch, c.persist, st);
  return launch_mode<256, 3>(mode, a, b, p, batch, c.persist, st);
}

int fill_epilogue(GemmParams& p, const o2345_epilogue* ep, int N, int64_t ldc) {
  p.bias = nullptr, p.rowbias = nullptr, p.rowbias_ld = 0, p.rows_per_group = 1, p.residual = nullptr;
  p.out_f32 = 0, p.act = 0, p.alpha = 1.f, p.trace = g_trace;
  p.diag = nullptr, p.bn = p.mode = 0;
  if (!ep) return O2345_OK;
  O2345_CHECK_ARG(ep->act >= 0 && ep->act <= 4, "unknown activation");
  O2345_CHECK_ARG(!ep->rowbias || (ep->rows_per_group > 0 && (ep->rowbias_ld % 8) == 0 && ((uintptr_t)ep->rowbias % 16) == 0),
                  "row bias: rows_per_group > 0, 16-byte aligned, row stride a multiple of 8");
  O2345_CHECK_ARG(ep->act != 3 || ((N % 32) == 0 && (ldc % 8) == 0 && !ep->residual && !ep->rowbias),
                  "GEGLU epilogue: N must be a multiple of 32, ldc of 8, no residual / row bias");
  p.bias = ep->bias, p.rowbias = reinterpret_cast<const __half*>(ep->rowbias), p.rowbias_ld = ep->rowbias_ld;
  p.rows_per_group = ep->rowbias ? ep->rows_per_group : 1;
  p.residual = reinterpret_cast<const __half*>(ep->residual), p.out_f32 = ep->out_f32, p.act = ep->act, p.alpha = ep->alpha;
  return O2345_OK;
}

void set_workspace(GemmParams& p, float* ws, int64_t ws_floats) { p.ws = ws_floats > 0 ? ws : nullptr; }

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" void o2345_debug_gemm_trace(long long* device_buf16) { g_trace = device_buf16; }

extern "C" void o2345_debug_gemm_force(int ctas, int bn, int splits) {
  read_force_env();
  g_force[0] = ctas, g_force[1] = bn, g_force[2] = splits;
}


extern "C" void o2345_debug_gemm_persist(int mode, int min_tiles) { g_persist = mode, g_persist_min_tiles = min_tiles; }

extern "C" void o2345_debug_gemm_model(const float* seven) {
  for (int i = 0; i < 7; ++i) g_model[i] = seven[i];
}

extern "C" int o2345_last_trap(char* buf, size_t n) {
  if (!buf || n == 0) return O2345_EINVAL;
  buf[0] = 0;
  const TrapRecord* d = g_diag;
  if (!d || d->magic != TRAP_MAGIC) return 0;
  static const char* names[] = {"?", "empty (producer waiting for the MMA to free a stage)", "full (MMA issuer waiting for TMA bytes)",
                                };
  snprintf(buf, n,
           "gemm_tc_kernel<BN=%d, MODE=%d> M=%d N=%d K=%d conv=%d splits=%d: CTA (%d,%d,%d) rank %d gave up after 4 s "
           "on barrier '%s' stage %d",
           d->bn, d->mode, d->M, d->N, d->K, d->conv, d->splits, d->bx, d->by, d->bz, d->rank,
           names[d->tag >= 1 && d->tag <= 2 ? d->tag : 0], d->stage);
  return 1;
}

namespace o2345 {
namespace {
// One implicit convolution launch over the channel-last activation x [B, H, W, C]: `taps` taps in rows of `tx`, tap j shifted by
// (j % tx + ox, j / tx + oy); weight [N, taps * C] in (tap, channel) order; up / upa / upb: see GemmParams.
int conv_launch(const void* x, int B, int H, int W, int C, const void* weight, int N, void* out, int64_t ldc, const o2345_epilogue* ep,
                float* splitk_ws, int64_t ws_floats, int taps, int tx, int ox, int oy, int up, int upa, int upb, cudaStream_t st) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return O2345_ECUDA; }
  const int tw = W >= 128 ? 128 : W;
  const int th = W >= 128 ? 1 : (128 / W < H ? 128 / W : H);
  const int tb = 128 / (tw * th);
  CUtensorMap ma, mb;
  {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)tw, (cuuint32_t)th, (cuuint32_t)tb};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (conv activation) failed with %d", (int)r); return O2345_ECUDA; }
  }
  GemmParams p;
  p.M = B * H * W, p.N = N, p.K = taps * C, p.ldc = ldc, p.nh = 1, p.stride_c_h = 0, p.stride_c_b = 0, p.C = out;
  int rc = fill_epilogue(p, ep, N, ldc);
  if (rc) return rc;
  p.batched = 0, p.conv = 1, p.cC = C, p.cH = H, p.cW = W, p.cblocks = (C + BK - 1) / BK;
  p.ctaps = taps, p.ctx = tx, p.cox = ox, p.coy = oy, p.up = up, p.upa = upa, p.upb = upb;
  set_workspace(p, splitk_ws, ws_floats);
  const Config c = pick_config(p, taps * p.cblocks, true, ws_floats);
  p.splits = c.splits;
  rc = make_map(&mb, weight, N, taps * (int64_t)C, taps * (int64_t)C, 0, 0, 0, 0, c.bn);
  if (rc) return rc;
  return dispatch(c, pick_mode(p, c), ma, mb, p, 0, st);
}

// an output tile is 128 consecutive pixels fetched as ONE box (tw, th, tb): either whole multiples of 128 along a row,
// or whole rows that tile the image exactly (H a multiple of 128 / W), or whole images (H * W divides 128).  Any other
// shape would wrap a tile across the image border (silently wrong rows) or give a box of fewer than 128 rows (the
// stage's byte count would never be reached): refused, callers take the im2col route.
bool conv_tiles(int H, int W) {
  return (W % 128) == 0 || ((128 % W) == 0 && (((int64_t)H * W >= 128 && (H % (128 / W)) == 0) || ((int64_t)H * W < 128 && (128 % (H * W)) == 0)));
}
}  // namespace
}  // namespace o2345

extern "C" int o2345_conv3x3_f16(const void* x, int B, int H, int W, int C, const void* weight, int N, void* out, int64_t ldc,
                                 const o2345_epilogue* ep, float* splitk_ws, int64_t ws_floats, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && weight && out, "null pointer");
  O2345_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && (C % 8) == 0 && N > 0, "bad sizes (C must be a multiple of 8)");
  O2345_CHECK_ARG(conv_tiles(H, W),
                  "implicit 3x3 conv: the image must tile into 128-pixel boxes (W % 128 == 0, or 128 % W == 0 with "
                  "H % (128 / W) == 0, or 128 % (H * W) == 0)");
  O2345_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)weight % 16) == 0, "operands must be 16-byte aligned");
  return conv_launch(x, B, H, W, C, weight, N, out, ldc, ep, splitk_ws, ws_floats, 9, 3, -1, -1, 0, 0, 0, (cudaStream_t)stream);
}

extern "C" int o2345_conv_up2x_f16(const void* x, int B, int H, int W, int C, const void* weight4, int N, void* out, int64_t ldc,
                                   const o2345_epilogue* ep, float* splitk_ws, int64_t ws_floats, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && weight4 && out, "null pointer");
  O2345_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && (C % 8) == 0 && N > 0, "bad sizes (C must be a multiple of 8)");
  O2345_CHECK_ARG(conv_tiles(H, W), "up-sampling conv: the LOW-resolution image must tile into 128-pixel boxes (see o2345_conv3x3_f16)");
  O2345_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)weight4 % 16) == 0, "operands must be 16-byte aligned");
  O2345_CHECK_ARG(!ep || (!ep->residual && !ep->rowbias && ep->act != 3),
                  "up-sampling conv: bias / activation epilogues only (no residual, row bias, GEGLU)");
  O2345_CHECK_ARG((int64_t)B * 4 * H * W < (1ll << 31), "output rows must fit 31 bits");
  const __half* w = reinterpret_cast<const __half*>(weight4);
  for (int ph = 0; ph < 4; ++ph) {   // phase (a, b) = (row parity, column parity) of the output pixel
    const int a = ph >> 1, b = ph & 1;
    int rc = conv_launch(x, B, H, W, C, w + (int64_t)ph * N * 4 * C, N, out, ldc, ep, splitk_ws, ws_floats, 4, 2, b - 1, a - 1, 1, a, b,
                         (cudaStream_t)stream);
    if (rc) return rc;
  }
  return O2345_OK;
}

extern "C" int o2345_gemm_f16(const void* A, const void* B, void* C, int M, int N, int K, int64_t lda, int64_t ldb,
                              int64_t ldc, int nh, int nb, int64_t stride_a_h, int64_t stride_a_b, int64_t stride_b_h,
                              int64_t stride_b_b, int64_t stride_c_h, int64_t stride_c_b, const o2345_epilogue* ep,
                              float* splitk_ws, int64_t ws_floats, o2345_stream_t stream) {
  O2345_CHECK_ARG(A && B && C, "null pointer");
  O2345_CHECK_ARG(M > 0 && N > 0 && K > 0 && nh >= 0 && (nh == 0 || nb >= 1), "bad sizes");
  O2345_CHECK_ARG((lda % 8) == 0 && (ldb % 8) == 0, "row strides of A and B must be multiples of 8 fp16 (16 bytes) for TMA");
  O2345_CHECK_ARG(((uintptr_t)A % 16) == 0 && ((uintptr_t)B % 16) == 0, "A and B must be 16-byte aligned");
  O2345_CHECK_ARG(nh == 0 || ((stride_a_h % 8) == 0 && (stride_a_b % 8) == 0 && (stride_b_h % 8) == 0 && (stride_b_b % 8) == 0),
                  "batch strides must be multiples of 8 fp16");
  GemmParams p;
  p.M = M, p.N = N, p.K = K, p.ldc = ldc, p.nh = nh > 0 ? nh : 1, p.stride_c_h = stride_c_h, p.stride_c_b = stride_c_b, p.C = C;
  int rc = fill_epilogue(p, ep, N, ldc);
  if (rc) return rc;
  O2345_CHECK_ARG(nh == 0 || (!p.rowbias && p.act != 3), "row bias / GEGLU are not available in batched mode");
  p.batched = nh > 0 ? 1 : 0;
  p.conv = 0, p.cC = p.cH = p.cW = p.cblocks = 0;
  p.ctaps = p.ctx = p.cox = p.coy = p.up = p.upa = p.upb = 0;
  set_workspace(p, splitk_ws, ws_floats);
  cudaStream_t st = (cudaStream_t)stream;
  const Config c = pick_config(p, cdiv(K, BK), nh == 0, ws_floats);
  p.splits = c.splits;
  CUtensorMap ma, mb;
  rc = make_map(&ma, A, M, K, lda, nh, nb, stride_a_h, stride_a_b, BM);
  if (rc) return rc;
  rc = make_map(&mb, B, N, K, ldb, nh, nb, stride_b_h, stride_b_b, c.bn);
  if (rc) return rc;
  return dispatch(c, pick_mode(p, c), ma, mb, p, nh > 0 ? nh * nb : 0, st);
}
