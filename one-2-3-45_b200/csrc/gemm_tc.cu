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
//                 while the previous one is released, then runs the epilogue of its 64 rows.
// MODE selects the epilogue at compile time:
//   0 staged, no activation   1 staged, GEGLU gate   2 staged, SiLU / GELU / QuickGELU (runtime switch per tile)
//      Each consumer warpgroup applies alpha / bias / row-group bias / activation / GEGLU gate to its own wgmma fragment
//      registers, rounds to fp16 and writes them into its private 64-row output half tile in shared memory, where TMA has
//      already put the residual (loaded during the main loop) -- the residual is added in place -- and one thread stores
//      the half tile with an asynchronous TMA store.  The operand ring is handed back at the last MMA, so the producer
//      fills the next tile's first stages while the epilogue runs, and the two warpgroups never wait for each other.
//   3 generic (fp32 output, batched, unaligned N) and SPLIT-K: the fp32 accumulator tile goes through the (idle) operand
//      ring and the eight consumer warps store it from there.
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

enum { WAIT_EMPTY = 1, WAIT_FULL = 2, WAIT_RESIDUAL = 3 };   // which wait timed out (o2345_last_trap)

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
// asynchronous TMA stores of a shared-memory box (bulk async-group of the issuing thread)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's stores have finished reading shared memory / have completed
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // the eight MMA / epilogue warps only
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }   // one consumer warpgroup

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

constexpr int EPI_RB_GROUPS = 8;                 // row-bias groups (images) one warpgroup's 64 rows may span when staged in smem
__host__ __device__ constexpr int epi_smem_bytes(int bn) { return bn * 4 + EPI_RB_GROUPS * bn * 2; }   // per consumer warpgroup
// the two column ranges of the eight MODE 3 epilogue warps split the tile at a multiple of 32
__host__ __device__ constexpr int col_split(int bn) { return ((bn / 2 + 31) / 32) * 32; }

// Staged modes: the fp16 output columns of a tile (GEGLU halves them), and the TMA box width the output half tile of a
// warpgroup is cut into -- the widest of 64 / 32 / 16 columns that divides it, with the 128 / 64 / 32-byte swizzle of that
// row length.
__host__ __device__ constexpr int out_cols(int bn, int mode) { return mode == 1 ? bn / 2 : bn; }
__host__ __device__ constexpr int out_box(int ow) { return ow % 64 == 0 ? 64 : (ow % 32 == 0 ? 32 : 16); }
__host__ __device__ constexpr int out_half_bytes(int ow) { return 64 * ow * 2; }

// Byte offset of (row r, output column c) in a warpgroup's half tile: boxes of BOX columns x 64 rows, 2 BOX bytes per row,
// laid out as TMA's swizzle for that row length places them (16-byte chunk index ^= offset bits 7..).  The eight rows one
// fragment store of a warp touches then fall into eight different bank groups.
template <int BOX>
__device__ __forceinline__ uint32_t out_off(int r, int c) {
  const uint32_t o = (uint32_t)(r * (2 * BOX) + (c % BOX) * 2);
  return (uint32_t)(c / BOX) * (128 * BOX) + (o ^ (((o >> 7) & (BOX / 8 - 1)) << 4));
}
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 bits_h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }

// Called by a consumer warpgroup while its first k-block's MMAs run: the tile's bias slice and the row-group-bias slices
// of the warpgroup's rows [rm0, rm0 + 64) go to its shared-memory copy, so that the epilogue never waits on a first-touch
// global load.
template <int BN>
__device__ __forceinline__ void epilogue_preload(const GemmParams& p, int rm0, int n0, float* sbias, __half* srb, int tw) {
  for (int i = tw; i < BN; i += 128) sbias[i] = (p.bias && n0 + i < p.N) ? __ldg(p.bias + n0 + i) : 0.f;
  if (p.rowbias && rm0 < p.M) {
    const int g0 = rm0 / p.rows_per_group;
    const int last = (rm0 + 63 < p.M ? rm0 + 63 : p.M - 1) / p.rows_per_group;
    const int ng = last - g0 + 1;
    if (ng <= EPI_RB_GROUPS)
      for (int i = tw; i < ng * BN; i += 128) {
        const int gi = i / BN, c = i - gi * BN;
        srb[i] = (n0 + c < p.N) ? p.rowbias[(int64_t)(g0 + gi) * p.rowbias_ld + n0 + c] : __float2half(0.f);
      }
  }
}

template <int ACT>
__device__ __forceinline__ float act_fn(float x) {
  if (ACT == 1) return __fdividef(x, 1.f + __expf(-x));
  if (ACT == 2) return gelu_erf(x);
  if (ACT == 4) return __fdividef(x, 1.f + __expf(-1.702f * x));
  return x;
}

// Staged epilogue of one consumer thread (tw = its index in the warpgroup) on its m64nBN fragment d, whose element
// d[4 j + 2 h + e] is row 16 (tw / 32) + (tw % 32) / 4 + 8 h, tile column 8 j + 2 (tw % 4) + e of the warpgroup's rows:
// alpha / bias / row-group bias / activation (ACT 3: GEGLU gate) in fp32, rounded to fp16 (where autocast rounds the layer
// output), then the residual -- already in the half tile -- added in fp32 and rounded again.  rb[h]: row-group bias of the
// thread's row h indexed by tile column, nullptr for none; rb_global: it points to global memory (mind the N tail).
template <int BN, int MODE, int ACT>
__device__ __forceinline__ void epilogue_regs(const GemmParams& p, const float (&d)[BN / 2], uint32_t tile, int tw, int n0,
                                              const float* sbias, const __half* const (&rb)[2], bool rb_global) {
  constexpr int BOX = out_box(out_cols(BN, MODE));
  const int q = tw & 3, r = 16 * (tw >> 5) + ((tw & 31) >> 2);
  if constexpr (MODE == 1) {   // chunk k of 32 columns = 16 values + their 16 gates: a value and its gate sit in the same thread
#pragma unroll
    for (int k = 0; k < BN / 32; ++k)
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 4 * k + jj, c = 8 * j + 2 * q;
        const float2 bv = *reinterpret_cast<const float2*>(sbias + c), bg = *reinterpret_cast<const float2*>(sbias + c + 16);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float a0 = fmaf(d[4 * j + 2 * h], p.alpha, bv.x), a1 = fmaf(d[4 * j + 2 * h + 1], p.alpha, bv.y);
          const float g0 = fmaf(d[4 * (j + 2) + 2 * h], p.alpha, bg.x), g1 = fmaf(d[4 * (j + 2) + 2 * h + 1], p.alpha, bg.y);
          st_shared_u32(tile + out_off<BOX>(r + 8 * h, 16 * k + 8 * jj + 2 * q),
                        h2_bits(__floats2half2_rn(a0 * gelu_erf_fast(g0), a1 * gelu_erf_fast(g1))));
        }
      }
  } else {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * q;
    const float2 b = *reinterpret_cast<const float2*>(sbias + c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = b.x, v1 = b.y;
      if (rb[h] && (!rb_global || n0 + c < p.N)) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(rb[h] + c));
        v0 += f.x, v1 += f.y;
      }
      const float x0 = fmaf(d[4 * j + 2 * h], p.alpha, v0), x1 = fmaf(d[4 * j + 2 * h + 1], p.alpha, v1);
      __half2 o = __floats2half2_rn(act_fn<ACT>(x0), act_fn<ACT>(x1));
      const uint32_t a = tile + out_off<BOX>(r + 8 * h, c);
      if (p.residual) {
        const float2 fa = __half22float2(o), fb = __half22float2(bits_h2(ld_shared_u32(a)));
        o = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
      }
      st_shared_u32(a, h2_bits(o));
    }
  }
  }
}

// One thread of a consumer warpgroup moves its half tile (rows [rm0, rm0 + 64), output columns from ocol0) between shared
// memory and the output / residual tensor map, one TMA box of BOX columns at a time; boxes wholly past the last column are
// skipped, the map clips the rest.  A load first announces on `bar` exactly the bytes of the boxes it issues.  The
// up-sampling conv writes its phase (upa, upb) through the 5-D map [B H][2][W][2][N]: the half tile's 64 low-resolution
// pixels are one box of (W_tile, rows) (make_out_map).
template <int BOX, int NBOX, bool STORE>
__device__ __forceinline__ void out_tile_tma(const GemmParams& p, const CUtensorMap* map, uint8_t* tile, int rm0, int ocol0, int nout,
                                             uint64_t* bar) {
  const int nb = min(NBOX, (nout - ocol0 + BOX - 1) / BOX);
  if (!STORE) mbar_expect_tx(bar, (uint32_t)nb * (128 * BOX));
#pragma unroll
  for (int b = 0; b < NBOX; ++b) {
    if (b >= nb) break;
    const int c = ocol0 + b * BOX;
    uint8_t* s = tile + b * (128 * BOX);
    if (!STORE) tma_load_2d(s, map, bar, c, rm0);
    else if (p.up) tma_store_5d(map, s, c, p.upb, rm0 % p.cW, p.upa, rm0 / p.cW);
    else tma_store_2d(map, s, c, rm0);
  }
}

constexpr int smem_bytes(int bn, int stages, int mode) {
  return stages * (BM * BK * 2 + bn * BK * 2) + (mode == 3 ? 0 : 2 * out_half_bytes(out_cols(bn, mode))) + (2 * stages + 2) * 8 + 16 +
         2 * epi_smem_bytes(bn) + 1024;
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

// MODE 3: a warpgroup's m64nBN accumulator fragment -> rows [row0, row0 + 64) of the shared-memory accumulator tile
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
// tmC / tmR (staged modes): the fp16 output and the residual seen in boxes of one warpgroup's half tile (make_out_map)
template <int BN, int STAGES, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
               const __grid_constant__ CUtensorMap tmR, const __grid_constant__ GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by SWIZZLE_128B
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
  static_assert(B_BYTES % 1024 == 0, "stage bases must stay 1024-byte aligned for SWIZZLE_128B");
  static_assert(BN % 32 == 0 && BN >= 64 && BN <= 256, "tile width: a multiple of 32 (GEGLU chunks, 32-column epilogue reads)");
  static_assert(BM * acc_ld(BN) * 4 <= STAGES * (A_BYTES + B_BYTES), "the accumulator tile must fit in the operand ring");
  constexpr int CSPLIT = col_split(BN);
  constexpr int OW = out_cols(BN, MODE), BOX = out_box(OW), OUT_HALF = out_half_bytes(OW);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint8_t* sOut = sB + STAGES * B_BYTES;                      // staged modes: one fp16 half tile per consumer warpgroup
  uint64_t* full = reinterpret_cast<uint64_t*>(sOut + (MODE == 3 ? 0 : 2 * OUT_HALF));
  uint64_t* empty = full + STAGES;
  uint64_t* resbar = empty + STAGES;                          // per consumer warpgroup: its residual half tile has landed
  float* sbias = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(resbar + 2) + 15) & ~(uintptr_t)15);   // [2][BN]
  __half* srb = reinterpret_cast<__half*>(sbias + 2 * BN);                                                     // [2][8 BN]
  float* acc = reinterpret_cast<float*>(smem);                // MODE 3: the operand ring, once the K loop is done

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
    if (MODE != 3) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmC) : "memory");
    for (int s = 0; s < STAGES; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 2);   // empty: one arrival per MMA warpgroup
    mbar_init(resbar, 1), mbar_init(resbar + 1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
  }
  __syncthreads();
  pdl_wait();      // everything above touched no global memory: it overlaps the tail of the previous kernel
  pdl_trigger();
  if (threadIdx.x == 0) stamp(p, 1);

  // Tiles of this CTA: one (blockIdx.x, blockIdx.y), or -- persistent launch (p.persist, staged epilogues only) -- tiles
  // blockIdx.x, blockIdx.x + gridDim.x, ... of the column-major tile order.  The ring's stage / phase counters run on across
  // tiles, so the producer fills the next tile's first stages as soon as the last MMA of a tile has released its stage.
  const int tiles_m = (p.M + BM - 1) / BM, tiles = tiles_m * ((p.N + BN - 1) / BN);
  const bool persist = MODE != 3 && p.persist;
  uint32_t cnt = 0;       // k-blocks consumed so far by this CTA
  uint32_t rphase = 0;    // residual half tiles this warpgroup has loaded so far (parity of resbar)
  for (int t = persist ? blockIdx.x : blockIdx.y * tiles_m + blockIdx.x; t < tiles; t += persist ? gridDim.x : tiles) {
  const int m0 = (t % tiles_m) * BM, n0 = (t / tiles_m) * BN;
  if (warp < 4) {
    if (threadIdx.x == 0) {  // ---------------- TMA producer
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
    const int wg = (warp >> 2) - 1, e = warp - 4, quarter = e & 3, te = threadIdx.x - 128, tw = threadIdx.x & 127;
    // staged modes: this warpgroup's rows, output columns, half tile and bias slices
    const int rm0 = m0 + 64 * wg, ocol0 = MODE == 1 ? n0 / 2 : n0, nout = MODE == 1 ? p.N / 2 : p.N;
    const bool rows = rm0 < p.M;
    uint8_t* tile = sOut + wg * OUT_HALF;
    float* wbias = sbias + wg * BN;
    __half* wrb = srb + wg * EPI_RB_GROUPS * BN;
    {
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t c = cnt + (kb - kb0);
        const int s = c % STAGES;
        const uint32_t ph = (c / STAGES) & 1;
        mbar_wait(full + s, ph, p, WAIT_FULL, s);
        if (kb == kb0 && te == 0) {
          if (p.trace && t != (int)blockIdx.x && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) p.trace[9] = p.trace[5];
          stamp(p, 4);
        }
        const uint32_t a0 = smem_u32(sA + s * A_BYTES) + wg * (64 * 128), b0 = smem_u32(sB + s * B_BYTES);
        wg::fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)   // advancing 16 fp16 along K inside the 128-byte swizzle atom = +32 bytes on the start address
          wg::mma_f16<BN>(d, wg::desc_sw128(a0 + k * 32), wg::desc_sw128(b0 + k * 32), 1);
        wg::commit();
        if (MODE != 3 && kb == kb0) {
          // under the first k-block's MMAs: once the previous tile's store has read the half tile, the residual is loaded
          // into it; the bias slices are refreshed (the previous epilogue is done with them: it ended at a wg_bar)
          if (tw == 0) {
            bulk_wait_read();
            if (p.residual && rows) out_tile_tma<BOX, OW / BOX, false>(p, &tmR, tile, rm0, ocol0, nout, resbar + wg);
          }
          epilogue_preload<BN>(p, rm0, n0, wbias, wrb, tw);
          wg_bar(wg);
        }
        wg::wait<1>();                      // the previous stage's MMAs are done: hand that stage back to the producer
        if (kb > kb0 && tw == 0) mbar_arrive(empty + (c - 1) % STAGES);
      }
      wg::wait<0>();
      if (tw == 0) mbar_arrive(empty + (cnt + kb1 - kb0 - 1) % STAGES);   // the ring is the producer's again
      if (te == 0) stamp(p, 5);
      if (MODE != 3) {
        if (rows) {
          if (p.residual) mbar_wait(resbar + wg, rphase & 1, p, WAIT_RESIDUAL, wg);
          if (te == 0) stamp(p, 6);
          // row-group bias of the thread's two rows: from the smem copy when the warpgroup's rows span few groups
          const __half* rb[2] = {nullptr, nullptr};
          bool rb_global = false;
          if (MODE != 1 && p.rowbias) {
            const int g0 = rm0 / p.rows_per_group, last = (rm0 + 63 < p.M ? rm0 + 63 : p.M - 1) / p.rows_per_group;
            rb_global = last - g0 + 1 > EPI_RB_GROUPS;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = rm0 + 16 * (tw >> 5) + ((tw & 31) >> 2) + 8 * h, g = (row < p.M ? row : p.M - 1) / p.rows_per_group;
              rb[h] = rb_global ? p.rowbias + (int64_t)g * p.rowbias_ld + n0 : wrb + (g - g0) * BN;
            }
          }
          const uint32_t ts = smem_u32(tile);
          if constexpr (MODE == 0) {
            epilogue_regs<BN, 0, 0>(p, d, ts, tw, n0, wbias, rb, rb_global);
          } else if constexpr (MODE == 1) {
            epilogue_regs<BN, 1, 3>(p, d, ts, tw, n0, wbias, rb, rb_global);
          } else {   // the activation switch is hoisted out of the element loops: one branch per tile
            switch (p.act) {
              case 1: epilogue_regs<BN, 2, 1>(p, d, ts, tw, n0, wbias, rb, rb_global); break;
              case 2: epilogue_regs<BN, 2, 2>(p, d, ts, tw, n0, wbias, rb, rb_global); break;
              default: epilogue_regs<BN, 2, 4>(p, d, ts, tw, n0, wbias, rb, rb_global); break;
            }
          }
          fence_proxy_async();              // the half tile's generic writes, before the TMA store reads it
          wg_bar(wg);
          if (tw == 0) {
            out_tile_tma<BOX, OW / BOX, true>(p, &tmC, tile, rm0, ocol0, nout, nullptr);
            bulk_commit();
          }
          if (p.residual) ++rphase;
        }
      } else {
        epi_bar();                          // both warpgroups are done reading the ring: it becomes the accumulator tile
        acc_store<BN>(acc, d, 64 * wg, tw);
      }
    }
    if (MODE == 3) {
      epi_bar();
      if (te == 0) stamp(p, 6);
      const float* acc_row = acc + (quarter * 32 + lane) * acc_ld(BN);
      const int c_lo = e < 4 ? 0 : CSPLIT, c_hi = e < 4 ? CSPLIT : BN;   // this warp's tile columns
      const int row = m0 + quarter * 32 + lane;
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
  if (MODE == 3) __syncthreads();   // one tile per CTA: the accumulator tile is done with before the split-K exchange
  }
  if (MODE != 3 && warp >= 4 && (threadIdx.x & 127) == 0) bulk_wait();   // the last half tile is in global memory
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

// Staged modes: the fp16 output (or residual) [M rows, nout columns, row stride ldc] in boxes of `box` columns x 64 rows, one
// consumer warpgroup's half tile, with the swizzle out_off() lays the half tile out in.  Rows past M and columns past nout
// are clipped by the map (stores) or zero-filled (loads).  The up-sampling conv's phase (upa, upb) scatters low-resolution
// pixel (b, y, x) to output row (2 (b H + y) + upa) 2 W + 2 x + upb: a 5-D view [B H][2][W][2][nout] whose box is
// (box, 1, W_tile, 1, 64 / W_tile) with W_tile = min(W, 64) -- the half tile's 64 consecutive pixels.
int make_out_map(CUtensorMap* m, const void* ptr, const GemmParams& p, int nout, int box) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return O2345_ECUDA; }
  const CUtensorMapSwizzle sw = box == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (box == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  const cuuint64_t row = (cuuint64_t)p.ldc * 2;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r;
  if (p.up) {
    // a half tile's 64 consecutive pixels are whole rows of W_tile pixels only when W divides 64 or is a multiple of it
    // (conv_tiles() admits W that divide 128 or are multiples of 128); any other W would scatter wrong rows
    O2345_CHECK_ARG(64 % p.cW == 0 || p.cW % 64 == 0, "up-sampling conv output map: W must divide 64 or be a multiple of 64");
    const int wt = p.cW < 64 ? p.cW : 64;
    cuuint64_t dims[5] = {(cuuint64_t)nout, 2, (cuuint64_t)p.cW, 2, (cuuint64_t)(p.M / p.cW)};
    cuuint64_t strides[4] = {row, 2 * row, 2 * (cuuint64_t)p.cW * row, 4 * (cuuint64_t)p.cW * row};
    cuuint32_t boxd[5] = {(cuuint32_t)box, 1, (cuuint32_t)wt, 1, (cuuint32_t)(64 / wt)};
    r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(ptr), dims, strides, boxd, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    cuuint64_t dims[2] = {(cuuint64_t)nout, (cuuint64_t)p.M};
    cuuint64_t strides[1] = {row};
    cuuint32_t boxd[2] = {(cuuint32_t)box, 64};
    r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, boxd, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (GEMM output) failed with %d (M=%d nout=%d ldc=%lld)", (int)r, p.M, nout, (long long)p.ldc); return O2345_ECUDA; }
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
// small cost model.  A batch-64 tools/gemm_sweep.py on an H100 (DESIGN section 6) found no other constants that pick faster
// configurations without changing a split count, and a split count that changes regroups the fp32 partial sums, i.e. the
// layer's rounding:
//   * a launch costs ~5 us of fixed latency (launch, prologue, first TMA round trip, tear-down) + ~3 us of epilogue per
//     160 columns of tile and wave of CTAs; the main loop's cycles are converted at 1 750 cycles per us;
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
  // Two or more waves of tiles: one CTA per SM walks them, so that launch, prologue and the wave tail are paid once per SM
  // and the next tile's loads run under the previous tile's epilogue (tools/gemm_persist_ab.py, DESIGN section 6)
  const int tiles = cdiv(M, BM) * cdiv(N, c.bn);
  const int min_tiles = g_persist_min_tiles > 0 ? g_persist_min_tiles : 2 * sm_count();
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
  constexpr int SMEM = smem_bytes(BN, STAGES, MODE);
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
  CUtensorMap mc, mr;
  memset(&mc, 0, sizeof(mc)), memset(&mr, 0, sizeof(mr));
  if (MODE != 3) {
    constexpr int OW = out_cols(BN, MODE);
    O2345_TRY(make_out_map(&mc, p.C, p, p.act == 3 ? p.N / 2 : p.N, out_box(OW)));
    if (p.residual) O2345_TRY(make_out_map(&mr, p.residual, p, p.N, out_box(OW)));
  }
  O2345_CUDA(launch_pdl_cluster(gemm_tc_kernel<BN, STAGES, MODE>, grid, dim3(GEMM_THREADS), (size_t)SMEM, st, 1, splits, a, b, mc, mr, p));
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

// ring depth per tile width: as many stages as fit next to the two output half tiles in 227 KB (one CTA per SM)
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
                                "residual (epilogue waiting for the TMA load of its residual half tile)"};
  snprintf(buf, n,
           "gemm_tc_kernel<BN=%d, MODE=%d> M=%d N=%d K=%d conv=%d splits=%d: CTA (%d,%d,%d) rank %d gave up after 4 s "
           "on barrier '%s' stage %d",
           d->bn, d->mode, d->M, d->N, d->K, d->conv, d->splits, d->bx, d->by, d->bz, d->rank,
           names[d->tag >= 1 && d->tag <= 3 ? d->tag : 0], d->stage);
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
