// View-blending network on the Hopper warpgroup MMA (wgmma.mma_async, fp32 accumulators in registers): precision =
// O2345_BLEND_TC5.  SURVEY.md rows B11 / B12, the hot kernel of the ray march (section 8(d)); same function as
// render_blend_kernel (render.cu, reference reconstruction/models/rendering_network.py:75-129 fused with the Projector's
// per-view fetch, projector.py:96-228).
//
// The per-(sample, view) MLPs as register-chained mma.sync products (render_tc.cu) are instruction-fetch / issue bound.  Here a
// CTA -- one warpgroup -- owns a 128-row tile = 4 samples x 32 view slots: a warp is one sample and a LANE IS ONE SOURCE VIEW,
// which is also the accumulator row it reads back, so
//   * the projection, the validity mask, the ray difference, the pooling weight and every per-sample reduction over the views
//     (weighted mean / variance, soft-max) are plain per-lane values and warp shuffles -- no compaction, no fragment layouts;
//   * each thread gathers the 59 channels of ITS view (4 bilinear taps x 240 contiguous bytes) into registers;
//   * the seven wide layers (16->64, 64->64, 64->32, 32->32, 32->33, 32->32, 37->16) are M = 128 wgmma products (two m64
//     instructions per k-step): the thread writes its fp16 activation row into a SWIZZLE_128B shared-memory operand, the
//     warpgroup multiplies it by weights resident in shared memory, the accumulator fragments go to an fp32 row buffer and
//     each thread reads back ITS row; the narrow layers (4->16, 32->1, 16->8->1) stay on the FMA pipe;
//   * the per-sample part of base_fc ([geo | mean | var] -> 64, identical for the 32 views) is computed once per sample and
//     added when the accumulator is read.
// Numerics as render_tc.cu: features, statistics, soft-max and the colour blend in fp32, MMA operands rounded to fp16.
#include <cuda_fp16.h>

#include "common.cuh"
#include "render_pack.cuh"
#include "wgmma.cuh"

namespace o2345 {
namespace {
using namespace rpack;

constexpr int T5_THREADS = 128;          // one warpgroup; warp = sample, lane = view
constexpr int ST_LD = 65;                // floats per row of the fp32 accumulator / feature rows (odd stride: conflict-free row access)

// ---- shared memory map (bytes from the 1024-byte aligned base)
constexpr int W_D1 = 0;                      // ray_dir_fc[2]   [64 n][64 k] (k < 16 used)  SWIZZLE_128B K-major
constexpr int W_B0 = W_D1 + 64 * 128;        // base_fc[0], per-view part [64][64] (k < 59)
constexpr int W_B1 = W_B0 + 64 * 128;        // base_fc[2]      [32][64]
constexpr int W_V0 = W_B1 + 32 * 128;        // vis_fc[0]       [32][64] (k < 32)
constexpr int W_V1 = W_V0 + 32 * 128;        // vis_fc[2]       [48][64]: rows 0..31 residual, row 32 visibility (k < 32)
constexpr int W_U0 = W_V1 + 48 * 128;        // vis_fc2[0]      [32][64] (k < 32)
constexpr int W_R0 = W_U0 + 32 * 128;        // rgb_fc[0]       [16][64] (k < 37: x 0..31 | vis 32 | ray_diff 33..36)
constexpr int A_BUF = W_R0 + 16 * 128;       // activation operand [128 rows][64 k] fp16, SWIZZLE_128B
constexpr int S_PS = A_BUF + 128 * 128;      // base_fc[0], per-sample part, fp16 [134 k][64 n] (k: geo 0..15 | mean 16..74 | var 75..133)
constexpr int S_F32 = S_PS + 134 * 64 * 2;   // small fp32 vectors (below)
// fp32 block (float offsets)
constexpr int F_D0W = 0, F_D0B = 64, F_D1B = 80, F_B0B = 144, F_B1B = 208, F_V0B = 240, F_V1B = 272 /* 32 + visibility bias */,
              F_U0B = 320, F_U1W = 352, F_U1B = 384, F_R0B = 388, F_R1W = 404 /* [16][8] */, F_R1B = 532, F_R2W = 540, F_R2B = 548,
              F_S = 549, F_TOTAL = 552;
constexpr int S_STAGE = S_F32 + F_TOTAL * 4;             // fp32 rows [128][ST_LD]: the accumulator of a round, a warp's features
constexpr int S_VEC = S_STAGE + 4 * 32 * ST_LD * 4;      // per-warp [134] geo|mean|var + [64] per-sample base_fc part + [32] pooling weights
constexpr int VEC_F = 134 + 64 + 32 + 2;
constexpr int T5_SMEM = S_VEC + 4 * VEC_F * 4 + 1024;   // + alignment slack
static_assert(A_BUF % 1024 == 0 && W_B0 % 1024 == 0 && W_B1 % 1024 == 0 && W_V0 % 1024 == 0 && W_V1 % 1024 == 0 && W_U0 % 1024 == 0 &&
              W_R0 % 1024 == 0, "SWIZZLE_128B operands start on 1024-byte boundaries");
static_assert(S_F32 % 16 == 0 && S_STAGE % 4 == 0, "alignment");
static_assert(2 * T5_SMEM <= 227 * 1024, "two CTAs per SM");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float ex2_(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float elu_(float x) {
  const float e = ex2_(fminf(x, 0.f) * 1.4426950408889634f) - 1.f;
  return x > 0.f ? x : e;
}
__device__ __forceinline__ float sigm_(float x) { return __fdividef(1.f, 1.f + ex2_(-1.4426950408889634f * x)); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// K-major SWIZZLE_128B operand: element (row, k) of a [rows][64] fp16 matrix lives at
//   (row / 8) * 1024 + (row % 8) * 128 + (((k / 8) ^ (row % 8)) * 16) + (k % 8) * 2
__device__ __forceinline__ uint32_t sw128_off(int row, int k) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7))) << 4) + ((k & 7) << 1));
}
// the first NC columns of this thread's accumulator row
template <int NC>
__device__ __forceinline__ void acc_row(const float* row, float (&v)[NC]) {
#pragma unroll
  for (int i = 0; i < NC; ++i) v[i] = row[i];
}

// fp32 [in][out] pack -> fp16 [n][64] SWIZZLE_128B operand; rows >= n_used / columns >= k_used are zero
__device__ void fill_operand(uint8_t* dst, int n_rows, const float* __restrict__ src, int src_ld, int n_used, int k_used, int tid,
                             int nthreads) {
  for (int i = tid; i < n_rows * 64; i += nthreads) {
    const int nrow = i >> 6, k = i & 63;
    const float v = (nrow < n_used && k < k_used) ? __ldg(src + (int64_t)k * src_ld + nrow) : 0.f;
    *reinterpret_cast<__half*>(dst + sw128_off(nrow, k)) = __float2half_rn(v);
  }
}

// one thread's activation row: NK fp32 values -> fp16, written as 16-byte chunks of the swizzled operand
template <int NK>
__device__ __forceinline__ void write_row(uint8_t* abuf, int row, const float (&x)[NK]) {
  static_assert(NK % 8 == 0, "whole 16-byte chunks");
#pragma unroll
  for (int c = 0; c < NK / 8; ++c) {
    __half2 h[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(x[8 * c + 2 * e], x[8 * c + 2 * e + 1]);
    *reinterpret_cast<uint4*>(abuf + (row >> 3) * 1024 + (row & 7) * 128 + ((c ^ (row & 7)) << 4)) = *reinterpret_cast<uint4*>(h);
  }
}

// One layer for the whole tile: every thread has written its operand row -> accumulator [128 rows][N] = A . W^T over
// KSTEPS x 16 inputs (two m64 halves) -> fragments into the fp32 row buffer -> every thread may read its row.
template <int N, int KSTEPS>
__device__ __forceinline__ void mma_round(uint32_t a_addr, uint32_t b_addr, float* rows, int tid) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");          // generic-proxy stores -> visible to the tensor core's reads
  __syncthreads();                                                      // every row written, every previous accumulator row read
  float d0[N / 2], d1[N / 2];
  wg::fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    wg::mma_f16<N>(d0, wg::desc_sw128(a_addr + k * 32), wg::desc_sw128(b_addr + k * 32), k);
    wg::mma_f16<N>(d1, wg::desc_sw128(a_addr + 64 * 128 + k * 32), wg::desc_sw128(b_addr + k * 32), k);
  }
  wg::commit();
  wg::wait<0>();
  const int r = 16 * (tid >> 5) + ((tid & 31) >> 2), c = 2 * (tid & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    float* p = rows + r * ST_LD + 8 * j + c;
    p[0] = d0[4 * j], p[1] = d0[4 * j + 1], p[8 * ST_LD] = d0[4 * j + 2], p[8 * ST_LD + 1] = d0[4 * j + 3];
    p += 64 * ST_LD;
    p[0] = d1[4 * j], p[1] = d1[4 * j + 1], p[8 * ST_LD] = d1[4 * j + 2], p[8 * ST_LD + 1] = d1[4 * j + 3];
  }
  __syncthreads();
}

__device__ __forceinline__ void sample_point(const o2345_points& src, int64_t gi, float& x, float& y, float& z) {
  if (src.mode == O2345_PTS_EXPLICIT) {
    x = __ldg(src.pts + 3 * gi), y = __ldg(src.pts + 3 * gi + 1), z = __ldg(src.pts + 3 * gi + 2);
  } else {
    int64_t r = gi / src.S;
    int s = (int)(gi - r * src.S);
    float t = __ldg(src.z + r * src.z_stride + s);
    x = __fadd_rn(__ldg(src.rays_o + 3 * r), __fmul_rn(__ldg(src.rays_d + 3 * r), t));
    y = __fadd_rn(__ldg(src.rays_o + 3 * r + 1), __fmul_rn(__ldg(src.rays_d + 3 * r + 1), t));
    z = __fadd_rn(__ldg(src.rays_o + 3 * r + 2), __fmul_rn(__ldg(src.rays_d + 3 * r + 2), t));
  }
}

__global__ void __launch_bounds__(T5_THREADS, 2)
render_blend_t5_kernel(o2345_points src, int64_t n, const uint8_t* __restrict__ active, const float* __restrict__ vol,
                       const float* __restrict__ occ, int D, o2345_views views, int dir_mode,
                       const float* __restrict__ query_center, const float* __restrict__ dirs,
                       const float* __restrict__ pack, float* __restrict__ rgb_out, int32_t* __restrict__ nvalid_out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* sF = reinterpret_cast<float*>(sm + S_F32);
  __half* sPS = reinterpret_cast<__half*>(sm + S_PS);
  const int tid = threadIdx.x, nth = blockDim.x, lane = tid & 31, warp = tid >> 5;

  // ---- weights: the seven MMA operands, the per-sample part of base_fc[0], the small fp32 vectors
  fill_operand(sm + W_D1, 64, pack + P_D1W, 64, 64, 16, tid, nth);
  fill_operand(sm + W_B0, 64, pack + P_B0W + 134 * 64, 64, 64, NF, tid, nth);
  fill_operand(sm + W_B1, 32, pack + P_B1W, 32, 32, 64, tid, nth);
  fill_operand(sm + W_V0, 32, pack + P_V0W, 32, 32, 32, tid, nth);
  fill_operand(sm + W_V1, 48, pack + P_V1W, 32, 32, 32, tid, nth);
  fill_operand(sm + W_U0, 32, pack + P_U0W, 32, 32, 32, tid, nth);
  fill_operand(sm + W_R0, 16, pack + P_R0W, 16, 16, 37, tid, nth);
  for (int i = tid; i < 134 * 64; i += nth) sPS[i] = __float2half_rn(__ldg(pack + P_B0W + i));
  for (int i = tid; i < F_TOTAL; i += nth) {
    float v = 0.f;
    if (i < F_D0B) v = pack[P_D0W + i];
    else if (i < F_D1B) v = pack[P_D0B + i - F_D0B];
    else if (i < F_B0B) v = pack[P_D1B + i - F_D1B];
    else if (i < F_B1B) v = pack[P_B0B + i - F_B0B];
    else if (i < F_V0B) v = pack[P_B1B + i - F_B1B];
    else if (i < F_V1B) v = pack[P_V0B + i - F_V0B];
    else if (i < F_U0B) v = i - F_V1B < 32 ? pack[P_V1B + i - F_V1B] : (i - F_V1B == 32 ? pack[P_V1VB] : 0.f);
    else if (i < F_U1W) v = pack[P_U0B + i - F_U0B];
    else if (i < F_U1B) v = pack[P_U1W + i - F_U1W];
    else if (i < F_R0B) v = i == F_U1B ? pack[P_U1B] : 0.f;
    else if (i < F_R1W) v = pack[P_R0B + i - F_R0B];
    else if (i < F_R1B) v = pack[P_R1W + i - F_R1W];
    else if (i < F_R2W) v = pack[P_R1B + i - F_R1B];
    else if (i < F_R2B) v = pack[P_R2W + i - F_R2W];
    else if (i == F_R2B) v = pack[P_R2B];
    else if (i == F_S) v = pack[P_S];
    sF[i] = v;
  }
  __syncthreads();
  for (int k = tid; k < 32; k += nth)   // visibility row of vis_fc[2]
    *reinterpret_cast<__half*>(sm + W_V1 + sw128_off(32, k)) = __float2half_rn(__ldg(pack + P_V1V + k));
  const uint32_t a_addr = smem_u32(sm + A_BUF);
  const int64_t groups = (n + 3) >> 2;

  {
    // ---------------- seven wgmma rounds per group of four samples
    const int row = warp * 32 + lane;                                   // operand row = accumulator row
    float* rows = reinterpret_cast<float*>(sm + S_STAGE);
    const float* myrow = rows + row * ST_LD;
    uint8_t* abuf = sm + A_BUF;
    float* stage = rows + warp * 32 * ST_LD;                            // this warp's rows (features between rounds 1 and 2)
    float* svec = reinterpret_cast<float*>(sm + S_VEC) + warp * VEC_F;  // [0,134) geo|mean|var, [134,198) per-sample base_fc part, [198,230) weights
    const int V = views.V, H = views.H, W = views.W;
    const float abs_s = sF[F_S];
    for (int64_t grp = blockIdx.x; grp < groups; grp += gridDim.x) {
      const int64_t gi = grp * 4 + warp;
      const bool live = gi < n && !(active && active[gi] == 0);
      float px = 0.f, py = 0.f, pz = 0.f;
      if (gi < n) sample_point(src, gi, px, py, pz);
      // ---- geometry feature (ATen trilinear, zeros padding, align_corners=True) + occupancy: as render_blend_kernel
      float geo = 0.f, occv = 0.f;
      if (live) {
        float p[3] = {px, py, pz};
        float f[3], w1[3];
        bool fin = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          float tt = ((p[a] + 1.f) / 2.f) * (float)(D - 1);
          f[a] = floorf(tt);
          w1[a] = tt - f[a];
          fin = fin && (f[a] >= -1.f) && (f[a] <= (float)(D - 1));
        }
        if (fin) {
#pragma unroll
          for (int corner = 0; corner < 8; ++corner) {
            int dx = corner >> 2, dy = (corner >> 1) & 1, dz = corner & 1;
            int ix = (int)f[0] + dx, iy = (int)f[1] + dy, iz = (int)f[2] + dz;
            if (ix < 0 || iy < 0 || iz < 0 || ix >= D || iy >= D || iz >= D) continue;
            float w = (dx ? w1[0] : 1.f - w1[0]) * (dy ? w1[1] : 1.f - w1[1]) * (dz ? w1[2] : 1.f - w1[2]);
            int64_t cell = ((int64_t)ix * D + iy) * D + iz;
            if (lane < 16) geo = fmaf(__ldg(vol + cell * 16 + lane), w, geo);
            occv = fmaf(__ldg(occ + cell), w, occv);
          }
        }
      }
      const bool gmask = live && (fabsf(px) < 1.f) && (fabsf(py) < 1.f) && (fabsf(pz) < 1.f) && (occv > 0.f);
      // ---- lane = view: projection, mask, ray difference, pooling weight
      float gx = 2.f, gy = 2.f, rd[4] = {0.f, 0.f, 0.f, 0.f}, ev = 3.4e38f;
      bool vmask = false;
      if (live) {
        float tx, ty, tz;
        if (dir_mode == 0) {
          tx = query_center[0] - px, ty = query_center[1] - py, tz = query_center[2] - pz;
          float nn = sqrtf(tx * tx + ty * ty + tz * tz) + 1e-6f;
          tx /= nn, ty /= nn, tz /= nn;
        } else {
          tx = dirs[3 * gi], ty = dirs[3 * gi + 1], tz = dirs[3 * gi + 2];
        }
        if (lane < V) {
          const float* P = views.proj + 12 * lane;
          float X = P[0] * px + P[1] * py + P[2] * pz + P[3];
          float Y = P[4] * px + P[5] * py + P[6] * pz + P[7];
          float Z = fmaxf(P[8] * px + P[9] * py + P[10] * pz + P[11], 1e-3f);
          gx = 2.f * (X / Z) / (views.sizeW - 1.f) - 1.f;
          gy = 2.f * (Y / Z) / (views.sizeH - 1.f) - 1.f;
          if (!(gx <= 1.f && gx >= -1.f)) gx = 2.f;
          if (!(gy <= 1.f && gy >= -1.f)) gy = 2.f;
          vmask = gmask && (fabsf(gx) < 1.f) && (fabsf(gy) < 1.f);
          float cx = views.centers[3 * lane] - px, cy = views.centers[3 * lane + 1] - py, cz = views.centers[3 * lane + 2] - pz;
          float nn = sqrtf(cx * cx + cy * cy + cz * cz) + 1e-6f;
          cx /= nn, cy /= nn, cz /= nn;
          float ddx = tx - cx, ddy = ty - cy, ddz = tz - cz;
          float dn = fmaxf(sqrtf(ddx * ddx + ddy * ddy + ddz * ddz), 1e-6f);
          rd[0] = ddx / dn, rd[1] = ddy / dn, rd[2] = ddz / dn;
          rd[3] = tx * cx + ty * cy + tz * cz;
          ev = expf(abs_s * (rd[3] - 1.f));
        }
      }
      float emin = ev;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) emin = fminf(emin, __shfl_xor_sync(0xffffffffu, emin, o));
      float wv = vmask ? (ev - emin) : 0.f;
      const float wtot = warp_sum(wv);
      wv = wv / (wtot + 1e-8f);
      const int nvalid = __popc(__ballot_sync(0xffffffffu, vmask));
      if (gi < n) {
        if (lane == 0 && nvalid_out) nvalid_out[gi] = live ? nvalid : 0;
        if (!live && lane < 3) rgb_out[3 * gi + lane] = 0.f;   // weight of this sample is exactly 0 in the compositing
      }
      if (live && nvalid == 0) {
        // every logit is -1e9: softmax is uniform over ALL views (reference rendering_network.py:119-121)
        float acc = 0.f;
        for (int v = 0; v < V; ++v) {
          float vgx = __shfl_sync(0xffffffffu, gx, v), vgy = __shfl_sync(0xffffffffu, gy, v);
          float fx = ((vgx + 1.f) / 2.f) * (float)(W - 1), fy = ((vgy + 1.f) / 2.f) * (float)(H - 1);
          float x0 = floorf(fx), y0 = floorf(fy);
          if (!(x0 >= -1.f && x0 <= (float)(W - 1) && y0 >= -1.f && y0 <= (float)(H - 1)) || lane >= 3) continue;
          int ix = (int)x0, iy = (int)y0;
          const float* m = views.maps + (int64_t)v * H * W * CM;
#pragma unroll
          for (int tap = 0; tap < 4; ++tap) {
            int xx = ix + (tap & 1), yy = iy + (tap >> 1);
            if (xx < 0 || xx > W - 1 || yy < 0 || yy > H - 1) continue;
            float wq = ((tap & 1) ? fx - x0 : x0 + 1.f - fx) * ((tap >> 1) ? fy - y0 : y0 + 1.f - fy);
            acc = fmaf(__ldg(m + ((int64_t)yy * W + xx) * CM + lane), wq, acc);
          }
        }
        if (lane < 3) rgb_out[3 * gi + lane] = acc / (float)V;
      }
      const bool run = live && nvalid > 0;          // warp-uniform: this sample goes through the network

      // ---- my view's 59 channels: four bilinear taps of 240 contiguous bytes each
      float rf[60];
#pragma unroll
      for (int c = 0; c < 60; ++c) rf[c] = 0.f;
      if (vmask) {
        const float fx = ((gx + 1.f) / 2.f) * (float)(W - 1), fy = ((gy + 1.f) / 2.f) * (float)(H - 1);
        const float x0 = floorf(fx), y0 = floorf(fy);
        const int ix = (int)x0, iy = (int)y0;
        const float* m = views.maps + (int64_t)lane * H * W * CM;
#pragma unroll
        for (int tap = 0; tap < 4; ++tap) {
          const int xx = ix + (tap & 1), yy = iy + (tap >> 1);
          if (xx < 0 || xx > W - 1 || yy < 0 || yy > H - 1) continue;
          const float wq = ((tap & 1) ? fx - x0 : x0 + 1.f - fx) * ((tap >> 1) ? fy - y0 : y0 + 1.f - fy);
          const float4* tp = reinterpret_cast<const float4*>(m + ((int64_t)yy * W + xx) * CM);
#pragma unroll
          for (int i = 0; i < 15; ++i) {
            const float4 v = __ldg(tp + i);
            rf[4 * i] = fmaf(v.x, wq, rf[4 * i]), rf[4 * i + 1] = fmaf(v.y, wq, rf[4 * i + 1]);
            rf[4 * i + 2] = fmaf(v.z, wq, rf[4 * i + 2]), rf[4 * i + 3] = fmaf(v.w, wq, rf[4 * i + 3]);
          }
        }
      }
      const float rgb_in[3] = {rf[0], rf[1], rf[2]};

      // ---- round 1: direction feature  ELU(D1 . ELU(D0 . rd + b0) + b1), added to the fetched feature
      {
        float h16[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float a = sF[F_D0B + j];
#pragma unroll
          for (int i = 0; i < 4; ++i) a = fmaf(sF[F_D0W + 16 * i + j], rd[i], a);
          h16[j] = elu_(a);
        }
        if (run) write_row<16>(abuf, row, h16);
      }
      mma_round<64, 1>(a_addr, smem_u32(sm + W_D1), rows, tid);
      {
        float d[32];
        acc_row<32>(myrow + 0, d);
#pragma unroll
        for (int c = 0; c < 32; ++c) rf[c] = vmask ? rf[c] + elu_(d[c] + sF[F_D1B + c]) : 0.f;
        acc_row<32>(myrow + 32, d);
#pragma unroll
        for (int c = 0; c < 27; ++c) rf[32 + c] = vmask ? rf[32 + c] + elu_(d[c] + sF[F_D1B + 32 + c]) : 0.f;
        rf[59] = 0.f;
      }
      // ---- weighted mean / variance over the views (lanes), the per-sample part of base_fc[0]
      if (run) {
#pragma unroll
        for (int c = 0; c < 59; ++c) stage[lane * ST_LD + c] = rf[c];
        svec[198 + lane] = wv;
        if (lane < 16) svec[lane] = geo;
        __syncwarp();
        const float wsum1 = wtot / (wtot + 1e-8f);
#pragma unroll
        for (int half_ = 0; half_ < 2; ++half_) {
          const int c = lane + 32 * half_;
          if (c < 59) {
            float s1 = 0.f, s2 = 0.f;
            for (int v = 0; v < 32; ++v) {
              const float w = svec[198 + v], x = stage[v * ST_LD + c];
              s1 = fmaf(w, x, s1), s2 = fmaf(w * x, x, s2);
            }
            svec[16 + c] = s1;
            svec[75 + c] = fmaxf(s2 - s1 * s1 * (2.f - wsum1), 0.f);     // sum_v w (f - mean)^2 = sum_v w f^2 - mean^2 (2 - sum_v w)
          }
        }
        __syncwarp();
        float p0 = sF[F_B0B + 2 * lane], p1 = sF[F_B0B + 2 * lane + 1];
        for (int k = 0; k < 134; ++k) {
          const float s = svec[k];
          const float2 w2 = __half22float2(*reinterpret_cast<const __half2*>(sPS + k * 64 + 2 * lane));
          p0 = fmaf(s, w2.x, p0), p1 = fmaf(s, w2.y, p1);
        }
        svec[134 + 2 * lane] = p0, svec[134 + 2 * lane + 1] = p1;
        __syncwarp();
        // ---- round 2 operand: my feature row (fp16, k = channel, 59 used)
        float a64[64];
#pragma unroll
        for (int c = 0; c < 60; ++c) a64[c] = rf[c];
        a64[60] = a64[61] = a64[62] = a64[63] = 0.f;
        write_row<64>(abuf, row, a64);
      }
      mma_round<64, 4>(a_addr, smem_u32(sm + W_B0), rows, tid);
      // ---- base_fc: x1 = ELU(per-sample part + Wf f) -> round 3 operand
      {
        float a64[64];
        float d[32];
        acc_row<32>(myrow + 0, d);
#pragma unroll
        for (int c = 0; c < 32; ++c) a64[c] = elu_(d[c] + svec[134 + c]);
        acc_row<32>(myrow + 32, d);
#pragma unroll
        for (int c = 0; c < 32; ++c) a64[32 + c] = elu_(d[c] + svec[166 + c]);
        if (run) write_row<64>(abuf, row, a64);
      }
      mma_round<32, 4>(a_addr, smem_u32(sm + W_B1), rows, tid);
      float x[32];
      {
        float d[32];
        acc_row<32>(myrow + 0, d);
        float a32[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) x[c] = elu_(d[c] + sF[F_B1B + c]), a32[c] = x[c] * wv;   // vis_fc input: x * pooling weight
        if (run) write_row<32>(abuf, row, a32);
      }
      mma_round<32, 2>(a_addr, smem_u32(sm + W_V0), rows, tid);
      {
        float d[32];
        acc_row<32>(myrow + 0, d);
#pragma unroll
        for (int c = 0; c < 32; ++c) d[c] = elu_(d[c] + sF[F_V0B + c]);
        if (run) write_row<32>(abuf, row, d);
      }
      mma_round<48, 2>(a_addr, smem_u32(sm + W_V1), rows, tid);
      float vis;
      {
        float d[32];
        acc_row<32>(myrow + 0, d);
        float e16[16];
        acc_row<16>(myrow + 32, e16);
        vis = vmask ? sigm_(elu_(e16[0] + sF[F_V1B + 32])) : 0.f;
        float a32[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) x[c] += elu_(d[c] + sF[F_V1B + c]), a32[c] = x[c] * vis;       // vis_fc2 input: x * visibility
        if (run) write_row<32>(abuf, row, a32);
      }
      mma_round<32, 2>(a_addr, smem_u32(sm + W_U0), rows, tid);
      {
        float d[32];
        acc_row<32>(myrow + 0, d);
        float u = sF[F_U1B];
#pragma unroll
        for (int c = 0; c < 32; ++c) u = fmaf(elu_(d[c] + sF[F_U0B + c]), sF[F_U1W + c], u);
        const float vis2 = vmask ? sigm_(u) : 0.f;
        float a48[48];
#pragma unroll
        for (int c = 0; c < 32; ++c) a48[c] = x[c];
        a48[32] = vis2, a48[33] = rd[0], a48[34] = rd[1], a48[35] = rd[2], a48[36] = rd[3];
#pragma unroll
        for (int c = 37; c < 48; ++c) a48[c] = 0.f;
        if (run) write_row<48>(abuf, row, a48);
      }
      mma_round<16, 3>(a_addr, smem_u32(sm + W_R0), rows, tid);
      {
        float q1[16];
        acc_row<16>(myrow + 0, q1);
#pragma unroll
        for (int c = 0; c < 16; ++c) q1[c] = elu_(q1[c] + sF[F_R0B + c]);
        float logit = sF[F_R2B];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float a = sF[F_R1B + j];
#pragma unroll
          for (int k = 0; k < 16; ++k) a = fmaf(q1[k], sF[F_R1W + 8 * k + j], a);
          logit = fmaf(elu_(a), sF[F_R2W + j], logit);
        }
        // ---- soft-max over the valid views (lanes), blend of the ORIGINAL colours
        const float lg = vmask ? logit : -3.4e38f;
        const float lmax = warp_max(lg);
        const float e = vmask ? __expf(lg - lmax) : 0.f;
        const float den = warp_sum(e);
        const float r = warp_sum(e * rgb_in[0]), g = warp_sum(e * rgb_in[1]), b = warp_sum(e * rgb_in[2]);
        if (run && lane == 0) rgb_out[3 * gi] = r / den, rgb_out[3 * gi + 1] = g / den, rgb_out[3 * gi + 2] = b / den;
      }
    }
  }
}

}  // namespace

int launch_render_blend_t5(const o2345_points* src, int64_t n, const uint8_t* active, const float* vol_cl, const float* occ, int D,
                           const o2345_views* views, int dir_mode, const float* query_center, const float* dirs,
                           const float* rnet_pack, float* rgb, int32_t* nvalid, cudaStream_t st) {
  if (views->V > 32) {
    set_error("o2345_render_blend (wgmma): at most 32 source views (a lane is a view)");
    return O2345_EUNSUPPORTED;
  }
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(render_blend_t5_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T5_SMEM));
  }
  const int64_t groups = (n + 3) / 4;
  const int64_t cap = 2 * (int64_t)sm_count();
  const int grid = (int)(groups < cap ? groups : cap);
  if (grid <= 0) return O2345_OK;
  render_blend_t5_kernel<<<grid, T5_THREADS, T5_SMEM, st>>>(*src, n, active, vol_cl, occ, D, *views, dir_mode, query_center, dirs,
                                                            rnet_pack, rgb, nvalid);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

}  // namespace o2345
