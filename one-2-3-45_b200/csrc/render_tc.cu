// View-blending network on tensor cores (SURVEY.md rows B11/B12, the ray-march hot kernel of section 8(d)).
//
// Same function as render_blend_kernel in render.cu (reference reconstruction/models/rendering_network.py:75-129 fused
// with the Projector's per-view fetch, projector.py:96-228), but the per-(sample, view) MLPs run as warp-level
// mma.sync.m16n8k16 products (fp16 operands, fp32 accumulate) instead of fp32 FMA mat-vecs:
//
//   * one warp owns one sample point; its VALID source views (masked views carry softmax weight exactly 0 in the
//     reference, skipping them is exact) are compacted into the 16 rows of an MMA tile (two tiles above 16 views);
//   * every thread fetches the bilinear taps of its two rows directly in accumulator-fragment layout
//     (float2 at channels 2t + 8h + 16kb: eight lanes read one 32-byte sector of a [V,H,W,60] channel-last map), so the
//     59-wide feature never passes through shared memory; the direction feature ray_dir_fc(ray_diff) is two MMAs whose
//     output lands in the same registers;
//   * layers chain in registers: the fp32 accumulator fragment of layer i, after ELU, is re-packed as the fp16 A
//     fragment of layer i+1 (the FlashAttention-2 re-use); weights sit in shared memory as fp16 [out][in] rows padded
//     so that the 32-bit B-fragment loads are conflict free;
//   * the per-sample reductions (weighted mean / variance over views, softmax over views) are shuffles across the
//     eight row groups of the warp; the per-sample part of base_fc[0] ([geo | mean | var] -> 64) is an MMA with
//     replicated rows whose result is the accumulator initialiser of the per-view part.
//
// Numerics: features, statistics, softmax and the colour blend are fp32; only MMA operands are rounded to fp16
// (|rel| 5e-4), which moves the blended colours by ~1e-3.  The fp32 kernel stays available (precision = 0) and is the
// one the tight oracle parity tests use.
#include <cuda_fp16.h>

#include "blend_common.cuh"
#include "common.cuh"
#include "mma_sync.cuh"

namespace o2345 {
namespace {
using namespace rpack;

// warps per CTA: ONE CTA of 20 warps per SM, so that all the warps of the SM start every sample together (see the sample loop)
// and the 48 KB of fp16 weights are staged once per SM
constexpr int TW = 20;

// fp16 weights in shared memory: matrix [n][LD], LD = K + 8 halves (conflict-free 32-bit loads by (g, t))
constexpr int LD16 = 24, LD32 = 40, LD48 = 56, LD64 = 72, LD144 = 152;
constexpr int H_D0 = 0;                     // ray_dir_fc[0]  [16][16]  (k 0..3 used)
constexpr int H_D1 = H_D0 + 16 * LD16;      // ray_dir_fc[2]  [64][16]
constexpr int H_BS = H_D1 + 64 * LD16;      // base_fc[0], per-sample part [64][144]: k = geo 0..15 | mean 16..79 | var 80..143
constexpr int H_BV = H_BS + 64 * LD144;     // base_fc[0], per-view part   [64][64]
constexpr int H_B1 = H_BV + 64 * LD64;      // base_fc[2]     [32][64]
constexpr int H_V0 = H_B1 + 32 * LD64;      // vis_fc[0]      [32][32]
constexpr int H_V1 = H_V0 + 32 * LD32;      // vis_fc[2]      [40][32]: 32 residual rows, row 32 = visibility, 7 zero rows
constexpr int H_U0 = H_V1 + 40 * LD32;      // vis_fc2[0]     [32][32]
constexpr int H_U1 = H_U0 + 32 * LD32;      // vis_fc2[2]     [8][32]: row 0 used
constexpr int H_R0 = H_U1 + 8 * LD32;       // rgb_fc[0]      [16][48]: k = x 0..31 | vis 32 | ray_diff 33..36
constexpr int H_R1 = H_R0 + 16 * LD48;      // rgb_fc[2]      [8][16]
constexpr int H_TOTAL = H_R1 + 8 * LD16;
// fp32 biases / small vectors
constexpr int F_D0B = 0, F_D1B = 16, F_B0B = 80, F_B1B = 144, F_V0B = 176, F_V1B = 208, F_U0B = 248, F_U1B = 280, F_R0B = 288,
              F_R1B = 304, F_R2W = 312, F_R2B = 320, F_S = 321, F_TOTAL = 324;
constexpr int REC = 12;                     // floats per view record
constexpr int WARP_SMEM = 32 * REC * 4 + 2 * 16 * 32 * 4;
constexpr int TC_SMEM = H_TOTAL * 2 + F_TOTAL * 4 + TW * WARP_SMEM;
static_assert((H_TOTAL * 2) % 16 == 0, "bias block must stay 16-byte aligned");

// Branch-free ELU: one MUFU.EX2 on min(x, 0) and a select (the ternary around __expf compiled to a divergent branch per
// element: r1 ncu of this kernel showed BSSY/BSYNC/FSETP/PLOP3 at 20 % of the issued instructions).
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
// ELU on a packed pair that only feeds the next layer's fp16 operand: max(x, 0) + (2^(min(x, 0) log2 e) - 1) in half2
__device__ __forceinline__ uint32_t elu_h2(uint32_t v) {
  const __half2 x = *reinterpret_cast<const __half2*>(&v);
  const __half2 zero = __float2half2_rn(0.f);
  const __half2 e = h2exp2(__hmul2(__hmin2(x, zero), __float2half2_rn(1.4426950408889634f)));
  const __half2 r = __hadd2(__hmax2(x, zero), __hsub2(e, __float2half2_rn(1.f)));
  return *reinterpret_cast<const uint32_t*>(&r);
}
// c[16 x 8 NT] += a[16 x 16 KB] . W^T, W stored [n][LD] halves
template <int KB, int NT>
__device__ __forceinline__ void mm(float (&c)[NT][4], const uint32_t (&a)[KB][4], const __half* W, int LD, int g, int t) {
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const __half* p = W + (8 * j + g) * LD + 16 * kb + 2 * t;
      mma16816(c[j], a[kb], *reinterpret_cast<const uint32_t*>(p), *reinterpret_cast<const uint32_t*>(p + 8));
    }
}
template <int NT>
__device__ __forceinline__ void init_bias(float (&c)[NT][4], const float* b, int t) {
#pragma unroll
  for (int j = 0; j < NT; ++j) c[j][0] = c[j][2] = b[8 * j + 2 * t], c[j][1] = c[j][3] = b[8 * j + 2 * t + 1];
}
// accumulator fragments (2 n-tiles per k-block) -> A fragments of the next layer
template <int KB>
__device__ __forceinline__ void to_frags(uint32_t (&a)[KB][4], const float (&c)[2 * KB][4]) {
#pragma unroll
  for (int kb = 0; kb < KB; ++kb) {
    a[kb][0] = pack2(c[2 * kb][0], c[2 * kb][1]), a[kb][1] = pack2(c[2 * kb][2], c[2 * kb][3]);
    a[kb][2] = pack2(c[2 * kb + 1][0], c[2 * kb + 1][1]), a[kb][3] = pack2(c[2 * kb + 1][2], c[2 * kb + 1][3]);
  }
}
// ... with the ELU applied to the packed halves (layers whose output is only the next MMA operand)
template <int KB>
__device__ __forceinline__ void to_frags_elu(uint32_t (&a)[KB][4], const float (&c)[2 * KB][4]) {
  to_frags<KB>(a, c);
#pragma unroll
  for (int kb = 0; kb < KB; ++kb)
#pragma unroll
    for (int i = 0; i < 4; ++i) a[kb][i] = elu_h2(a[kb][i]);
}
template <int NT>
__device__ __forceinline__ void elu_all(float (&c)[NT][4]) {
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) c[j][i] = elu_(c[j][i]);
}

// sum over the eight row groups (lanes with equal t)
__device__ __forceinline__ float rows_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}
__device__ __forceinline__ float rows_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
  return v;
}

// Feature-channel order inside the MMA fragments.  A thread's four accumulator columns of one 16-column block are
// {2t, 2t+1, 8+2t, 9+2t}; mapping fragment column p to map channel chan(p) = 16 (p / 16) + 4 t + 2 h + e makes them the
// four CONSECUTIVE channels 16 kb + 4 t .. + 3, i.e. one 16-byte load per tap.  Every matrix whose k (or n) index is a
// feature channel is stored with that permutation, so the arithmetic is unchanged.
__host__ __device__ constexpr int chan(int p) { return 16 * (p / 16) + 4 * ((p % 8) / 2) + 2 * ((p % 16) / 8) + (p % 2); }

// dst[n][col0 + k] = src[kmap(k) * src_ld + nmap(n)] for nmap(n) < n_used, kmap(k) < k_used; zero elsewhere in
// [n_rows][k_span].  perm_k / perm_n: the index is a feature channel, stored in fragment order (chan()).
__device__ void fill_w(__half* dst, int LD, int n_rows, int col0, int k_span, const float* __restrict__ src, int src_ld, int n_used,
                       int k_used, int tid, int nthreads, bool perm_k = false, bool perm_n = false) {
  for (int i = tid; i < n_rows * k_span; i += nthreads) {
    int nrow = i / k_span, k = i - nrow * k_span;
    const int ns = perm_n ? chan(nrow) : nrow, ks = perm_k ? chan(k) : k;
    float v = (ns < n_used && ks < k_used) ? __ldg(src + (int64_t)ks * src_ld + ns) : 0.f;
    dst[nrow * LD + col0 + k] = __float2half_rn(v);
  }
}

__global__ void __launch_bounds__(TW * 32, 1)
render_blend_tc_kernel(o2345_points src, int64_t n, const uint8_t* __restrict__ active, const float* __restrict__ vol,
                       const float* __restrict__ occ, int D, o2345_views views, int dir_mode,
                       const float* __restrict__ query_center, const float* __restrict__ dirs,
                       const float* __restrict__ pack, float* __restrict__ rgb_out, int32_t* __restrict__ nvalid_out) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sW = reinterpret_cast<__half*>(smem_raw);
  float* sB = reinterpret_cast<float*>(sW + H_TOTAL);
  const int tid = threadIdx.x, nth = blockDim.x;
  // ---- weights: fp32 [in][out] pack -> fp16 [out][in] rows
  fill_w(sW + H_D0, LD16, 16, 0, 16, pack + P_D0W, 16, 16, 4, tid, nth);
  fill_w(sW + H_D1, LD16, 64, 0, 16, pack + P_D1W, 64, 64, 16, tid, nth, false, true);
  fill_w(sW + H_BS, LD144, 64, 0, 16, pack + P_B0W, 64, 64, 16, tid, nth);
  fill_w(sW + H_BS, LD144, 64, 16, 64, pack + P_B0W + 16 * 64, 64, 64, NF, tid, nth, true);
  fill_w(sW + H_BS, LD144, 64, 80, 64, pack + P_B0W + 75 * 64, 64, 64, NF, tid, nth, true);
  fill_w(sW + H_BV, LD64, 64, 0, 64, pack + P_B0W + 134 * 64, 64, 64, NF, tid, nth, true);
  fill_w(sW + H_B1, LD64, 32, 0, 64, pack + P_B1W, 32, 32, 64, tid, nth);
  fill_w(sW + H_V0, LD32, 32, 0, 32, pack + P_V0W, 32, 32, 32, tid, nth);
  fill_w(sW + H_V1, LD32, 40, 0, 32, pack + P_V1W, 32, 32, 32, tid, nth);
  fill_w(sW + H_U0, LD32, 32, 0, 32, pack + P_U0W, 32, 32, 32, tid, nth);
  fill_w(sW + H_U1, LD32, 8, 0, 32, pack + P_U1W, 1, 1, 32, tid, nth);
  fill_w(sW + H_R0, LD48, 16, 0, 48, pack + P_R0W, 16, 16, 37, tid, nth);
  fill_w(sW + H_R1, LD16, 8, 0, 16, pack + P_R1W, 8, 8, 16, tid, nth);
  __syncthreads();
  for (int k = tid; k < 32; k += nth) sW[H_V1 + 32 * LD32 + k] = __float2half_rn(__ldg(pack + P_V1V + k));  // visibility row
  for (int i = tid; i < F_TOTAL; i += nth) {
    float v = 0.f;
    if (i < F_D1B) v = pack[P_D0B + i];
    else if (i < F_B0B) v = pack[P_D1B + chan(i - F_D1B)];   // output = feature channel: fragment order
    else if (i < F_B1B) v = pack[P_B0B + i - F_B0B];
    else if (i < F_V0B) v = pack[P_B1B + i - F_B1B];
    else if (i < F_V1B) v = pack[P_V0B + i - F_V0B];
    else if (i < F_U0B) v = i - F_V1B < 32 ? pack[P_V1B + i - F_V1B] : (i - F_V1B == 32 ? pack[P_V1VB] : 0.f);
    else if (i < F_U1B) v = pack[P_U0B + i - F_U0B];
    else if (i < F_R0B) v = i == F_U1B ? pack[P_U1B] : 0.f;
    else if (i < F_R1B) v = pack[P_R0B + i - F_R0B];
    else if (i < F_R2W) v = pack[P_R1B + i - F_R1B];
    else if (i < F_R2B) v = pack[P_R2W + i - F_R2W];
    else if (i == F_R2B) v = pack[P_R2B];
    else if (i == F_S) v = pack[P_S];
    sB[i] = v;
  }
  __syncthreads();

  const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  uint8_t* wbase = reinterpret_cast<uint8_t*>(sB + F_TOTAL) + warp * WARP_SMEM;
  float* sRec = reinterpret_cast<float*>(wbase);                       // [32 slots][REC]
  uint32_t* sF = reinterpret_cast<uint32_t*>(wbase + 32 * REC * 4);    // [2 tiles][16 regs][32 lanes]
  const int V = views.V, H = views.H, W = views.W;
  const float abs_s = sB[F_S];

  // The per-sample path is ~4 600 straight-line warp instructions (73 KB of SASS): ten warps at ten different places of it
  // starve on instruction fetch (ncu: no_instruction = 4.5 stall cycles per issue).  So all the warps of the CTA start
  // every sample together (one barrier per ~4 600 instructions): they walk the code within a few cache lines of each other
  // and share the fetches.  Per 8 192 rays, two CTAs of ten warps took 10.47 ms without the barrier and 8.74 ms with it; ONE
  // CTA of twenty warps per SM takes 8.53 ms.  (Two more meeting points inside the sample -- before pass A and before pass B,
  // early-leaving warps arriving without waiting -- gave nothing: 8.71 ms.)
  for (int64_t g0 = (int64_t)blockIdx.x * TW; g0 < n; g0 += (int64_t)gridDim.x * TW) {
    __syncthreads();
    const int64_t gi = g0 + warp;
    if (gi >= n) continue;
    if (skip_inactive(active, gi, lane, rgb_out, nvalid_out)) continue;
    const BlendSample s = blend_front_end(src, gi, vol, occ, D, views, dir_mode, query_center, dirs, abs_s, lane);
    if (lane == 0 && nvalid_out) nvalid_out[gi] = s.nvalid;

    if (s.nvalid == 0) {
      // every logit is -1e9: softmax is uniform over ALL views (reference rendering_network.py:119-121)
      float acc = 0.f;
      for (int v = 0; v < V; ++v) {
        float vgx = __shfl_sync(0xffffffffu, s.gx, v), vgy = __shfl_sync(0xffffffffu, s.gy, v);
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
      continue;
    }

    // ---- per-view records, compacted by slot (= rank of the view among the valid ones)
    __syncwarp();
    if (s.vmask) {
      const int slot = __popc(s.valid & ((1u << lane) - 1u));
      float fx = ((s.gx + 1.f) / 2.f) * (float)(W - 1), fy = ((s.gy + 1.f) / 2.f) * (float)(H - 1);
      float x0 = floorf(fx), y0 = floorf(fy);
      int ix = (int)x0, iy = (int)y0;
      float x1 = x0 + 1.f, y1 = y0 + 1.f;
      bool inx0 = ix >= 0, inx1 = ix + 1 <= W - 1, iny0 = iy >= 0, iny1 = iy + 1 <= H - 1;
      float* r = sRec + slot * REC;
      r[0] = (iny0 && inx0) ? (x1 - fx) * (y1 - fy) : 0.f;
      r[1] = (iny0 && inx1) ? (fx - x0) * (y1 - fy) : 0.f;
      r[2] = (iny1 && inx0) ? (x1 - fx) * (fy - y0) : 0.f;
      r[3] = (iny1 && inx1) ? (fx - x0) * (fy - y0) : 0.f;
      r[4] = __int_as_float(ix), r[5] = __int_as_float(iy), r[6] = __int_as_float(lane);
      r[7] = s.rd0, r[8] = s.rd1, r[9] = s.rd2, r[10] = s.rd3, r[11] = s.wv;
    }
    __syncwarp();

    const int ntile = (s.nvalid + 15) >> 4;
    float S[8][2], Q[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) S[j][0] = S[j][1] = Q[j][0] = Q[j][1] = 0.f;
    float rgA[6], rgB[6];   // original r, g, b of rows g and g + 8 in tile 0 / 1 (meaningful in the t == 0 lanes)

    // ================= pass A: features of every valid view, weighted first and second moments
    for (int tile = 0; tile < ntile; ++tile) {
      float F[8][4];
      float rdr[2][4], wr[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int slot = 16 * tile + g + 8 * rr;
        const bool ok = slot < s.nvalid;
        const float* r = sRec + (ok ? slot : 0) * REC;
        const float4 w4 = *reinterpret_cast<const float4*>(r);
        const float wq[4] = {ok ? w4.x : 0.f, ok ? w4.y : 0.f, ok ? w4.z : 0.f, ok ? w4.w : 0.f};
        const int ix = __float_as_int(r[4]), iy = __float_as_int(r[5]), view = __float_as_int(r[6]);
        rdr[rr][0] = ok ? r[7] : 0.f, rdr[rr][1] = ok ? r[8] : 0.f, rdr[rr][2] = ok ? r[9] : 0.f, rdr[rr][3] = ok ? r[10] : 0.f;
        wr[rr] = ok ? r[11] : 0.f;
        const float* m = views.maps + (int64_t)view * H * W * CM;
        const int cx0 = min(max(ix, 0), W - 1), cx1 = min(max(ix + 1, 0), W - 1);
        const int cy0 = min(max(iy, 0), H - 1), cy1 = min(max(iy + 1, 0), H - 1);
        const float* tp[4] = {m + ((int64_t)cy0 * W + cx0) * CM, m + ((int64_t)cy0 * W + cx1) * CM,
                              m + ((int64_t)cy1 * W + cx0) * CM, m + ((int64_t)cy1 * W + cx1) * CM};
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
          const int c = 16 * kb + 4 * t;   // channels c .. c + 3 of this row = fragment columns {2t, 2t+1} of tiles 2kb, 2kb+1
          float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
          if (c < CM) {
#pragma unroll
            for (int tap = 0; tap < 4; ++tap) {
              const float4 v = __ldg(reinterpret_cast<const float4*>(tp[tap] + c));
              a0 = fmaf(v.x, wq[tap], a0), a1 = fmaf(v.y, wq[tap], a1), a2 = fmaf(v.z, wq[tap], a2), a3 = fmaf(v.w, wq[tap], a3);
            }
          }
          F[2 * kb][2 * rr] = a0, F[2 * kb][2 * rr + 1] = a1, F[2 * kb + 1][2 * rr] = a2, F[2 * kb + 1][2 * rr + 1] = a3;
        }
      }
      // original colours: channels 0, 1 = columns 0, 1 of tile 0, channel 2 = column 0 of tile 1 (chan()), all in t == 0
      if (tile == 0) rgA[0] = F[0][0], rgA[1] = F[0][1], rgA[2] = F[1][0], rgA[3] = F[0][2], rgA[4] = F[0][3], rgA[5] = F[1][2];
      else rgB[0] = F[0][0], rgB[1] = F[0][1], rgB[2] = F[1][0], rgB[3] = F[0][2], rgB[4] = F[0][3], rgB[5] = F[1][2];
      // direction feature: ray_dir_fc(ray_diff) = ELU(D1 . ELU(D0 . rd + b0) + b1), added to the fetched feature
      {
        uint32_t ard[1][4];
        ard[0][0] = t == 0 ? pack2(rdr[0][0], rdr[0][1]) : (t == 1 ? pack2(rdr[0][2], rdr[0][3]) : 0u);
        ard[0][1] = t == 0 ? pack2(rdr[1][0], rdr[1][1]) : (t == 1 ? pack2(rdr[1][2], rdr[1][3]) : 0u);
        ard[0][2] = 0u, ard[0][3] = 0u;
        float c16[2][4];
        init_bias<2>(c16, sB + F_D0B, t);
        mm<1, 2>(c16, ard, sW + H_D0, LD16, g, t);
        uint32_t a16[1][4];
        to_frags_elu<1>(a16, c16);
        float c64[8][4];
        init_bias<8>(c64, sB + F_D1B, t);
        mm<1, 8>(c64, a16, sW + H_D1, LD16, g, t);
        const bool ok0 = 16 * tile + g < s.nvalid, ok1 = 16 * tile + g + 8 < s.nvalid;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          F[j][0] = ok0 ? F[j][0] + elu_(c64[j][0]) : 0.f, F[j][1] = ok0 ? F[j][1] + elu_(c64[j][1]) : 0.f;
          F[j][2] = ok1 ? F[j][2] + elu_(c64[j][2]) : 0.f, F[j][3] = ok1 ? F[j][3] + elu_(c64[j][3]) : 0.f;
        }
      }
      const float w0 = wr[0], w1 = wr[1];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        S[j][0] += w0 * F[j][0] + w1 * F[j][2], S[j][1] += w0 * F[j][1] + w1 * F[j][3];
        Q[j][0] += w0 * F[j][0] * F[j][0] + w1 * F[j][2] * F[j][2], Q[j][1] += w0 * F[j][1] * F[j][1] + w1 * F[j][3] * F[j][3];
      }
      uint32_t aF[4][4];
      to_frags<4>(aF, F);
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)
#pragma unroll
        for (int i = 0; i < 4; ++i) sF[(tile * 16 + kb * 4 + i) * 32 + lane] = aF[kb][i];
    }
    // ---- weighted mean / variance over the views: sum over the eight row groups
    //      sum_v w (f - mean)^2 = sum_v w f^2 - mean^2 (2 - sum_v w)
    const float wsum1 = s.wtot / (s.wtot + 1e-8f);
    uint32_t aS[9][4];   // per-sample input [geo | mean | var] with all 16 rows equal
    {
      float g0 = __shfl_sync(0xffffffffu, s.geo, 2 * t), g1 = __shfl_sync(0xffffffffu, s.geo, 2 * t + 1);
      float g8 = __shfl_sync(0xffffffffu, s.geo, 2 * t + 8), g9 = __shfl_sync(0xffffffffu, s.geo, 2 * t + 9);
      aS[0][0] = aS[0][1] = pack2(g0, g1), aS[0][2] = aS[0][3] = pack2(g8, g9);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float m0 = rows_sum(S[j][0]), m1 = rows_sum(S[j][1]);
      float q0 = rows_sum(Q[j][0]), q1 = rows_sum(Q[j][1]);
      float v0 = fmaxf(q0 - m0 * m0 * (2.f - wsum1), 0.f), v1 = fmaxf(q1 - m1 * m1 * (2.f - wsum1), 0.f);
      const int kb = j >> 1, hi = (j & 1) * 2;
      aS[1 + kb][hi] = aS[1 + kb][hi + 1] = pack2(m0, m1);
      aS[5 + kb][hi] = aS[5 + kb][hi + 1] = pack2(v0, v1);
    }
    float hs[8][4];
    init_bias<8>(hs, sB + F_B0B, t);
    mm<9, 8>(hs, aS, sW + H_BS, LD144, g, t);

    // ================= pass B: per-view MLPs, logits
    float lgA0 = -3.4e38f, lgA1 = -3.4e38f, lgB0 = -3.4e38f, lgB1 = -3.4e38f;   // logits of rows g, g + 8 in tile 0 / 1
    for (int tile = 0; tile < ntile; ++tile) {
      const bool ok0 = 16 * tile + g < s.nvalid, ok1 = 16 * tile + g + 8 < s.nvalid;
      const float w0 = ok0 ? sRec[(16 * tile + g) * REC + 11] : 0.f, w1 = ok1 ? sRec[(16 * tile + g + 8) * REC + 11] : 0.f;
      uint32_t aF[4][4];
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)
#pragma unroll
        for (int i = 0; i < 4; ++i) aF[kb][i] = sF[(tile * 16 + kb * 4 + i) * 32 + lane];
      // base_fc: x1 = ELU(hs + Wf f), x2 = ELU(W x1 + b)
      float c1[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) c1[j][i] = hs[j][i];
      mm<4, 8>(c1, aF, sW + H_BV, LD64, g, t);
      uint32_t a1[4][4];
      to_frags_elu<4>(a1, c1);
      float x2[4][4];
      init_bias<4>(x2, sB + F_B1B, t);
      mm<4, 4>(x2, a1, sW + H_B1, LD64, g, t);
      elu_all<4>(x2);
      // vis_fc(x * weight): 32 -> 32 -> (32 residual + visibility)
      float xw[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) xw[j][0] = x2[j][0] * w0, xw[j][1] = x2[j][1] * w0, xw[j][2] = x2[j][2] * w1, xw[j][3] = x2[j][3] * w1;
      uint32_t a2[2][4];
      to_frags<2>(a2, xw);
      float hv[4][4];
      init_bias<4>(hv, sB + F_V0B, t);
      mm<2, 4>(hv, a2, sW + H_V0, LD32, g, t);
      to_frags_elu<2>(a2, hv);
      float rv[5][4];
      init_bias<5>(rv, sB + F_V1B, t);
      mm<2, 5>(rv, a2, sW + H_V1, LD32, g, t);
      // visibility = column 32 = tile 4, column 0: held by the t == 0 lane of each row group
      const float vr0 = __shfl_sync(0xffffffffu, rv[4][0], lane & ~3), vr1 = __shfl_sync(0xffffffffu, rv[4][2], lane & ~3);
      const float vis0 = sigm_(elu_(vr0)), vis1 = sigm_(elu_(vr1));   // mask is 1 for the views processed here
      float x3[4][4], xv[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int i = 0; i < 4; ++i) x3[j][i] = x2[j][i] + elu_(rv[j][i]);
        xv[j][0] = x3[j][0] * vis0, xv[j][1] = x3[j][1] * vis0, xv[j][2] = x3[j][2] * vis1, xv[j][3] = x3[j][3] * vis1;
      }
      // vis_fc2(x * vis): 32 -> 32 -> 1, sigmoid
      to_frags<2>(a2, xv);
      float h2[4][4];
      init_bias<4>(h2, sB + F_U0B, t);
      mm<2, 4>(h2, a2, sW + H_U0, LD32, g, t);
      to_frags_elu<2>(a2, h2);
      float u[1][4];
      init_bias<1>(u, sB + F_U1B, t);
      mm<2, 1>(u, a2, sW + H_U1, LD32, g, t);
      const float vis2_0 = sigm_(__shfl_sync(0xffffffffu, u[0][0], lane & ~3)), vis2_1 = sigm_(__shfl_sync(0xffffffffu, u[0][2], lane & ~3));
      // rgb_fc([x, vis, ray_diff]): 37 -> 16 -> 8 -> 1
      uint32_t a3[3][4];
      {
        uint32_t ax[2][4];
        to_frags<2>(ax, x3);
#pragma unroll
        for (int i = 0; i < 4; ++i) a3[0][i] = ax[0][i], a3[1][i] = ax[1][i];
        const float* r0p = sRec + (ok0 ? 16 * tile + g : 0) * REC;
        const float* r1p = sRec + (ok1 ? 16 * tile + g + 8 : 0) * REC;
        a3[2][0] = t == 0 ? pack2(vis2_0, r0p[7]) : (t == 1 ? pack2(r0p[8], r0p[9]) : (t == 2 ? pack2(r0p[10], 0.f) : 0u));
        a3[2][1] = t == 0 ? pack2(vis2_1, r1p[7]) : (t == 1 ? pack2(r1p[8], r1p[9]) : (t == 2 ? pack2(r1p[10], 0.f) : 0u));
        a3[2][2] = 0u, a3[2][3] = 0u;
      }
      float q1[2][4];
      init_bias<2>(q1, sB + F_R0B, t);
      mm<3, 2>(q1, a3, sW + H_R0, LD48, g, t);
      uint32_t a4[1][4];
      to_frags_elu<1>(a4, q1);
      float q2[1][4];
      init_bias<1>(q2, sB + F_R1B, t);
      mm<1, 1>(q2, a4, sW + H_R1, LD16, g, t);
      const float r2a = sB[F_R2W + 2 * t], r2b = sB[F_R2W + 2 * t + 1];
      float l0 = elu_(q2[0][0]) * r2a + elu_(q2[0][1]) * r2b, l1 = elu_(q2[0][2]) * r2a + elu_(q2[0][3]) * r2b;
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1), l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1), l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      l0 = ok0 ? l0 + sB[F_R2B] : -3.4e38f, l1 = ok1 ? l1 + sB[F_R2B] : -3.4e38f;
      if (tile == 0) lgA0 = l0, lgA1 = l1;
      else lgB0 = l0, lgB1 = l1;
    }
    // ---- softmax over the valid views, blend the ORIGINAL colours
    const float lmax = rows_max(fmaxf(fmaxf(lgA0, lgA1), fmaxf(lgB0, lgB1)));
    const float eA0 = lgA0 > -1e38f ? __expf(lgA0 - lmax) : 0.f, eA1 = lgA1 > -1e38f ? __expf(lgA1 - lmax) : 0.f;
    const float eB0 = lgB0 > -1e38f ? __expf(lgB0 - lmax) : 0.f, eB1 = lgB1 > -1e38f ? __expf(lgB1 - lmax) : 0.f;
    float den = eA0 + eA1 + eB0 + eB1;
    float accr = eA0 * rgA[0] + eA1 * rgA[3], accg = eA0 * rgA[1] + eA1 * rgA[4], accb = eA0 * rgA[2] + eA1 * rgA[5];
    if (ntile > 1) accr += eB0 * rgB[0] + eB1 * rgB[3], accg += eB0 * rgB[1] + eB1 * rgB[4], accb += eB0 * rgB[2] + eB1 * rgB[5];
    den = rows_sum(den), accr = rows_sum(accr), accg = rows_sum(accg), accb = rows_sum(accb);
    if (lane == 0) rgb_out[3 * gi] = accr / den, rgb_out[3 * gi + 1] = accg / den, rgb_out[3 * gi + 2] = accb / den;
    __syncwarp();
  }
}

}  // namespace

int launch_render_blend_tc(const o2345_points* src, int64_t n, const uint8_t* active, const float* vol_cl, const float* occ, int D,
                           const o2345_views* views, int dir_mode, const float* query_center, const float* dirs,
                           const float* rnet_pack, float* rgb, int32_t* nvalid, cudaStream_t st) {
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(render_blend_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
  }
  const int64_t need = (n + TW - 1) / TW;
  const int grid = (int)(need < (int64_t)sm_count() ? need : (int64_t)sm_count());
  render_blend_tc_kernel<<<grid, TW * 32, TC_SMEM, st>>>(*src, n, active, vol_cl, occ, D, *views, dir_mode, query_center, dirs,
                                                         rnet_pack, rgb, nvalid);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

}  // namespace o2345
