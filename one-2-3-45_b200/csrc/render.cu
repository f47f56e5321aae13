// Volume-rendering kernels: hierarchical sampling (B13), multi-view projector + view-blending
// network (B11/B12) and NeuS alpha compositing (B14).  SURVEY.md section 8.
//
//   ray_upsample_kernel   one thread per ray: section weights from the current (z, sdf) samples,
//                         deterministic inverse-CDF draw of n_new depths (up_sample + sample_pdf);
//   ray_merge_kernel      one thread per ray: merge of two sorted depth lists (cat_z_vals);
//   ray_mid_kernel        mid-point depths, section lengths and the nearest-occupancy flag;
//   render_blend_kernel   one WARP per sample point.  Lanes first act as views (projection,
//                         visibility, direction features, pooling weights), then as channels
//                         (59-wide feature fetch from a channel-last [V,H,W,60] map = one coalesced
//                         240-byte read per tap) and as MLP outputs.  Only views that pass the
//                         mask are run through the per-view MLPs: masked views carry softmax
//                         weight exactly 0 in the reference, so skipping them is exact and removes
//                         ~3/4 of the arithmetic and gathers at the demo camera layout.  The
//                         193-wide first layer is split into a per-sample part (geometry, mean,
//                         variance) and a 59-wide per-view part.
//   ray_composite_kernel  one thread per ray: NeuS alpha, transmittance, colour / depth.
#include "blend_common.cuh"
#include "common.cuh"

namespace o2345 {
namespace {
using namespace rpack;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
// Blend-network activations: ex2.approx based (absolute error <= 3e-7 on values of O(1), far below the
// stated colour tolerance); expm1f/expf cost ~40 / ~15 instructions each and dominated the kernel.
__device__ __forceinline__ float eluf_(float x) { return x > 0.f ? x : __expf(x) - 1.f; }
__device__ __forceinline__ float fsigmoid_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

__device__ __forceinline__ int occ_lookup(const float* __restrict__ occ, int D, float px, float py, float pz) {
  float p[3] = {px, py, pz};
  int idx[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float f = nearbyintf(((p[a] + 1.f) * (float)D - 1.f) / 2.f);
    ok = ok && (f >= 0.f) && (f <= (float)(D - 1));
    idx[a] = (int)fminf(fmaxf(f, 0.f), (float)(D - 1));
  }
  return (ok && occ[((int64_t)idx[0] * D + idx[1]) * D + idx[2]] > 0.f) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------
// B13: up_sample + sample_pdf(det=True)   (reference sparse_neus_renderer.py:73-115,
//                                          render_utils.py:8-51)
// ---------------------------------------------------------------------------------------
constexpr int UPT = 64;  // threads (= rays) per CTA

__global__ void __launch_bounds__(UPT)
ray_upsample_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, int64_t R,
                    const float* __restrict__ z, const float* __restrict__ sdf, int S, float inv_s,
                    const float* __restrict__ occ, int D, const float* __restrict__ u, int n_new,
                    float* __restrict__ new_z) {
  extern __shared__ float sm[];  // cdf [S][UPT]
  float* cdf = sm;
  int64_t r = (int64_t)blockIdx.x * UPT + threadIdx.x;
  if (r >= R) return;
  const int t = threadIdx.x;
  const float ox = rays_o[3 * r], oy = rays_o[3 * r + 1], oz = rays_o[3 * r + 2];
  const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
  const float* zr = z + r * S;
  const float* sr = sdf + r * S;
  float z0 = zr[0], s0 = sr[0];
  int m0 = occ_lookup(occ, D, __fadd_rn(ox, __fmul_rn(dx, z0)), __fadd_rn(oy, __fmul_rn(dy, z0)), __fadd_rn(oz, __fmul_rn(dz, z0)));
  float prev_dot = 0.f, T = 1.f, wsum = 0.f;
  // pass 1: section weights (stored un-normalised in cdf[1..S-1]) and their sum
  for (int s = 0; s < S - 1; ++s) {
    float z1 = zr[s + 1], s1 = sr[s + 1];
    int m1 = occ_lookup(occ, D, __fadd_rn(ox, __fmul_rn(dx, z1)), __fadd_rn(oy, __fmul_rn(dy, z1)), __fadd_rn(oz, __fmul_rn(dz, z1)));
    float mask = (float)(m0 * m1);
    float mid = (s0 + s1) * 0.5f;
    float dist = z1 - z0;
    float dot = (s1 - s0) / (dist + 1e-5f);
    float d = fminf(fmaxf(fminf(prev_dot, dot), -10.f), 0.f) * mask;
    prev_dot = dot;
    float pc = sigmoidf_((mid - d * dist * 0.5f) * inv_s);
    float nc = sigmoidf_((mid + d * dist * 0.5f) * inv_s);
    float alpha = mask * ((pc - nc + 1e-5f) / (pc + 1e-5f));
    float w = alpha * T + 1e-5f;
    T *= (1.f - alpha + 1e-7f);
    cdf[(s + 1) * UPT + t] = w;
    wsum += w;
    z0 = z1, s0 = s1, m0 = m1;
  }
  // pass 2: cdf = cumsum(w / sum), cdf[0] = 0
  cdf[t] = 0.f;
  float run = 0.f;
  for (int s = 1; s < S; ++s) {
    run += cdf[s * UPT + t] / wsum;
    cdf[s * UPT + t] = run;
  }
  // pass 3: inverse CDF at u_j (u increasing -> resume the search where the last one stopped)
  int ind = 0;  // number of cdf entries <= u  (searchsorted right=True)
  for (int j = 0; j < n_new; ++j) {
    float uj = u[j];
    while (ind < S && cdf[ind * UPT + t] <= uj) ++ind;
    int below = max(ind - 1, 0), above = min(ind, S - 1);
    float c0 = cdf[below * UPT + t], c1 = cdf[above * UPT + t];
    float b0 = zr[below], b1 = zr[above];
    float den = c1 - c0;
    if (den < 1e-5f) den = 1.f;
    float tt = (uj - c0) / den;
    new_z[r * n_new + j] = b0 + tt * (b1 - b0);
  }
}

// merge two ascending lists (old first on ties) -- cat_z_vals' torch.sort (reference :143-149)
__global__ void ray_merge_kernel(const float* __restrict__ z, const float* __restrict__ sdf, int S,
                                 const float* __restrict__ nz, const float* __restrict__ nsdf, int n_new, int64_t R,
                                 float* __restrict__ oz, float* __restrict__ osdf) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* a = z + r * S;
  const float* as = sdf + r * S;
  const float* b = nz + r * n_new;
  const float* bs = nsdf + r * n_new;
  float* o = oz + r * (S + n_new);
  float* os = osdf + r * (S + n_new);
  int i = 0, j = 0;
  for (int k = 0; k < S + n_new; ++k) {
    bool take_a = (j >= n_new) || (i < S && a[i] <= b[j]);
    if (take_a) { o[k] = a[i]; os[k] = as[i]; ++i; }
    else { o[k] = b[j]; os[k] = bs[j]; ++j; }
  }
}

// mid-point depths + section lengths + occupancy flag (reference sparse_neus_renderer.py:201-223) of sample i = r * S + s;
// last: the length of ray r's last section
__device__ __forceinline__ void ray_mid_sample(const float* __restrict__ rays_o, const float* __restrict__ rays_d, int64_t i,
                                               int64_t r, int s, const float* __restrict__ z, int S, float last,
                                               const float* __restrict__ occ, int D, float* __restrict__ mid_z,
                                               float* __restrict__ dists, uint8_t* __restrict__ active) {
  float zi = z[i];
  float d = (s + 1 < S) ? z[i + 1] - zi : last;
  float m = zi + d * 0.5f;
  mid_z[i] = m;
  dists[i] = d;
  float px = __fadd_rn(rays_o[3 * r], __fmul_rn(rays_d[3 * r], m));
  float py = __fadd_rn(rays_o[3 * r + 1], __fmul_rn(rays_d[3 * r + 1], m));
  float pz = __fadd_rn(rays_o[3 * r + 2], __fmul_rn(rays_d[3 * r + 2], m));
  active[i] = (uint8_t)occ_lookup(occ, D, px, py, pz);
}

__global__ void ray_mid_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, int64_t R,
                               const float* __restrict__ z, int S, float sample_dist, const float* __restrict__ occ,
                               int D, float* __restrict__ mid_z, float* __restrict__ dists, uint8_t* __restrict__ active) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * S) return;
  int64_t r = i / S;
  ray_mid_sample(rays_o, rays_d, i, r, (int)(i - r * S), z, S, sample_dist, occ, D, mid_z, dists, active);
}

// the same with each ray's own last section (rays of cameras with different near / far in one launch)
__global__ void ray_mid_per_ray_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, int64_t R,
                                       const float* __restrict__ z, int S, const float* __restrict__ sample_dist,
                                       const float* __restrict__ occ, int D, float* __restrict__ mid_z,
                                       float* __restrict__ dists, uint8_t* __restrict__ active) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * S) return;
  int64_t r = i / S;
  ray_mid_sample(rays_o, rays_d, i, r, (int)(i - r * S), z, S, sample_dist[r], occ, D, mid_z, dists, active);
}

// ---------------------------------------------------------------------------------------
// B11/B12: projector + GeneralRenderingNetwork
// ---------------------------------------------------------------------------------------
constexpr int BW = 24;             // warps per CTA
constexpr int WS_X = 512;                   // per-warp: two [64][4] activation buffers
constexpr int WS_RGB = 32 * 4;              // per-warp: rgb of each view
constexpr int WS_TOTAL = WS_X + WS_RGB;
constexpr int BLEND_SMEM = (P_TOTAL + BW * WS_TOTAL) * 4;

// y[lane] (and y[lane+32] when OUT > 32) = b + sum_i x[i] * W[i][.]; x in per-warp smem.
template <int IN, int OUT, int LD>
__device__ __forceinline__ void matvec(const float* __restrict__ W, const float* __restrict__ b,
                                       const float* __restrict__ x, int lane, float& y0, float& y1) {
  y0 = (lane < OUT) ? b[lane] : 0.f;
  y1 = (OUT > 32 && lane + 32 < OUT) ? b[lane + 32] : 0.f;
  const int l0 = lane < OUT ? lane : 0;
  const int l1 = (OUT > 32 && lane + 32 < OUT) ? lane + 32 : 0;
#pragma unroll 4
  for (int i = 0; i < IN; ++i) {
    float xi = x[i];
    y0 = fmaf(xi, W[i * LD + l0], y0);
    if (OUT > 32) y1 = fmaf(xi, W[i * LD + l1], y1);
  }
}

// Four views at once: xs[i*4 + q] is input i of view q.  y0[q] (output `lane`) and y1[q] (output
// lane+32, OUT > 32 only) start from init0 / init1; each weight is loaded once for the four views.
template <int IN, int OUT, int LD>
__device__ __forceinline__ void matvec4(const float* __restrict__ W, const float* __restrict__ xs, int lane,
                                        float init0, float init1, float (&y0)[4], float (&y1)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) y0[q] = init0, y1[q] = init1;
  const int l0 = lane < OUT ? lane : 0;
  const int l1 = (OUT > 32 && lane + 32 < OUT) ? lane + 32 : 0;
#pragma unroll 4
  for (int i = 0; i < IN; ++i) {
    float4 x = *reinterpret_cast<const float4*>(xs + 4 * i);
    float w0 = W[i * LD + l0];
    y0[0] = fmaf(x.x, w0, y0[0]), y0[1] = fmaf(x.y, w0, y0[1]), y0[2] = fmaf(x.z, w0, y0[2]), y0[3] = fmaf(x.w, w0, y0[3]);
    if (OUT > 32) {
      float w1 = W[i * LD + l1];
      y1[0] = fmaf(x.x, w1, y1[0]), y1[1] = fmaf(x.y, w1, y1[1]), y1[2] = fmaf(x.z, w1, y1[2]), y1[3] = fmaf(x.w, w1, y1[3]);
    }
  }
}

// bilinear (zeros padding, align_corners=True) of channels {lane, lane+32} at normalised (gx, gy)
__device__ __forceinline__ void fetch_map(const float* __restrict__ map, int H, int W, float gx, float gy, int lane,
                                          float& f0, float& f1) {
  f0 = 0.f, f1 = 0.f;
  float fx = ((gx + 1.f) / 2.f) * (float)(W - 1), fy = ((gy + 1.f) / 2.f) * (float)(H - 1);
  float x0 = floorf(fx), y0 = floorf(fy);
  if (!(x0 >= -1.f && x0 <= (float)(W - 1) && y0 >= -1.f && y0 <= (float)(H - 1))) return;
  float x1 = x0 + 1.f, y1 = y0 + 1.f;
  float wnw = (x1 - fx) * (y1 - fy), wne = (fx - x0) * (y1 - fy), wsw = (x1 - fx) * (fy - y0), wse = (fx - x0) * (fy - y0);
  int ix = (int)x0, iy = (int)y0;
  bool inx0 = ix >= 0, inx1 = ix + 1 <= W - 1, iny0 = iy >= 0, iny1 = iy + 1 <= H - 1;
  const float* base = map + ((int64_t)iy * W + ix) * CM;
  const bool c1 = lane + 32 < CM;
  if (iny0 && inx0) { f0 = fmaf(__ldg(base + lane), wnw, f0); if (c1) f1 = fmaf(__ldg(base + lane + 32), wnw, f1); }
  if (iny0 && inx1) { f0 = fmaf(__ldg(base + CM + lane), wne, f0); if (c1) f1 = fmaf(__ldg(base + CM + lane + 32), wne, f1); }
  if (iny1 && inx0) { f0 = fmaf(__ldg(base + (int64_t)W * CM + lane), wsw, f0); if (c1) f1 = fmaf(__ldg(base + (int64_t)W * CM + lane + 32), wsw, f1); }
  if (iny1 && inx1) { f0 = fmaf(__ldg(base + (int64_t)W * CM + CM + lane), wse, f0); if (c1) f1 = fmaf(__ldg(base + (int64_t)W * CM + CM + lane + 32), wse, f1); }
}

// Features of up to four valid views (slots g0..g0+3 of the `valid` mask): bilinear fetch of the 59 channels
// (lanes own channels lane and lane+32) plus the direction feature ray_dir_fc(ray_diff) (reference
// rendering_network.py:44-47,88-90).  Padded slots return zeros and weight 0.  If sRGB != nullptr the original
// colours of the views are stored at sRGB[slot*4 + c].
__device__ __forceinline__ void view_group_features(const o2345_views& views, const BlendSample& s, int g0, const float* __restrict__ sP, float* sA4, float* sB4, int lane,
                                                    int (&vid)[4], float (&wq)[4], float (&a0)[4], float (&a1)[4],
                                                    float* sRGB) {
  const int H = views.H, W = views.W;
  unsigned m = s.valid;
  for (int k = 0; k < g0; ++k) m &= m - 1;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    vid[q] = m ? __ffs(m) - 1 : -1;
    m &= m - 1;
  }
  float f0[4], f1[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    int vq = vid[q] >= 0 ? vid[q] : 0;
    wq[q] = vid[q] >= 0 ? __shfl_sync(0xffffffffu, s.wv, vq) : 0.f;
    float vgx = __shfl_sync(0xffffffffu, s.gx, vq), vgy = __shfl_sync(0xffffffffu, s.gy, vq);
    fetch_map(views.maps + (int64_t)vq * H * W * CM, H, W, vgx, vgy, lane, f0[q], f1[q]);
    float r0 = __shfl_sync(0xffffffffu, s.rd0, vq), r1 = __shfl_sync(0xffffffffu, s.rd1, vq);
    float r2 = __shfl_sync(0xffffffffu, s.rd2, vq), r3 = __shfl_sync(0xffffffffu, s.rd3, vq);
    if (lane == 0) sA4[0 * 4 + q] = r0, sA4[1 * 4 + q] = r1, sA4[2 * 4 + q] = r2, sA4[3 * 4 + q] = r3;
  }
  __syncwarp();
  float hd[4], dmy[4], d0[4], d1[4];
  matvec4<4, 16, 16>(sP + P_D0W, sA4, lane, lane < 16 ? sP[P_D0B + lane] : 0.f, 0.f, hd, dmy);
  if (lane < 16) {
#pragma unroll
    for (int q = 0; q < 4; ++q) sB4[lane * 4 + q] = eluf_(hd[q]);
  }
  __syncwarp();
  matvec4<16, 64, 64>(sP + P_D1W, sB4, lane, sP[P_D1B + lane], sP[P_D1B + 32 + lane], d0, d1);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    bool on = g0 + q < s.nvalid;
    if (on && sRGB != nullptr && lane < 3) sRGB[(g0 + q) * 4 + lane] = f0[q];
    a0[q] = on ? f0[q] + eluf_(d0[q]) : 0.f;
    a1[q] = (on && lane + 32 < NF) ? f1[q] + eluf_(d1[q]) : 0.f;
  }
  __syncwarp();
}

__global__ void __launch_bounds__(BW * 32, 1)
render_blend_kernel(o2345_points src, int64_t n, const uint8_t* __restrict__ active, const float* __restrict__ vol,
                    const float* __restrict__ occ, int D, o2345_views views, int dir_mode,
                    const float* __restrict__ query_center, const float* __restrict__ dirs,
                    const float* __restrict__ pack, float* __restrict__ rgb_out, int32_t* __restrict__ nvalid_out) {
  extern __shared__ __align__(16) float smem[];
  float* sP = smem;
  for (int i = threadIdx.x; i < P_TOTAL; i += blockDim.x) sP[i] = __ldg(pack + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* sX = smem + P_TOTAL + warp * WS_TOTAL;
  float* sRGB = sX + WS_X;
  const int V = views.V, H = views.H, W = views.W;
  const float abs_s = sP[P_S];

  for (int64_t gi = (int64_t)blockIdx.x * BW + warp; gi < n; gi += (int64_t)gridDim.x * BW) {
    if (skip_inactive(active, gi, lane, rgb_out, nvalid_out)) continue;
    const BlendSample s = blend_front_end(src, gi, vol, occ, D, views, dir_mode, query_center, dirs, abs_s, lane);
    if (lane == 0 && nvalid_out) nvalid_out[gi] = s.nvalid;

    if (s.nvalid == 0) {
      // every logit is -1e9: softmax is uniform over ALL views (reference rendering_network.py:119-121)
      float r = 0.f, g = 0.f, b = 0.f;
      for (int v = 0; v < V; ++v) {
        float vgx = __shfl_sync(0xffffffffu, s.gx, v), vgy = __shfl_sync(0xffffffffu, s.gy, v);
        float f0, f1;
        fetch_map(views.maps + (int64_t)v * H * W * CM, H, W, vgx, vgy, lane, f0, f1);
        r += __shfl_sync(0xffffffffu, f0, 0), g += __shfl_sync(0xffffffffu, f0, 1), b += __shfl_sync(0xffffffffu, f0, 2);
      }
      if (lane == 0) { rgb_out[3 * gi] = r / (float)V; rgb_out[3 * gi + 1] = g / (float)V; rgb_out[3 * gi + 2] = b / (float)V; }
      continue;
    }

    // ---- pass A over the valid views, four at a time: fetch, direction feature, weighted mean.
    //      The features are recomputed in the later passes instead of being cached per warp: the 8 KB
    //      cache limited the kernel to 12 warps per SM and it was latency bound (ncu: issue active 43 %).
    float mean0 = 0.f, mean1 = 0.f, sq0 = 0.f, sq1 = 0.f;
    float* sA4 = sX;            // [<=64][4] activations, view-interleaved
    float* sB4 = sX + 256;      // second buffer
    for (int g0 = 0; g0 < s.nvalid; g0 += 4) {
      int vid[4];
      float wq[4], a0[4], a1[4];
      view_group_features(views, s, g0, sP, sA4, sB4, lane, vid, wq, a0, a1, sRGB);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        mean0 = fmaf(wq[q], a0[q], mean0), mean1 = fmaf(wq[q], a1[q], mean1);
        sq0 = fmaf(wq[q] * a0[q], a0[q], sq0), sq1 = fmaf(wq[q] * a1[q], a1[q], sq1);
      }
    }
    // sum_v w (f - mean)^2 = sum_v w f^2 - mean^2 (2 - sum_v w): one pass instead of a second fetch of every view
    // (|error| ~ 1e-6 * f^2, two orders below the colour tolerance)
    const float wsum1 = s.wtot / (s.wtot + 1e-8f);
    float var0 = fmaxf(sq0 - mean0 * mean0 * (2.f - wsum1), 0.f);
    float var1 = fmaxf(sq1 - mean1 * mean1 * (2.f - wsum1), 0.f);
    // ---- per-sample part of base_fc[0]: [geo(16), mean(59), var(59)] -> 64
    __syncwarp();
    if (lane < 16) sX[lane] = s.geo;
    sX[16 + lane] = mean0;
    if (lane + 32 < NF) sX[16 + 32 + lane] = mean1;
    sX[75 + lane] = var0;
    if (lane + 32 < NF) sX[75 + 32 + lane] = var1;
    __syncwarp();
    float hs0, hs1;
    matvec<134, 64, 64>(sP + P_B0W, sP + P_B0B, sX, lane, hs0, hs1);
    __syncwarp();

    // ---- groups of four valid views share every weight load (4 independent FMA chains per output)
    float logit = -3.4e38f;  // lane v keeps the logit of view v
    for (int g0 = 0; g0 < s.nvalid; g0 += 4) {
      int vid[4];
      float wq[4], a0[4], a1[4];
      view_group_features(views, s, g0, sP, sA4, sB4, lane, vid, wq, a0, a1, nullptr);
      // base_fc[0], per-view part: x1 = elu(hs + Wf . f_v)
#pragma unroll
      for (int q = 0; q < 4; ++q) sA4[lane * 4 + q] = a0[q], sA4[(lane + 32) * 4 + q] = a1[q];
      __syncwarp();
      float y0[4], y1[4];
      matvec4<NF, 64, 64>(sP + P_B0W + 134 * 64, sA4, lane, hs0, hs1, y0, y1);
#pragma unroll
      for (int q = 0; q < 4; ++q) sB4[lane * 4 + q] = eluf_(y0[q]), sB4[(lane + 32) * 4 + q] = eluf_(y1[q]);
      __syncwarp();
      // base_fc[2]: 64 -> 32
      float x2[4], dmy[4];
      matvec4<64, 32, 32>(sP + P_B1W, sB4, lane, sP[P_B1B + lane], 0.f, x2, dmy);
#pragma unroll
      for (int q = 0; q < 4; ++q) x2[q] = eluf_(x2[q]), sA4[lane * 4 + q] = x2[q] * wq[q];
      __syncwarp();
      // vis_fc(x * weight): 32 -> 32 -> (32 residual + 1 visibility)
      float hv[4];
      matvec4<32, 32, 32>(sP + P_V0W, sA4, lane, sP[P_V0B + lane], 0.f, hv, dmy);
#pragma unroll
      for (int q = 0; q < 4; ++q) hv[q] = eluf_(hv[q]), sB4[lane * 4 + q] = hv[q];
      __syncwarp();
      float res[4], x3[4], vis[4];
      matvec4<32, 32, 32>(sP + P_V1W, sB4, lane, sP[P_V1B + lane], 0.f, res, dmy);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float visr = eluf_(warp_sum(hv[q] * sP[P_V1V + lane]) + sP[P_V1VB]);
        vis[q] = fsigmoid_(visr);                       // mask is 1 for the views processed here
        x3[q] = x2[q] + eluf_(res[q]);
        sA4[lane * 4 + q] = x3[q] * vis[q];
      }
      __syncwarp();
      // vis_fc2(x * vis): 32 -> 32 -> 1, sigmoid
      float h2[4];
      matvec4<32, 32, 32>(sP + P_U0W, sA4, lane, sP[P_U0B + lane], 0.f, h2, dmy);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float vis2 = fsigmoid_(warp_sum(eluf_(h2[q]) * sP[P_U1W + lane]) + sP[P_U1B]);
        // rgb_fc input [x(32), vis(1), ray_diff(4)]
        sB4[lane * 4 + q] = x3[q];
        int vq = vid[q] >= 0 ? vid[q] : 0;
        float r0 = __shfl_sync(0xffffffffu, s.rd0, vq), r1 = __shfl_sync(0xffffffffu, s.rd1, vq);
        float r2 = __shfl_sync(0xffffffffu, s.rd2, vq), r3 = __shfl_sync(0xffffffffu, s.rd3, vq);
        if (lane == 0) {
          sB4[32 * 4 + q] = vis2;
          sB4[33 * 4 + q] = r0, sB4[34 * 4 + q] = r1, sB4[35 * 4 + q] = r2, sB4[36 * 4 + q] = r3;
        }
      }
      __syncwarp();
      float q1[4];
      matvec4<37, 16, 16>(sP + P_R0W, sB4, lane, lane < 16 ? sP[P_R0B + lane] : 0.f, 0.f, q1, dmy);
      if (lane < 16) {
#pragma unroll
        for (int q = 0; q < 4; ++q) sA4[lane * 4 + q] = eluf_(q1[q]);
      }
      __syncwarp();
      float q2[4];
      matvec4<16, 8, 8>(sP + P_R1W, sA4, lane, lane < 8 ? sP[P_R1B + lane] : 0.f, 0.f, q2, dmy);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float lg = warp_sum(lane < 8 ? eluf_(q2[q]) * sP[P_R2W + lane] : 0.f) + sP[P_R2B];
        if (lane == vid[q]) logit = lg;
      }
      __syncwarp();
    }
    // ---- softmax over the valid views, blend the ORIGINAL colours
    float lmax = logit;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    float ex = s.vmask ? expf(logit - lmax) : 0.f;
    float den = warp_sum(ex);
    float r = 0.f, g = 0.f, b = 0.f;
    int slot = 0;
    for (unsigned m = s.valid; m; m &= m - 1, ++slot) {
      int v = __ffs(m) - 1;
      float bw = __shfl_sync(0xffffffffu, ex, v) / den;
      r = fmaf(bw, sRGB[slot * 4], r), g = fmaf(bw, sRGB[slot * 4 + 1], g), b = fmaf(bw, sRGB[slot * 4 + 2], b);
    }
    if (lane == 0) { rgb_out[3 * gi] = r; rgb_out[3 * gi + 1] = g; rgb_out[3 * gi + 2] = b; }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------
// B14: NeuS alpha + compositing (reference sparse_neus_renderer.py:340-432)
// ---------------------------------------------------------------------------------------
__global__ void ray_composite_kernel(const float* __restrict__ rays_d, int64_t R, int S,
                                     const float* __restrict__ mid_z, const float* __restrict__ dists,
                                     const float* __restrict__ sdf, const float* __restrict__ grad,
                                     const float* __restrict__ color, const uint8_t* __restrict__ active,
                                     const int32_t* __restrict__ nvalid, float inv_s, float ratio, int has_bg,
                                     float bg, float* __restrict__ o_color, float* __restrict__ o_depth,
                                     float* __restrict__ o_weights, float* __restrict__ o_cdf,
                                     float* __restrict__ o_alpha, float* __restrict__ o_wsum,
                                     uint8_t* __restrict__ o_cmask) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
  float T = 1.f, wsum = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, depth = 0.f;
  int seen = 0;
  for (int s = 0; s < S; ++s) {
    int64_t i = r * S + s;
    float m = active[i] ? 1.f : 0.f;
    float cosv = dx * grad[3 * i] + dy * grad[3 * i + 1] + dz * grad[3 * i + 2];
    float it = -(fmaxf(-cosv * 0.5f + 0.5f, 0.f) * (1.f - ratio) + fmaxf(-cosv, 0.f) * ratio) * m;
    float e = fminf(fmaxf(it, -10.f), 10.f) * dists[i] * 0.5f;
    float sd = sdf[i];
    float pc = sigmoidf_((sd - e) * inv_s), nc = sigmoidf_((sd + e) * inv_s);
    float alpha = fminf(fmaxf((pc - nc + 1e-5f) / (pc + 1e-5f), 0.f), 1.f) * m;
    float w = alpha * T;
    T *= (1.f - alpha + 1e-7f);
    if (o_weights) o_weights[i] = w;
    if (o_cdf) o_cdf[i] = pc;
    if (o_alpha) o_alpha[i] = alpha;
    wsum += w;
    cr = fmaf(color[3 * i], w, cr), cg = fmaf(color[3 * i + 1], w, cg), cb = fmaf(color[3 * i + 2], w, cb);
    depth = fmaf(mid_z[i], w, depth);
    seen += (nvalid[i] >= 2) ? 1 : 0;
  }
  if (has_bg) { float k = bg * (1.f - wsum); cr += k, cg += k, cb += k; }
  o_color[3 * r] = cr, o_color[3 * r + 1] = cg, o_color[3 * r + 2] = cb;
  o_depth[r] = depth;
  if (o_wsum) o_wsum[r] = wsum;
  if (o_cmask) o_cmask[r] = seen > 8 ? 1 : 0;
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int o2345_ray_upsample(const float* rays_o, const float* rays_d, int64_t R, const float* z,
                                  const float* sdf, int S, float inv_s, const float* occ, int D, const float* u,
                                  int n_new, float* new_z, o2345_stream_t stream) {
  O2345_CHECK_ARG(rays_o && rays_d && z && sdf && occ && u && new_z, "null pointer");
  O2345_CHECK_ARG(S >= 2 && S <= 512 && n_new >= 1, "bad sample counts");
  if (R == 0) return O2345_OK;
  size_t smem = (size_t)S * UPT * sizeof(float);
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(ray_upsample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 512 * UPT * 4));
  }
  ray_upsample_kernel<<<cdiv(R, UPT), UPT, smem, (cudaStream_t)stream>>>(rays_o, rays_d, R, z, sdf, S, inv_s, occ, D, u, n_new, new_z);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_ray_merge(const float* z, const float* sdf, int S, const float* new_z, const float* new_sdf,
                               int n_new, int64_t R, float* out_z, float* out_sdf, o2345_stream_t stream) {
  O2345_CHECK_ARG(z && sdf && new_z && new_sdf && out_z && out_sdf, "null pointer");
  if (R == 0) return O2345_OK;
  ray_merge_kernel<<<cdiv(R, 128), 128, 0, (cudaStream_t)stream>>>(z, sdf, S, new_z, new_sdf, n_new, R, out_z, out_sdf);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_ray_midpoints(const float* rays_o, const float* rays_d, int64_t R, const float* z, int S,
                                   float sample_dist, const float* occ, int D, float* mid_z, float* dists,
                                   uint8_t* active, o2345_stream_t stream) {
  O2345_CHECK_ARG(rays_o && rays_d && z && occ && mid_z && dists && active, "null pointer");
  if (R == 0) return O2345_OK;
  ray_mid_kernel<<<cdiv(R * S, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, R, z, S, sample_dist, occ, D, mid_z, dists, active);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_ray_midpoints_per_ray(const float* rays_o, const float* rays_d, int64_t R, const float* z, int S,
                                           const float* sample_dist, const float* occ, int D, float* mid_z, float* dists,
                                           uint8_t* active, o2345_stream_t stream) {
  O2345_CHECK_ARG(rays_o && rays_d && z && sample_dist && occ && mid_z && dists && active, "null pointer");
  if (R == 0) return O2345_OK;
  ray_mid_per_ray_kernel<<<cdiv(R * S, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, R, z, S, sample_dist, occ, D, mid_z,
                                                                             dists, active);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

namespace o2345 {
int launch_render_blend_tc(const o2345_points* src, int64_t n, const uint8_t* active, const float* vol_cl, const float* occ, int D,
                           const o2345_views* views, int dir_mode, const float* query_center, const float* dirs,
                           const float* rnet_pack, float* rgb, int32_t* nvalid, cudaStream_t st);   // render_tc.cu
}

extern "C" int o2345_render_blend(const o2345_points* src, int64_t n, const uint8_t* active, const float* vol_cl,
                                  const float* occ, int D, const o2345_views* views, int dir_mode,
                                  const float* query_center, const float* dirs, const float* rnet_pack, int precision,
                                  float* rgb, int32_t* nvalid, o2345_stream_t stream) {
  O2345_CHECK_ARG(src && vol_cl && occ && views && rnet_pack && rgb, "null pointer");
  O2345_CHECK_ARG(src->mode == O2345_PTS_EXPLICIT || src->mode == O2345_PTS_RAYS, "explicit or ray points only");
  O2345_CHECK_ARG(views->V >= 1 && views->V <= 32 && views->maps && views->proj && views->centers, "1..32 views");
  O2345_CHECK_ARG((dir_mode == 0 && query_center) || (dir_mode == 1 && dirs) || dir_mode == 2, "direction source missing");
  O2345_CHECK_ARG(dir_mode != 2 || src->mode == O2345_PTS_RAYS, "dir_mode 2 (ray origins) needs ray points");
  O2345_CHECK_ARG(precision == O2345_BLEND_FP32 || precision == O2345_BLEND_TC_FP16, "unknown precision");
  if (n == 0) return O2345_OK;
  if (precision == O2345_BLEND_TC_FP16)
    return launch_render_blend_tc(src, n, active, vol_cl, occ, D, views, dir_mode, query_center, dirs, rnet_pack, rgb, nvalid,
                                  (cudaStream_t)stream);
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(render_blend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BLEND_SMEM));
  }
  int64_t need = (n + BW - 1) / BW;
  int grid = (int)(need < (int64_t)sm_count() ? need : (int64_t)sm_count());
  render_blend_kernel<<<grid, BW * 32, BLEND_SMEM, (cudaStream_t)stream>>>(*src, n, active, vol_cl, occ, D, *views, dir_mode,
                                                                         query_center, dirs, rnet_pack, rgb, nvalid);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_ray_composite(const float* rays_d, int64_t R, int S, const float* mid_z, const float* dists,
                                   const float* sdf, const float* grad, const float* color, const uint8_t* active,
                                   const int32_t* nvalid, float inv_s, float alpha_inter_ratio, int has_background,
                                   float background, float* color_out, float* depth_out, float* weights_out,
                                   float* cdf_out, float* alpha_out, float* weights_sum_out,
                                   uint8_t* color_mask_out, o2345_stream_t stream) {
  O2345_CHECK_ARG(rays_d && mid_z && dists && sdf && grad && color && active && nvalid && color_out && depth_out, "null pointer");
  if (R == 0) return O2345_OK;
  ray_composite_kernel<<<cdiv(R, 128), 128, 0, (cudaStream_t)stream>>>(rays_d, R, S, mid_z, dists, sdf, grad, color, active, nvalid,
                                                                       inv_s, alpha_inter_ratio, has_background, background,
                                                                       color_out, depth_out, weights_out, cdf_out,
                                                                       alpha_out, weights_sum_out, color_mask_out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
