// Shared pieces of the two view-blending kernels (render_blend_kernel in render.cu: fp32 FMA; render_blend_tc_kernel in
// render_tc.cu: mma.sync): the packed GeneralRenderingNetwork weights and the per-sample front end that runs before the
// MLPs.  One warp owns one sample point; in the front end lane v < V stands for source view v.
#pragma once
#include "common.cuh"

namespace o2345 {
namespace rpack {

// Layout of the packed GeneralRenderingNetwork weights (O2345_RNET_PACK_FLOATS floats, every matrix stored [in][out]);
// written by o2345/rendering_network.py::GeneralRenderingNetwork.packed().
// Reference: reconstruction/models/rendering_network.py:40-73 (layer shapes).
constexpr int CM = O2345_MAP_CH;   // 60 channels per pixel: rgb(3) + feat(56) + pad(1)
constexpr int NF = 59;

constexpr int P_D0W = 0;                    // ray_dir_fc[0]  [4][16]
constexpr int P_D0B = P_D0W + 64;           // [16]
constexpr int P_D1W = P_D0B + 16;           // ray_dir_fc[2]  [16][64]  (59 used)
constexpr int P_D1B = P_D1W + 1024;         // [64]
constexpr int P_B0W = P_D1B + 64;           // base_fc[0]     [193][64]: rows 0..15 geo, 16..74 mean, 75..133 var, 134..192 feat
constexpr int P_B0B = P_B0W + 193 * 64;     // [64]
constexpr int P_B1W = P_B0B + 64;           // base_fc[2]     [64][32]
constexpr int P_B1B = P_B1W + 2048;         // [32]
constexpr int P_V0W = P_B1B + 32;           // vis_fc[0]      [32][32]
constexpr int P_V0B = P_V0W + 1024;         // [32]
constexpr int P_V1W = P_V0B + 32;           // vis_fc[2]      [32][32]  residual outputs
constexpr int P_V1B = P_V1W + 1024;         // [32]
constexpr int P_V1V = P_V1B + 32;           // [32]      visibility output row
constexpr int P_V1VB = P_V1V + 32;          // [4]       its bias (first element)
constexpr int P_U0W = P_V1VB + 4;           // vis_fc2[0]     [32][32]
constexpr int P_U0B = P_U0W + 1024;         // [32]
constexpr int P_U1W = P_U0B + 32;           // vis_fc2[2]     [32]
constexpr int P_U1B = P_U1W + 32;           // [4]
constexpr int P_R0W = P_U1B + 4;            // rgb_fc[0]      [37][16]
constexpr int P_R0B = P_R0W + 592;          // [16]
constexpr int P_R1W = P_R0B + 16;           // rgb_fc[2]      [16][8]
constexpr int P_R1B = P_R1W + 128;          // [8]
constexpr int P_R2W = P_R1B + 8;            // rgb_fc[4]      [8]
constexpr int P_R2B = P_R2W + 8;            // [4]
constexpr int P_S = P_R2B + 4;              // [4]  |s| of the pooling weight
constexpr int P_TOTAL = P_S + 4;
static_assert(P_TOTAL == O2345_RNET_PACK_FLOATS, "header and kernels disagree on the rendering-net pack");

}  // namespace rpack

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// An inactive sample carries weight exactly 0 in the compositing: it gets colour 0 and no valid views.
__device__ __forceinline__ bool skip_inactive(const uint8_t* __restrict__ active, int64_t gi, int lane, float* __restrict__ rgb_out,
                                              int32_t* __restrict__ nvalid_out) {
  if (!active || active[gi] != 0) return false;
  if (lane < 3) rgb_out[3 * gi + lane] = 0.f;
  if (lane == 0 && nvalid_out) nvalid_out[gi] = 0;
  return true;
}

// What the front end knows about one sample.  Per-lane fields describe source view `lane` (lane < V); the rest is
// the same in every lane.
struct BlendSample {
  float geo;                  // lane < 16: channel `lane` of the geometry feature
  float gx, gy;               // projection into view `lane`, normalised to [-1, 1]; 2 outside the image
  float rd0, rd1, rd2, rd3;   // ray difference of view `lane`: unit direction difference and cosine
  float wv;                   // normalised pooling weight of view `lane`, 0 for masked views
  float wtot;                 // sum of the un-normalised pooling weights
  bool vmask;                 // view `lane` sees the sample
  unsigned valid;             // ballot of vmask
  int nvalid;                 // number of valid views
};

// Sample point gi, its geometry feature and occupancy (ATen trilinear, zeros padding, align_corners=True; reference
// render_utils.py:54-85, projector.py:168-183), then the lanes as views: projection, view mask, ray difference and pooling
// weight.  dir_mode 0: the target direction is camera-to-point (rendering); 1: dirs[gi] (the normals of vertex colours);
// 2: ray-origin-to-point, the origin of sample gi's own ray (ray points only: cameras that differ from ray to ray).
__device__ __forceinline__ BlendSample blend_front_end(const o2345_points& src, int64_t gi, const float* __restrict__ vol,
                                                       const float* __restrict__ occ, int D, const o2345_views& views, int dir_mode,
                                                       const float* __restrict__ query_center, const float* __restrict__ dirs,
                                                       float abs_s, int lane) {
  BlendSample s;
  float px, py, pz;
  __builtin_assume(src.mode != O2345_PTS_LATTICE);   // o2345_render_blend refuses lattice points: no code for them
  load_point(src, gi, px, py, pz);
  s.geo = 0.f;
  float occv = 0.f;
  {
    float p[3] = {px, py, pz};
    float f[3], w1[3];
    bool fin = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      float t = ((p[a] + 1.f) / 2.f) * (float)(D - 1);
      f[a] = floorf(t);
      w1[a] = t - f[a];
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
        if (lane < 16) s.geo = fmaf(__ldg(vol + cell * 16 + lane), w, s.geo);
        occv = fmaf(__ldg(occ + cell), w, occv);
      }
    }
  }
  const bool gmask = (fabsf(px) < 1.f) && (fabsf(py) < 1.f) && (fabsf(pz) < 1.f) && (occv > 0.f);
  // ---- lanes as views
  s.gx = 2.f, s.gy = 2.f, s.rd0 = 0.f, s.rd1 = 0.f, s.rd2 = 0.f, s.rd3 = 0.f;
  float ev = 3.4e38f;
  s.vmask = false;
  float tx, ty, tz;
  if (dir_mode != 1) {
    // mode 2: every ray is its own camera centre (rays of several cameras in one launch), so c = rays_o[ray]
    const float* c = dir_mode == 0 ? query_center : src.rays_o + 3 * (gi / src.S);
    tx = c[0] - px, ty = c[1] - py, tz = c[2] - pz;
    float nn = sqrtf(tx * tx + ty * ty + tz * tz) + 1e-6f;
    tx /= nn, ty /= nn, tz /= nn;
  } else {
    tx = dirs[3 * gi], ty = dirs[3 * gi + 1], tz = dirs[3 * gi + 2];
  }
  if (lane < views.V) {
    const float* P = views.proj + 12 * lane;
    float X = P[0] * px + P[1] * py + P[2] * pz + P[3];
    float Y = P[4] * px + P[5] * py + P[6] * pz + P[7];
    float Z = fmaxf(P[8] * px + P[9] * py + P[10] * pz + P[11], 1e-3f);
    s.gx = 2.f * (X / Z) / (views.sizeW - 1.f) - 1.f;
    s.gy = 2.f * (Y / Z) / (views.sizeH - 1.f) - 1.f;
    if (!(s.gx <= 1.f && s.gx >= -1.f)) s.gx = 2.f;
    if (!(s.gy <= 1.f && s.gy >= -1.f)) s.gy = 2.f;
    s.vmask = gmask && (fabsf(s.gx) < 1.f) && (fabsf(s.gy) < 1.f);
    float cx = views.centers[3 * lane] - px, cy = views.centers[3 * lane + 1] - py, cz = views.centers[3 * lane + 2] - pz;
    float nn = sqrtf(cx * cx + cy * cy + cz * cz) + 1e-6f;
    cx /= nn, cy /= nn, cz /= nn;
    float ddx = tx - cx, ddy = ty - cy, ddz = tz - cz;
    float dn = fmaxf(sqrtf(ddx * ddx + ddy * ddy + ddz * ddz), 1e-6f);
    s.rd0 = ddx / dn, s.rd1 = ddy / dn, s.rd2 = ddz / dn;
    s.rd3 = tx * cx + ty * cy + tz * cz;
    ev = expf(abs_s * (s.rd3 - 1.f));
  }
  float emin = ev;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) emin = fminf(emin, __shfl_xor_sync(0xffffffffu, emin, o));
  float wv = s.vmask ? (ev - emin) : 0.f;
  s.wtot = warp_sum(wv);
  s.wv = wv / (s.wtot + 1e-8f);
  s.valid = __ballot_sync(0xffffffffu, s.vmask);
  s.nvalid = __popc(s.valid);
  return s;
}

}  // namespace o2345
