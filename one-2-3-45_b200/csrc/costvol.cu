// Cost-volume build: frustum mask, fused back-project + variance/mean.
// Rows B3/B4/B5/B7 of SURVEY.md section 8.  The kept voxels are compacted by o2345_compact (scan.cu) in ascending
// x*D*D + y*D + z order, as reference sparse_sdf_network.py:321-334 keeps them.
//
//   frustum_mask_kernel   one thread per lattice voxel, all views: bit-exact restatement of
//                         reference ops/back_project.py:44-61 (separately rounded mul/add so
//                         that the CPU oracle reproduces every threshold decision);
//   costvol_gather_kernel four threads per kept voxel, each owning 4 of the 16 channels:
//                         per view one projection, four 16-byte taps from the channel-last
//                         feature map, running sum / sum of squares; the [Nv,V,16] tensor of
//                         the reference (1.76 GB at 96^3 x 32 views) is never materialised.
#include "common.cuh"

namespace o2345 {
namespace {

struct Proj {
  float gx, gy, z;
  bool vis;
};

// world -> normalised grid of one view; operation order matches oracle project_voxels().
__device__ __forceinline__ Proj project(const float* __restrict__ P, float wx, float wy, float wz,
                                        float size_w1, float size_h1) {
  float ix = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[0], wx), __fmul_rn(P[1], wy)), __fmul_rn(P[2], wz)), P[3]);
  float iy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4], wx), __fmul_rn(P[5], wy)), __fmul_rn(P[6], wz)), P[7]);
  float iz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[8], wx), __fmul_rn(P[9], wy)), __fmul_rn(P[10], wz)), P[11]);
  if (iz >= 0.f) iz = fmaxf(iz, 1e-6f);
  float u = __fdiv_rn(ix, iz), v = __fdiv_rn(iy, iz);
  Proj r;
  r.gx = __fadd_rn(__fdiv_rn(__fmul_rn(2.f, u), size_w1), -1.f);
  r.gy = __fadd_rn(__fdiv_rn(__fmul_rn(2.f, v), size_h1), -1.f);
  r.z = iz;
  r.vis = (fabsf(r.gx) <= 1.f) && (fabsf(r.gy) <= 1.f) && (iz > 0.f);
  return r;
}

__device__ __forceinline__ void voxel_world(int64_t lin, int D, float vs, const float* __restrict__ origin,
                                            float& wx, float& wy, float& wz) {
  int z = (int)(lin % D);
  int y = (int)((lin / D) % D);
  int x = (int)(lin / ((int64_t)D * D));
  wx = __fadd_rn(__fmul_rn((float)x, vs), origin[0]);
  wy = __fadd_rn(__fmul_rn((float)y, vs), origin[1]);
  wz = __fadd_rn(__fmul_rn((float)z, vs), origin[2]);
}

__global__ void frustum_mask_kernel(const float* __restrict__ proj, int V, const float* __restrict__ origin,
                                    float vs, int D, float size_w1, float size_h1, int min_views,
                                    uint32_t* __restrict__ bits, uint8_t* __restrict__ keep) {
  extern __shared__ float sP[];  // [V][12]
  for (int i = threadIdx.x; i < V * 12; i += blockDim.x) sP[i] = proj[(i / 12) * 16 + (i % 12)];
  __syncthreads();
  int64_t n = (int64_t)D * D * D;
  int64_t lin = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (lin >= n) return;
  float wx, wy, wz;
  voxel_world(lin, D, vs, origin, wx, wy, wz);
  uint32_t m = 0;
  for (int v = 0; v < V; ++v)
    if (project(sP + 12 * v, wx, wy, wz, size_w1, size_h1).vis) m |= (1u << v);
  bits[lin] = m;
  keep[lin] = __popc(m) > min_views ? 1 : 0;
}

// ---------------------------------------------------------------------------------------
// fused back-projection + variance/mean
// ---------------------------------------------------------------------------------------
// C channels per view (C / 4 threads per kept voxel, one channel quad each).  cost row = [var(C), mean(C)], followed by
// the 16 features of the voxel's parent (pre_feats[parent[lin]]) when PARENT (lod > 0, reference
// sparse_sdf_network.py:336-374: cat([volume, up_feat])).
template <int C, bool PARENT>
__global__ void __launch_bounds__(256)
costvol_gather_kernel(const float* __restrict__ feats, int V, int h, int w, float size_w1, float size_h1,
                      const float* __restrict__ proj, const float* __restrict__ origin, float vs, int D,
                      const int32_t* __restrict__ rows, const int32_t* __restrict__ count,
                      const uint32_t* __restrict__ bits, const int32_t* __restrict__ parent,
                      const float* __restrict__ pre_feats, float* __restrict__ cost) {
  constexpr int Q = C / 4;                       // threads per row
  constexpr int LD = 2 * C + (PARENT ? 16 : 0);  // floats per cost row
  extern __shared__ float sP[];
  for (int i = threadIdx.x; i < V * 12; i += blockDim.x) sP[i] = proj[(i / 12) * 16 + (i % 12)];
  __syncthreads();
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = t / Q;
  int q = (int)(t % Q);  // channel quad
  if (row >= *count) return;
  int64_t lin = rows[row];
  float wx, wy, wz;
  voxel_world(lin, D, vs, origin, wx, wy, wz);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), sq = s;
  const float wm1 = (float)(w - 1), hm1 = (float)(h - 1);
  for (int v = 0; v < V; ++v) {
    Proj p = project(sP + 12 * v, wx, wy, wz, size_w1, size_h1);
    // ATen grid_sampler_2d, bilinear, zeros padding, align_corners=True
    float fx = ((p.gx + 1.f) / 2.f) * wm1, fy = ((p.gy + 1.f) / 2.f) * hm1;
    float x0 = floorf(fx), y0 = floorf(fy);
    // all four taps outside the map (or non-finite coordinates): the view contributes zeros
    if (!(x0 >= -1.f && x0 <= wm1 && y0 >= -1.f && y0 <= hm1)) continue;
    float x1 = x0 + 1.f, y1 = y0 + 1.f;
    float wnw = (x1 - fx) * (y1 - fy), wne = (fx - x0) * (y1 - fy);
    float wsw = (x1 - fx) * (fy - y0), wse = (fx - x0) * (fy - y0);
    int ix0 = (int)x0, iy0 = (int)y0;
    bool inx0 = ix0 >= 0, inx1 = ix0 + 1 <= w - 1, iny0 = iy0 >= 0, iny1 = iy0 + 1 <= h - 1;
    const float* base = feats + (((int64_t)v * h + iy0) * w + ix0) * C + 4 * q;
    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
    if (iny0 && inx0) { float4 a = ldg4(base); f.x = fmaf(a.x, wnw, f.x); f.y = fmaf(a.y, wnw, f.y); f.z = fmaf(a.z, wnw, f.z); f.w = fmaf(a.w, wnw, f.w); }
    if (iny0 && inx1) { float4 a = ldg4(base + C); f.x = fmaf(a.x, wne, f.x); f.y = fmaf(a.y, wne, f.y); f.z = fmaf(a.z, wne, f.z); f.w = fmaf(a.w, wne, f.w); }
    if (iny1 && inx0) { float4 a = ldg4(base + (int64_t)w * C); f.x = fmaf(a.x, wsw, f.x); f.y = fmaf(a.y, wsw, f.y); f.z = fmaf(a.z, wsw, f.z); f.w = fmaf(a.w, wsw, f.w); }
    if (iny1 && inx1) { float4 a = ldg4(base + (int64_t)w * C + C); f.x = fmaf(a.x, wse, f.x); f.y = fmaf(a.y, wse, f.y); f.z = fmaf(a.z, wse, f.z); f.w = fmaf(a.w, wse, f.w); }
    s.x += f.x; s.y += f.y; s.z += f.z; s.w += f.w;
    sq.x = fmaf(f.x, f.x, sq.x); sq.y = fmaf(f.y, f.y, sq.y); sq.z = fmaf(f.z, f.z, sq.z); sq.w = fmaf(f.w, f.w, sq.w);
  }
  float inv = 1.f / ((float)__popc(bits[lin]) + 1e-5f);
  float4 mean = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
  float4 var = make_float4(sq.x * inv - mean.x * mean.x, sq.y * inv - mean.y * mean.y,
                           sq.z * inv - mean.z * mean.z, sq.w * inv - mean.w * mean.w);
  *reinterpret_cast<float4*>(cost + row * LD + 4 * q) = var;
  *reinterpret_cast<float4*>(cost + row * LD + C + 4 * q) = mean;
  if (PARENT) {
    constexpr int PF = 16 / Q;                   // parent features copied per thread
    const float* src = pre_feats + (int64_t)parent[lin] * 16 + PF * q;
#pragma unroll
    for (int k = 0; k < PF; k += 4) *reinterpret_cast<float4*>(cost + row * LD + 2 * C + PF * q + k) = ldg4(src + k);
  }
}

// ---------------------------------------------------------------------------------------
// lod-0 pruning (reference SparseNeuSRenderer.get_valid_sparse_coords_by_sdf, sparse_neus_renderer.py:835-857):
// avg_pool3d(|sdf| < t, k=7, s=1, p=3) > 0 is "the minimum of |sdf| over the 7^3 window (clipped at the border) is < t",
// for every t at once.  Separable: a 7-tap minimum along z, then y, then x.
// ---------------------------------------------------------------------------------------
constexpr int PRUNE_R = 3;
constexpr int MAX_RUNGS = 16;
struct Ladder {
  int n;
  float t[MAX_RUNGS];
};

// out[i] = min over |k| <= 3 along the axis of stride `stride` (clipped), of (ABS ? |in| : in)
template <bool ABS>
__global__ void window_min_kernel(const float* __restrict__ in, int D, int64_t stride, float* __restrict__ out) {
  int64_t n = (int64_t)D * D * D;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = (int)((i / stride) % D);
  float m = INFINITY;
  for (int k = max(0, c - PRUNE_R); k <= min(D - 1, c + PRUNE_R); ++k) {
    float v = __ldg(in + i + (int64_t)(k - c) * stride);
    m = fminf(m, ABS ? fabsf(v) : v);
  }
  out[i] = m;
}

// last (x) pass: minabs = occ > 0 ? window minimum : +inf, and per rung the number of voxels with minabs < ladder[r]
__global__ void prune_final_kernel(const float* __restrict__ in, const float* __restrict__ occ, int D,
                                   Ladder ladder, float* __restrict__ minabs, int32_t* __restrict__ counts) {
  int64_t n = (int64_t)D * D * D;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float m = INFINITY;
  if (i < n) {
    int c = (int)(i / ((int64_t)D * D));
    float w = INFINITY;
    for (int k = max(0, c - PRUNE_R); k <= min(D - 1, c + PRUNE_R); ++k)
      w = fminf(w, __ldg(in + i + (int64_t)(k - c) * D * D));
    if (occ[i] > 0.f) m = w;
    minabs[i] = m;
  }
  for (int r = 0; r < ladder.n; ++r) {
    int c = __syncthreads_count(m < ladder.t[r]);   // (NaN < t is false, as in torch)
    if (threadIdx.x == 0 && c) atomicAdd(counts + r, c);
  }
}

__global__ void prune_select_kernel(const float* __restrict__ minabs, int64_t n, float t, uint8_t* __restrict__ keep) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[i] = minabs[i] < t ? 1 : 0;
}

__global__ void clear_flags_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ idx, int64_t n,
                                   uint8_t* __restrict__ flags) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[rows[idx[i]]] = 0;
}

__global__ void gather_rows_kernel(const int32_t* __restrict__ rows, int64_t n, int D, const float* __restrict__ vol_cf,
                                   int C, float* __restrict__ coords, float* __restrict__ feats) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t lin = rows[i], cells = (int64_t)D * D * D;
  coords[4 * i] = 0.f;
  coords[4 * i + 1] = (float)(lin / ((int64_t)D * D));
  coords[4 * i + 2] = (float)((lin / D) % D);
  coords[4 * i + 3] = (float)(lin % D);
  for (int c = 0; c < C; ++c) feats[i * C + c] = vol_cf[c * cells + lin];
}

// ---------------------------------------------------------------------------------------
// lod-1 children (reference SparseSdfNetwork.upsample + the `> 1` view filter, sparse_sdf_network.py:198-219,340-359)
// ---------------------------------------------------------------------------------------
__global__ void lod_children_kernel(const float* __restrict__ pre_coords, int64_t n, int D1,
                                    const uint8_t* __restrict__ fkeep, uint8_t* __restrict__ keep,
                                    int32_t* __restrict__ parent, int32_t* __restrict__ err) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c[3];
  for (int a = 0; a < 3; ++a) {
    float f = pre_coords[4 * i + 1 + a];
    // children x .. x+1 must lie in [0, D1); integer coordinates only
    if (!(f >= 0.f && f + 1.f < (float)D1 && f == floorf(f))) { atomicOr(err, 1); return; }
    c[a] = (int)f;
  }
  for (int k = 0; k < 8; ++k) {
    int64_t lin = ((int64_t)(c[0] + (k >> 2)) * D1 + (c[1] + ((k >> 1) & 1))) * D1 + (c[2] + (k & 1));
    if (atomicCAS(parent + lin, -1, (int32_t)i) != -1) { atomicOr(err, 2); continue; }
    keep[lin] = fkeep[lin];
  }
}

__global__ void dense_scatter_kernel(const float* __restrict__ feat, const int32_t* __restrict__ rows,
                                     const int32_t* __restrict__ count, int64_t n_cells,
                                     float* __restrict__ vol_cl, float* __restrict__ vol_cf, float* __restrict__ occ) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = t >> 2;
  int q = (int)(t & 3);
  if (row >= *count) return;
  int64_t lin = rows[row];
  float4 v = ldg4(feat + row * 16 + 4 * q);
  *reinterpret_cast<float4*>(vol_cl + lin * 16 + 4 * q) = v;
  if (vol_cf) {
    vol_cf[(int64_t)(4 * q + 0) * n_cells + lin] = v.x;
    vol_cf[(int64_t)(4 * q + 1) * n_cells + lin] = v.y;
    vol_cf[(int64_t)(4 * q + 2) * n_cells + lin] = v.z;
    vol_cf[(int64_t)(4 * q + 3) * n_cells + lin] = v.w;
  }
  if (q == 0) occ[lin] = 1.f;
}

// occupancy lookup: ATen grid_sample(mode='nearest', align_corners=False) after the xyz->zyx flip
// (reference sparse_neus_renderer.py:153-169); idx = nearbyint(((p+1)*D-1)/2) per axis.
__global__ void occ_nearest_kernel(o2345_points src, int64_t n, const float* __restrict__ occ, int D,
                                   uint8_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float p[3];
  if (src.mode == O2345_PTS_EXPLICIT) {
    p[0] = src.pts[3 * i], p[1] = src.pts[3 * i + 1], p[2] = src.pts[3 * i + 2];
  } else {
    int64_t r = i / src.S;
    int s = (int)(i - r * src.S);
    float t = src.z[r * src.z_stride + s];
    for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(src.rays_o[3 * r + a], __fmul_rn(src.rays_d[3 * r + a], t));
  }
  int idx[3];
  bool ok = true;
  for (int a = 0; a < 3; ++a) {
    float f = nearbyintf(((p[a] + 1.f) * (float)D - 1.f) / 2.f);
    ok = ok && (f >= 0.f) && (f <= (float)(D - 1));
    idx[a] = (int)fminf(fmaxf(f, 0.f), (float)(D - 1));
  }
  float v = ok ? occ[((int64_t)idx[0] * D + idx[1]) * D + idx[2]] : 0.f;
  out[i] = v > 0.f ? 1 : 0;
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int o2345_frustum_mask(const float* proj, int V, const float* origin, float voxel_size, int D,
                                  int sizeH, int sizeW, int min_views, uint32_t* mask_bits, uint8_t* keep,
                                  o2345_stream_t stream) {
  O2345_CHECK_ARG(proj && origin && mask_bits && keep, "null pointer");
  O2345_CHECK_ARG(V >= 1 && V <= 32, "1..32 views supported (mask is one 32-bit word per voxel)");
  O2345_CHECK_ARG(D >= 2 && D <= 1024 && sizeH > 1 && sizeW > 1, "bad sizes");
  int64_t n = (int64_t)D * D * D;
  frustum_mask_kernel<<<cdiv(n, 256), 256, V * 12 * sizeof(float), (cudaStream_t)stream>>>(
      proj, V, origin, voxel_size, D, (float)(sizeW - 1), (float)(sizeH - 1), min_views, mask_bits, keep);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_costvol_gather(const float* feats_nhwc, int V, int h, int w, int sizeH, int sizeW,
                                    const float* proj, const float* origin, float voxel_size, int D,
                                    const int32_t* rows, const int32_t* count, int64_t max_rows,
                                    const uint32_t* mask_bits, float* cost, o2345_stream_t stream) {
  O2345_CHECK_ARG(feats_nhwc && proj && origin && rows && count && mask_bits && cost, "null pointer");
  O2345_CHECK_ARG(V >= 1 && V <= 32 && h > 1 && w > 1 && sizeH > 1 && sizeW > 1 && max_rows > 0, "bad sizes");
  costvol_gather_kernel<16, false><<<cdiv(max_rows * 4, 256), 256, V * 12 * sizeof(float), (cudaStream_t)stream>>>(
      feats_nhwc, V, h, w, (float)(sizeW - 1), (float)(sizeH - 1), proj, origin, voxel_size, D, rows, count,
      mask_bits, nullptr, nullptr, cost);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_dense_scatter(const float* feat, const int32_t* rows, const int32_t* count, int64_t max_rows,
                                   int D, float* vol_cl, float* vol_cf, float* occ, o2345_stream_t stream) {
  O2345_CHECK_ARG(feat && rows && count && vol_cl && occ, "null pointer");
  int64_t n = (int64_t)D * D * D;
  cudaStream_t st = (cudaStream_t)stream;
  O2345_CUDA(cudaMemsetAsync(vol_cl, 0, n * 16 * sizeof(float), st));
  if (vol_cf) O2345_CUDA(cudaMemsetAsync(vol_cf, 0, n * 16 * sizeof(float), st));
  O2345_CUDA(cudaMemsetAsync(occ, 0, n * sizeof(float), st));
  dense_scatter_kernel<<<cdiv(max_rows * 4, 256), 256, 0, st>>>(feat, rows, count, n, vol_cl, vol_cf, occ);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_occ_nearest(const o2345_points* src, int64_t n, const float* occ, int D, uint8_t* out,
                                 o2345_stream_t stream) {
  O2345_CHECK_ARG(src && occ && out, "null pointer");
  O2345_CHECK_ARG(src->mode == O2345_PTS_EXPLICIT || src->mode == O2345_PTS_RAYS, "explicit or ray points only");
  if (n == 0) return O2345_OK;
  occ_nearest_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(*src, n, occ, D, out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_costvol_gather_lod(const float* feats_nhwc, int C, int V, int h, int w, int sizeH, int sizeW,
                                        const float* proj, const float* origin, float voxel_size, int D,
                                        const int32_t* rows, const int32_t* count, int64_t max_rows,
                                        const uint32_t* mask_bits, const int32_t* parent, const float* pre_feats,
                                        float* cost, o2345_stream_t stream) {
  O2345_CHECK_ARG(feats_nhwc && proj && origin && rows && count && mask_bits && cost, "null pointer");
  O2345_CHECK_ARG(C == 8 || C == 16, "8 or 16 compressed channels");
  O2345_CHECK_ARG((parent == nullptr) == (pre_feats == nullptr), "parent and pre_feats go together");
  O2345_CHECK_ARG(V >= 1 && V <= 32 && h > 1 && w > 1 && sizeH > 1 && sizeW > 1 && max_rows > 0, "bad sizes");
  const int blocks = cdiv(max_rows * (C / 4), 256);
  const size_t smem = V * 12 * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  const float sw1 = (float)(sizeW - 1), sh1 = (float)(sizeH - 1);
  if (C == 8 && parent)
    costvol_gather_kernel<8, true><<<blocks, 256, smem, st>>>(feats_nhwc, V, h, w, sw1, sh1, proj, origin, voxel_size, D, rows,
                                                              count, mask_bits, parent, pre_feats, cost);
  else if (C == 8)
    costvol_gather_kernel<8, false><<<blocks, 256, smem, st>>>(feats_nhwc, V, h, w, sw1, sh1, proj, origin, voxel_size, D, rows,
                                                               count, mask_bits, nullptr, nullptr, cost);
  else if (parent)
    costvol_gather_kernel<16, true><<<blocks, 256, smem, st>>>(feats_nhwc, V, h, w, sw1, sh1, proj, origin, voxel_size, D, rows,
                                                               count, mask_bits, parent, pre_feats, cost);
  else
    costvol_gather_kernel<16, false><<<blocks, 256, smem, st>>>(feats_nhwc, V, h, w, sw1, sh1, proj, origin, voxel_size, D, rows,
                                                                count, mask_bits, nullptr, nullptr, cost);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_prune_by_sdf(const float* sdf, const float* occ, int D, const float* ladder, int n_ladder,
                                  float* scratch, float* minabs, int32_t* counts, o2345_stream_t stream) {
  O2345_CHECK_ARG(sdf && occ && ladder && scratch && minabs && counts, "null pointer");
  O2345_CHECK_ARG(D >= 1 && D <= 1024, "volume side out of range");
  O2345_CHECK_ARG(n_ladder >= 1 && n_ladder <= MAX_RUNGS, "1..16 thresholds");
  // the z and x passes read 3 neighbours on either side of the element they write: no output may alias an input
  O2345_CHECK_ARG(scratch != minabs && scratch != sdf && minabs != sdf, "sdf, scratch and minabs must not alias");
  Ladder lad{};
  lad.n = n_ladder;
  for (int r = 0; r < n_ladder; ++r) lad.t[r] = ladder[r];
  const int64_t n = (int64_t)D * D * D;
  cudaStream_t st = (cudaStream_t)stream;
  O2345_CUDA(cudaMemsetAsync(counts, 0, n_ladder * sizeof(int32_t), st));
  window_min_kernel<true><<<cdiv(n, 256), 256, 0, st>>>(sdf, D, 1, minabs);                // z, |sdf|
  window_min_kernel<false><<<cdiv(n, 256), 256, 0, st>>>(minabs, D, D, scratch);          // y
  prune_final_kernel<<<cdiv(n, 256), 256, 0, st>>>(scratch, occ, D, lad, minabs, counts);  // x, occupancy, counts
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_prune_select(const float* minabs, int64_t n, float threshold, uint8_t* keep, o2345_stream_t stream) {
  O2345_CHECK_ARG(minabs && keep, "null pointer");
  O2345_CHECK_ARG(n > 0, "element count out of range");
  prune_select_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(minabs, n, threshold, keep);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_clear_flags(const int32_t* rows, const int32_t* idx, int64_t n, uint8_t* flags, o2345_stream_t stream) {
  O2345_CHECK_ARG(n >= 0, "negative count");
  if (n == 0) return O2345_OK;
  O2345_CHECK_ARG(rows && idx && flags, "null pointer");
  clear_flags_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(rows, idx, n, flags);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_gather_rows(const int32_t* rows, int64_t n, int D, const float* vol_cf, int C, float* coords,
                                 float* feats, o2345_stream_t stream) {
  O2345_CHECK_ARG(n >= 0 && D >= 1 && D <= 1024 && C >= 1, "bad sizes");
  if (n == 0) return O2345_OK;
  O2345_CHECK_ARG(rows && vol_cf && coords && feats, "null pointer");
  gather_rows_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(rows, n, D, vol_cf, C, coords, feats);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_lod_children(const float* pre_coords, int64_t n, int D1, const uint8_t* frustum_keep, uint8_t* keep,
                                  int32_t* parent, int32_t* err_scratch, o2345_stream_t stream) {
  O2345_CHECK_ARG(pre_coords && frustum_keep && keep && parent && err_scratch, "null pointer");
  O2345_CHECK_ARG(n >= 1 && n < ((int64_t)1 << 31), "parent count out of range");
  O2345_CHECK_ARG(D1 >= 2 && D1 <= 1024, "volume side out of range");
  const int64_t cells = (int64_t)D1 * D1 * D1;
  cudaStream_t st = (cudaStream_t)stream;
  O2345_CUDA(cudaMemsetAsync(keep, 0, cells, st));
  O2345_CUDA(cudaMemsetAsync(parent, 0xff, cells * sizeof(int32_t), st));
  O2345_CUDA(cudaMemsetAsync(err_scratch, 0, sizeof(int32_t), st));
  lod_children_kernel<<<cdiv(n, 256), 256, 0, st>>>(pre_coords, n, D1, frustum_keep, keep, parent, err_scratch);
  O2345_LAUNCH_CHECK();
  int32_t err = 0;
  O2345_CUDA(cudaMemcpyAsync(&err, err_scratch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  O2345_CUDA(cudaStreamSynchronize(st));
  O2345_CHECK_ARG(!(err & 1), "pre_coords: a coordinate is not an integer with both children inside [0, D1)");
  O2345_CHECK_ARG(!(err & 2), "pre_coords: duplicate parent coordinates");
  return O2345_OK;
}
