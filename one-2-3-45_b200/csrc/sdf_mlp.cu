// SDF query kernel: quirky trilinear latent fetch + positional embedding + weight-normed MLP,
// with an optional analytic gradient (reverse mode through the three layers, the embedding
// and the trilinear weights).  Rows B8/B9/B10 of SURVEY.md section 8.
//
// One persistent CTA per SM (grid = #SMs).  A CTA processes tiles of 128 query points:
//   stage 0  gather the 16-channel latent (8 corners x 64 B, channel-last volume) and build
//            the 39-wide positional embedding; both land in shared memory k-major
//            ([feature][point]) so that the GEMM reads them as conflict-free float4s;
//   stage 1-3  three register-tiled fp32 GEMMs (8 points x 8 outputs per thread) against the
//            layer weights, which are streamed L2 -> shared memory once per tile and layer;
//   stage 4  (grad only) two transposed GEMMs for the backward pass and a per-point
//            contraction with d(embedding)/dx and d(trilinear weights)/dx.
// Arithmetic is fp32 FMA throughout (the reference is fp32; tolerance is stated in the tests).
#include "common.cuh"
#include "sdf_common.cuh"

namespace o2345 {
namespace {

using namespace sdfk;

// VOX: the points and latents come from VoxelSrc (o2345_sdf_voxels) instead of `src` + the trilinear fetch.
template <bool GRAD, bool VOX>
__global__ void __launch_bounds__(NT, 1)
sdf_query_kernel(o2345_points src, int64_t n, const float* __restrict__ vol, int D,
                 const float* __restrict__ wp, const uint8_t* __restrict__ active, float inactive_sdf,
                 float sign, float* __restrict__ o_sdf, float* __restrict__ o_feat,
                 float* __restrict__ o_lat, float* __restrict__ o_grad, VoxelSrc vx) {
  extern __shared__ __align__(16) float smem[];
  float* sAct = smem;                       // [144][TM]
  float* sW = sAct + SM_ACT;                // weights of the current layer / output staging
  float* sA0 = sW + SM_W;                   // [128][TM] layer-0 activations (GRAD only)
  float* sMisc = GRAD ? sA0 + SM_A0 : sA0;  // pts[3][TM], gpart[3][TM], flag[TM]
  float* sPts = sMisc;
  float* sGp = sMisc + 3 * TM;
  int* sFlag = reinterpret_cast<int*>(sMisc + 6 * TM);

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = tx * 8, n0 = ty * 8;
  const int pm = tid & (TM - 1), half = tid >> 7;
  const int64_t ntiles = (n + TM - 1) / TM;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t g0 = tile * TM;
    const int64_t gi = g0 + pm;
    // ---------------- stage 0: point, latent, embedding --------------------------------
    bool act = gi < n && (VOX ? __ldg(vx.occ + gi) > 0.f : (active == nullptr || active[gi] != 0));
    int any = __syncthreads_or(act ? 1 : 0);
    if (!any) {  // nothing to evaluate in this tile: defaults only (block-uniform branch)
      if (half == 0 && gi < n) {
        if (o_sdf) o_sdf[gi] = inactive_sdf;
        if (o_grad) { o_grad[3 * gi] = 0.f; o_grad[3 * gi + 1] = 0.f; o_grad[3 * gi + 2] = 0.f; }
      }
      int64_t cnt = min((int64_t)TM, n - g0);
      if (o_feat) for (int64_t e = tid; e < cnt * 127; e += NT) o_feat[g0 * 127 + e] = 0.f;
      if (o_lat) for (int64_t e = tid; e < cnt * LAT; e += NT) o_lat[g0 * LAT + e] = 0.f;
      continue;
    }
    float px = 0.f, py = 0.f, pz = 0.f;
    if (act) {
      if (VOX) voxel_point(vx, gi, D, px, py, pz);
      else load_point(src, gi, px, py, pz);
    }
    if (half == 0) {
      sPts[pm] = px, sPts[TM + pm] = py, sPts[2 * TM + pm] = pz;
      sFlag[pm] = act ? 1 : 0;
    }
    {
      // latent channels [8*half, 8*half+8)
      Tri t = tri_setup(px, py, pz, D);
      float lat[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) lat[c] = 0.f;
      if (VOX) {
        if (act) {
          float4 v0 = ldg4(vol + gi * LAT + 8 * half), v1 = ldg4(vol + gi * LAT + 8 * half + 4);
          lat[0] = v0.x, lat[1] = v0.y, lat[2] = v0.z, lat[3] = v0.w, lat[4] = v1.x, lat[5] = v1.y, lat[6] = v1.z, lat[7] = v1.w;
        }
      } else if (act && t.inb) {
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
          int dx = corner >> 2, dy = (corner >> 1) & 1, dz = corner & 1;
          int ix = dx ? t.hi[0] : t.base[0], iy = dy ? t.hi[1] : t.base[1], iz = dz ? t.hi[2] : t.base[2];
          // reference weight product order: (w_Z * w_Y) * w_X  (its ix is our z axis)
          float w = ((dz ? t.w1[2] : t.w0[2]) * (dy ? t.w1[1] : t.w0[1])) * (dx ? t.w1[0] : t.w0[0]);
          const float* v = vol + (((int64_t)ix * D + iy) * D + iz) * LAT + 8 * half;
          float4 v0 = ldg4(v), v1 = ldg4(v + 4);
          lat[0] = fmaf(v0.x, w, lat[0]); lat[1] = fmaf(v0.y, w, lat[1]);
          lat[2] = fmaf(v0.z, w, lat[2]); lat[3] = fmaf(v0.w, w, lat[3]);
          lat[4] = fmaf(v1.x, w, lat[4]); lat[5] = fmaf(v1.y, w, lat[5]);
          lat[6] = fmaf(v1.z, w, lat[6]); lat[7] = fmaf(v1.w, w, lat[7]);
        }
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) sAct[(HID + 8 * half + c) * TM + pm] = lat[c];
      // embedding: half 0 -> raw xyz + frequencies 0..2, half 1 -> frequencies 3..5
      float p[3] = {px, py, pz};
      if (half == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) sAct[a * TM + pm] = p[a];
      }
#pragma unroll
      for (int f = 0; f < 3; ++f) {
        int k = 3 * half + f;
        float fr = (float)(1 << k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          float s, c;
          sincosf(fr * p[a], &s, &c);
          sAct[(3 + 6 * k + a) * TM + pm] = s;
          sAct[(3 + 6 * k + 3 + a) * TM + pm] = c;
        }
      }
    }
    load_weights(sW, wp + OFF_W0T, PE * HID);
    __syncthreads();

    float acc[8][8];
    // ---------------- layer 0: 39 -> 128, softplus ------------------------------------
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float b = __ldg(wp + OFF_B0 + n0 + j);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i][j] = b;
    }
    gemm_fwd<PE>(sAct, sW, acc, m0, n0);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 v0 = make_float4(softplus100(acc[0][j]), softplus100(acc[1][j]), softplus100(acc[2][j]), softplus100(acc[3][j]));
      float4 v1 = make_float4(softplus100(acc[4][j]), softplus100(acc[5][j]), softplus100(acc[6][j]), softplus100(acc[7][j]));
      *reinterpret_cast<float4*>(sAct + (n0 + j) * TM + m0) = v0;
      *reinterpret_cast<float4*>(sAct + (n0 + j) * TM + m0 + 4) = v1;
      if (GRAD) {
        *reinterpret_cast<float4*>(sA0 + (n0 + j) * TM + m0) = v0;
        *reinterpret_cast<float4*>(sA0 + (n0 + j) * TM + m0 + 4) = v1;
      }
    }
    load_weights(sW, wp + OFF_W1T, IN1 * HID);
    __syncthreads();
    // ---------------- layer 1: 144 -> 128, softplus -----------------------------------
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float b = __ldg(wp + OFF_B1 + n0 + j);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i][j] = b;
    }
    gemm_fwd<IN1>(sAct, sW, acc, m0, n0);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<float4*>(sAct + (n0 + j) * TM + m0) =
          make_float4(softplus100(acc[0][j]), softplus100(acc[1][j]), softplus100(acc[2][j]), softplus100(acc[3][j]));
      *reinterpret_cast<float4*>(sAct + (n0 + j) * TM + m0 + 4) =
          make_float4(softplus100(acc[4][j]), softplus100(acc[5][j]), softplus100(acc[6][j]), softplus100(acc[7][j]));
    }
    load_weights(sW, wp + OFF_W2T, IN1 * HID);
    __syncthreads();
    // ---------------- layer 2: 144 -> 128 (no activation) -----------------------------
    const bool need_feat = (o_feat != nullptr);
    if (need_feat) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float b = __ldg(wp + OFF_B2 + n0 + j);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i][j] = b;
      }
      gemm_fwd<IN1>(sAct, sW, acc, m0, n0);
      __syncthreads();  // everyone is done reading sW -> reuse it as staging [TM][129]
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) sW[(m0 + i) * 129 + n0 + j] = acc[i][j];
      __syncthreads();
      int64_t cnt = min((int64_t)TM, n - g0);
      for (int64_t e = tid; e < cnt * 127; e += NT) {
        int m = (int)(e / 127), c = (int)(e - (int64_t)m * 127);
        o_feat[g0 * 127 + e] = sFlag[m] ? sW[m * 129 + 1 + c] : 0.f;
      }
      if (half == 0 && gi < n && o_sdf) o_sdf[gi] = sFlag[pm] ? sign * sW[pm * 129] : inactive_sdf;
    } else {
      // only the sdf column is needed: one dot product per point (K=144) by threads 0..127
      if (half == 0) {
        float s = __ldg(wp + OFF_B2);
#pragma unroll 8
        for (int k = 0; k < IN1; ++k) s = fmaf(sAct[k * TM + pm], sW[k * HID], s);
        if (gi < n && o_sdf) o_sdf[gi] = sFlag[pm] ? sign * s : inactive_sdf;
      }
    }
    if (o_lat) {
      int64_t cnt = min((int64_t)TM, n - g0);
      for (int64_t e = tid; e < cnt * LAT; e += NT) {
        int m = (int)(e >> 4), c = (int)(e & 15);
        o_lat[g0 * LAT + e] = sFlag[m] ? sAct[(HID + c) * TM + m] : 0.f;
      }
    }
    if (GRAD) {
      // ---------------- backward: d sdf / d (layer-2 input) = row 0 of W2 --------------
      // sW currently holds W2t [144][128] (or the staging copy if feat was written, so read
      // row 0 of W2 from global instead: W2t[k][0]).
      __syncthreads();
      // delta1[j][m] = W2[0][j] * softplus'(z1) ;  a1 lives in sAct rows 0..127
      for (int e = tid; e < HID * TM; e += NT) {
        int j = e >> 7;
        float w = __ldg(wp + OFF_W2T + j * HID);
        sAct[e] = w * dsoftplus_from_act(sAct[e]);
      }
      backward_from_delta1(sAct, sW, sA0, sPts, sGp, sFlag, wp, vol, D, gi, n, o_grad);
    }
    __syncthreads();  // smem is reused by the next tile
  }
}

__global__ void pack_weights_kernel(const float* w0, const float* b0, const float* w1, const float* b1,
                                    const float* w2, const float* b2, float* pack) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= PACK_FLOATS) return;
  float v;
  if (i < OFF_B0) { int k = i / HID, o = i % HID; v = w0[o * PE + k]; }
  else if (i < OFF_W1T) v = b0[i - OFF_B0];
  else if (i < OFF_B1) { int e = i - OFF_W1T; int k = e / HID, o = e % HID; v = w1[o * IN1 + k]; }
  else if (i < OFF_W2T) v = b1[i - OFF_B1];
  else if (i < OFF_B2) { int e = i - OFF_W2T; int k = e / HID, o = e % HID; v = w2[o * IN1 + k]; }
  else if (i < OFF_W1) v = b2[i - OFF_B2];
  else if (i < OFF_W0) v = w1[i - OFF_W1];
  else { int e = i - OFF_W0; int o = e / W0PAD, k = e % W0PAD; v = k < PE ? w0[o * PE + k] : 0.f; }
  pack[i] = v;
}

}  // namespace
}  // namespace o2345

using namespace o2345;

static_assert(PACK_FLOATS == O2345_SDF_PACK_FLOATS, "header and kernel disagree on the pack size");

extern "C" int o2345_sdf_pack_weights(const float* w0, const float* b0, const float* w1, const float* b1,
                                      const float* w2, const float* b2, float* pack, o2345_stream_t stream) {
  O2345_CHECK_ARG(w0 && b0 && w1 && b1 && w2 && b2 && pack, "null pointer");
  pack_weights_kernel<<<cdiv(PACK_FLOATS, 256), 256, 0, (cudaStream_t)stream>>>(w0, b0, w1, b1, w2, b2, pack);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

namespace o2345 {
int launch_sdf_query_tc(const o2345_points* src, int64_t n, const float* vol_cl, int D, const float* wpack, const uint8_t* active,
                        float inactive_sdf, float sign, float* sdf, float* feat, float* latent, float* grad, cudaStream_t st,
                        const sdfk::VoxelSrc* vx);
}

extern "C" int o2345_sdf_query(const o2345_points* src, int64_t n, const float* vol_cl, int D,
                               const float* wpack, const uint8_t* active, float inactive_sdf, int negate, int precision,
                               float* sdf, float* feat, float* latent, float* grad, o2345_stream_t stream) {
  O2345_CHECK_ARG(n >= 0, "negative point count");
  O2345_CHECK_ARG(precision == O2345_SDF_FP32 || precision == O2345_SDF_TC_SPLIT, "unknown precision");
  if (n == 0) return O2345_OK;
  O2345_CHECK_ARG(src && vol_cl && wpack, "null pointer");
  O2345_CHECK_ARG(D >= 2 && D <= 1024, "volume side out of range");
  if (src->mode == O2345_PTS_EXPLICIT) O2345_CHECK_ARG(src->pts, "explicit points missing");
  else if (src->mode == O2345_PTS_LATTICE) O2345_CHECK_ARG(src->lin && src->R > 0 && n == (int64_t)src->R * src->R * src->R, "bad lattice");
  else if (src->mode == O2345_PTS_RAYS) O2345_CHECK_ARG(src->rays_o && src->rays_d && src->z && src->S > 0 && src->z_stride >= src->S && n % src->S == 0, "bad ray source");
  else O2345_CHECK_ARG(false, "unknown point source mode");
  if (precision == O2345_SDF_TC_SPLIT)
    return launch_sdf_query_tc(src, n, vol_cl, D, wpack, active, inactive_sdf, negate ? -1.f : 1.f, sdf, feat, latent, grad,
                               (cudaStream_t)stream, nullptr);
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_FWD));
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_GRAD));
  }
  int64_t ntiles = (n + TM - 1) / TM;
  int grid = (int)(ntiles < (int64_t)sm_count() ? ntiles : (int64_t)sm_count());
  float sign = negate ? -1.f : 1.f;
  const VoxelSrc vx{};
  if (grad)
    sdf_query_kernel<true, false><<<grid, NT, SMEM_GRAD, (cudaStream_t)stream>>>(*src, n, vol_cl, D, wpack, active, inactive_sdf, sign, sdf, feat, latent, grad, vx);
  else
    sdf_query_kernel<false, false><<<grid, NT, SMEM_FWD, (cudaStream_t)stream>>>(*src, n, vol_cl, D, wpack, active, inactive_sdf, sign, sdf, feat, latent, grad, vx);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_sdf_voxels(const float* occ, const float* vol_cl, int D, const float* origin, float voxel_size,
                                const float* wpack, int precision, float* sdf_vol, o2345_stream_t stream) {
  O2345_CHECK_ARG(occ && vol_cl && origin && wpack && sdf_vol, "null pointer");
  O2345_CHECK_ARG(D >= 2 && D <= 1024, "volume side out of range");
  O2345_CHECK_ARG(precision == O2345_SDF_FP32 || precision == O2345_SDF_TC_SPLIT, "unknown precision");
  const int64_t n = (int64_t)D * D * D;
  const VoxelSrc vx{occ, origin, voxel_size};
  const o2345_points none{};
  if (precision == O2345_SDF_TC_SPLIT)
    return launch_sdf_query_tc(&none, n, vol_cl, D, wpack, nullptr, 1.f, 1.f, sdf_vol, nullptr, nullptr, nullptr,
                               (cudaStream_t)stream, &vx);
  static PerDeviceOnce attr_done;
  if (attr_done.need())
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_FWD));
  int64_t ntiles = (n + TM - 1) / TM;
  int grid = (int)(ntiles < (int64_t)sm_count() ? ntiles : (int64_t)sm_count());
  sdf_query_kernel<false, true><<<grid, NT, SMEM_FWD, (cudaStream_t)stream>>>(none, n, vol_cl, D, wpack, nullptr, 1.f, 1.f, sdf_vol,
                                                                              nullptr, nullptr, nullptr, vx);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
