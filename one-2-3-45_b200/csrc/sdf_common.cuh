// Shared pieces of the two SDF query kernels (sdf_mlp.cu: fp32 FMA; sdf_mlp_tc.cu: forward layers on tensor cores):
// tile sizes, the packed-weight layout, softplus(beta = 100) and its derivative, the reference's quirky trilinear setup
// (ops/grid_sampler.py:79-90), point sources and the register-tiled shared-memory GEMMs.
#pragma once
#include "common.cuh"

namespace o2345 {
namespace sdfk {

constexpr int TM = 128;   // points per tile
constexpr int NT = 256;   // threads per CTA
constexpr int PE = O2345_SDF_PE, HID = O2345_SDF_HID, LAT = O2345_SDF_LAT, IN1 = O2345_SDF_IN1;
constexpr int W0PAD = 48;  // W0 rows padded to 48 columns for the backward GEMM

constexpr int OFF_W0T = 0;
constexpr int OFF_B0 = OFF_W0T + PE * HID;
constexpr int OFF_W1T = OFF_B0 + HID;
constexpr int OFF_B1 = OFF_W1T + IN1 * HID;
constexpr int OFF_W2T = OFF_B1 + HID;
constexpr int OFF_B2 = OFF_W2T + IN1 * HID;
constexpr int OFF_W1 = OFF_B2 + HID;          // [128][144]
constexpr int OFF_W0 = OFF_W1 + HID * IN1;    // [128][48]
constexpr int PACK_FLOATS = OFF_W0 + HID * W0PAD;

constexpr int SM_ACT = IN1 * TM;              // 18432 floats
constexpr int SM_W = IN1 * HID;               // 18432 floats (also output staging [TM][129])
constexpr int SM_A0 = HID * TM;               // 16384 floats (grad only)
constexpr int SM_MISC = 8 * TM;               // pts(3) + grad partials(3) + flags
constexpr int SMEM_FWD = (SM_ACT + SM_W + SM_MISC) * 4;
constexpr int SMEM_GRAD = (SM_ACT + SM_W + SM_A0 + SM_MISC) * 4;

__device__ __forceinline__ float softplus100(float x) {
  float bx = 100.f * x;
  return bx > 20.f ? x : log1pf(expf(bx)) * 0.01f;
}
// d softplus / dx expressed through the activation a = softplus(x): sigmoid(100x) = 1 - exp(-100a)
__device__ __forceinline__ float dsoftplus_from_act(float a) { return -expm1f(-100.f * a); }

// MUFU versions for the tensor-core kernel (ex2 / lg2 approximations: absolute error < 2e-7 on activations of O(1),
// below that kernel's 2e-6 agreement with the fp32 one; the precise log1pf / expf / expm1f cost ~80 instructions each)
__device__ __forceinline__ float softplus100_fast(float x) {
  const float bx = 100.f * x;
  float e, l;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(bx * 1.4426950408889634f));
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.f + e));
  return bx > 20.f ? x : l * (0.6931471805599453f * 0.01f);
}
__device__ __forceinline__ float dsoftplus_from_act_fast(float a) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-144.26950408889634f * a));
  return 1.f - e;
}

struct Tri {
  int base[3];     // clamped floor index per axis (x,y,z)
  int hi[3];       // clamped floor+1 index
  float w0[3], w1[3];
  bool inb;
};

// reference ops/grid_sampler.py:79-90 (after the xyz->zyx flip of sparse_sdf_network.py:408)
__device__ __forceinline__ Tri tri_setup(float px, float py, float pz, int D) {
  Tri t;
  float p[3] = {px, py, pz};
  bool inb = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float tt = __fmul_rn(__fdiv_rn(__fadd_rn(p[a], 1.f), 2.f), (float)(D - 1));
    inb = inb && (tt > 0.f) && (tt < (float)D);
    float f = floorf(tt);
    t.w1[a] = tt - f;
    t.w0[a] = (f + 1.f) - tt;
    // clamp in float first: tt may be huge or NaN for far-away points
    float fl = fminf(fmaxf(f, 0.f), (float)(D - 1));
    float fh = fminf(fmaxf(f + 1.f, 0.f), (float)(D - 1));
    t.base[a] = (int)fl;
    t.hi[a] = (int)fh;
  }
  t.inb = inb;
  return t;
}

// Point and latent source of o2345_sdf_voxels (kernels instantiated with VOX = true): point i is lattice voxel
// i = (x*D + y)*D + z at coord * vs + origin (one rounded multiply, one rounded add, as `coords * voxel_size + origin`
// in fp32), its latent is row i of the channel-last volume as it is (no trilinear fetch), and it is evaluated iff
// occ[i] > 0 (reference SparseSdfNetwork.get_sdf_volume, sparse_sdf_network.py:441-474).
struct VoxelSrc {
  const float* occ;
  const float* origin;
  float vs;
};

__device__ __forceinline__ void voxel_point(const VoxelSrc& vx, int64_t gi, int D, float& x, float& y, float& z) {
  const int iz = (int)(gi % D), iy = (int)((gi / D) % D), ix = (int)(gi / ((int64_t)D * D));
  x = __fadd_rn(__fmul_rn((float)ix, vx.vs), __ldg(vx.origin));
  y = __fadd_rn(__fmul_rn((float)iy, vx.vs), __ldg(vx.origin + 1));
  z = __fadd_rn(__fmul_rn((float)iz, vx.vs), __ldg(vx.origin + 2));
}

// acc[i][j] += sum_k A[k][m0+i] * B[k][n0+j];  A k-major with row stride TM, B row stride 128.
template <int K>
__device__ __forceinline__ void gemm_fwd(const float* __restrict__ sA, const float* __restrict__ sB,
                                         float (&acc)[8][8], int m0, int n0) {
#pragma unroll 2
  for (int k = 0; k < K; ++k) {
    float4 a0 = *reinterpret_cast<const float4*>(sA + k * TM + m0);
    float4 a1 = *reinterpret_cast<const float4*>(sA + k * TM + m0 + 4);
    float4 b0 = *reinterpret_cast<const float4*>(sB + k * HID + n0);
    float4 b1 = *reinterpret_cast<const float4*>(sB + k * HID + n0 + 4);
    float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

// acc[i][j] += sum_{k<128} A[k][m0+i] * B[k][ty + 16 j];  B row stride LDB, NJ columns per thread.
template <int NJ, int LDB>
__device__ __forceinline__ void gemm_bwd(const float* __restrict__ sA, const float* __restrict__ sB,
                                         float (&acc)[8][NJ], int m0, int ty) {
#pragma unroll 2
  for (int k = 0; k < HID; ++k) {
    float4 a0 = *reinterpret_cast<const float4*>(sA + k * TM + m0);
    float4 a1 = *reinterpret_cast<const float4*>(sA + k * TM + m0 + 4);
    float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    float b[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) b[j] = sB[k * LDB + ty + 16 * j];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

__device__ __forceinline__ void load_weights(float* sW, const float* __restrict__ g, int nfloats) {
#pragma unroll 6   // several independent L2 loads in flight
  for (int i = threadIdx.x * 4; i < nfloats; i += NT * 4)
    *reinterpret_cast<float4*>(sW + i) = ldg4(g + i);
}

// Last step of the reverse pass, per point: contraction of d sdf / d PE (sGpe [48][TM]) with d PE / d xyz (threads
// 0..127) and of d sdf / d latent (sGlat [16][TM]) with the derivative of the trilinear weights (threads 128..255).
__device__ __forceinline__ void backward_point_tail(const float* sGpe, const float* sGlat, const float* sPts, float* sGp,
                                                    const int* sFlag, const float* __restrict__ vol, int D, int64_t gi,
                                                    int64_t n, float* __restrict__ o_grad) {
  const int tid = threadIdx.x;
  const int pm = tid & (TM - 1), half = tid >> 7;
  // ---------------- per point: embedding part (half 0) + trilinear part (half 1) ---
  {
    float qx = sPts[pm], qy = sPts[TM + pm], qz = sPts[2 * TM + pm];
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (half == 0) {
      float p[3] = {qx, qy, qz};
      float gg[3] = {sGpe[0 * TM + pm], sGpe[1 * TM + pm], sGpe[2 * TM + pm]};
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        float fr = (float)(1 << k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          float s, c;
          sincosf(fr * p[a], &s, &c);
          float gs = sGpe[(3 + 6 * k + a) * TM + pm], gc = sGpe[(3 + 6 * k + 3 + a) * TM + pm];
          gg[a] = fmaf(fr, gs * c - gc * s, gg[a]);
        }
      }
      gx = gg[0], gy = gg[1], gz = gg[2];
    } else {
      Tri t = tri_setup(qx, qy, qz, D);
      if (t.inb) {
        float gl[LAT];
#pragma unroll
        for (int c = 0; c < LAT; ++c) gl[c] = sGlat[c * TM + pm];
        float sc = 0.5f * (float)(D - 1);  // d t / d p
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
          int dx = corner >> 2, dy = (corner >> 1) & 1, dz = corner & 1;
          int ix = dx ? t.hi[0] : t.base[0], iy = dy ? t.hi[1] : t.base[1], iz = dz ? t.hi[2] : t.base[2];
          const float* v = vol + (((int64_t)ix * D + iy) * D + iz) * LAT;
          float dot = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < 4; ++c4) {
            float4 vv = ldg4(v + 4 * c4);
            dot = fmaf(vv.x, gl[4 * c4], dot); dot = fmaf(vv.y, gl[4 * c4 + 1], dot);
            dot = fmaf(vv.z, gl[4 * c4 + 2], dot); dot = fmaf(vv.w, gl[4 * c4 + 3], dot);
          }
          float wx = dx ? t.w1[0] : t.w0[0], wy = dy ? t.w1[1] : t.w0[1], wz = dz ? t.w1[2] : t.w0[2];
          float sx = dx ? sc : -sc, sy = dy ? sc : -sc, sz = dz ? sc : -sc;
          gx = fmaf(dot, sx * wy * wz, gx);
          gy = fmaf(dot, wx * sy * wz, gy);
          gz = fmaf(dot, wx * wy * sz, gz);
        }
      }
      sGp[pm] = gx, sGp[TM + pm] = gy, sGp[2 * TM + pm] = gz;
    }
    __syncthreads();
    if (half == 0 && gi < n && o_grad) {
      bool on = sFlag[pm] != 0;
      o_grad[3 * gi] = on ? gx + sGp[pm] : 0.f;
      o_grad[3 * gi + 1] = on ? gy + sGp[TM + pm] : 0.f;
      o_grad[3 * gi + 2] = on ? gz + sGp[2 * TM + pm] : 0.f;
    }
  }
}

// Reverse pass from delta1 = d sdf / d z1 (fp32, sAct rows 0..127, k-major [feature][point]) to d sdf / d xyz:
// two transposed GEMMs (W1, W0), the softplus derivative of layer 0 (activations in sA0), then per point the embedding
// and trilinear contractions.  Shared by both SDF kernels; every thread of the CTA must call it.
template <bool FAST = false>
__device__ __forceinline__ void backward_from_delta1(float* sAct, float* sW, float* sA0, const float* sPts, float* sGp,
                                                     const int* sFlag, const float* __restrict__ wp,
                                                     const float* __restrict__ vol, int D, int64_t gi, int64_t n,
                                                     float* __restrict__ o_grad) {
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = tx * 8;
  load_weights(sW, wp + OFF_W1, HID * IN1);
  __syncthreads();
  {
    float g[8][9];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 9; ++j) g[i][j] = 0.f;
    gemm_bwd<9, IN1>(sAct, sW, g, m0, ty);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      int nn = ty + 16 * j;
      float v[8];
      if (j < 8) {  // delta0 = g * softplus'(z0)
        float4 a0 = *reinterpret_cast<const float4*>(sA0 + nn * TM + m0);
        float4 a1 = *reinterpret_cast<const float4*>(sA0 + nn * TM + m0 + 4);
        float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = g[i][j] * (FAST ? dsoftplus_from_act_fast(a[i]) : dsoftplus_from_act(a[i]));
      } else {      // gradient w.r.t. the latent: direct path through layer 2 + layer 1
        float w = __ldg(wp + OFF_W2T + nn * HID);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = g[i][j] + w;
      }
      *reinterpret_cast<float4*>(sAct + nn * TM + m0) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(sAct + nn * TM + m0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
  load_weights(sW, wp + OFF_W0, HID * W0PAD);
  __syncthreads();
  {
    float g[8][3];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) g[i][j] = 0.f;
    gemm_bwd<3, W0PAD>(sAct, sW, g, m0, ty);
    // sA0 is free now (delta0 already formed): g_pe[n][m] -> sA0 rows 0..47
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      int nn = ty + 16 * j;
      *reinterpret_cast<float4*>(sA0 + nn * TM + m0) = make_float4(g[0][j], g[1][j], g[2][j], g[3][j]);
      *reinterpret_cast<float4*>(sA0 + nn * TM + m0 + 4) = make_float4(g[4][j], g[5][j], g[6][j], g[7][j]);
    }
  }
  __syncthreads();
  backward_point_tail(sA0, sAct + HID * TM, sPts, sGp, sFlag, vol, D, gi, n, o_grad);
}

}  // namespace sdfk
}  // namespace o2345
