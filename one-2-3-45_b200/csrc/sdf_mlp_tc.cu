// SDF query with the forward layers on tensor cores at fp32-grade accuracy (rows B8/B9/B10 of SURVEY.md section 8).
//
// Same function, tiling and outputs as sdf_query_kernel (sdf_mlp.cu); the three forward GEMMs (39 -> 128 -> 128 -> 128
// over [PE | latent] inputs) run as mma.sync.m16n8k16 with SPLIT operands: every activation and weight x is stored as
// two fp16 numbers hi = fp16(x), lo = fp16(x - hi), and a product a.w is accumulated in fp32 as
// a_hi w_hi + a_hi w_lo + a_lo w_hi.  Each fp16 x fp16 product is exact in the fp32 accumulator and the dropped
// a_lo w_lo term is 2^-22 relative, so the SDF values agree with the fp32 FMA kernel to ~1e-6 -- the NeuS alpha
// (inv_s * sdf) and marching cubes need that; plain fp16 / bf16 operands (1e-3) would not do.
//
//   smem   activations as two half planes [k][136] (k-major: a layer's output rows are the next layer's k rows),
//          the current layer's weights as two half planes [k][136]; fragments come from ldmatrix.trans, layer outputs
//          go back with stmatrix.trans; 136-half rows make every ldmatrix / stmatrix phase conflict free;
//   warps  4 (m) x 2 (n): a warp owns 32 points x 64 outputs = 2 x 8 accumulator tiles;
//   rest   stage 0 (trilinear latent fetch, positional embedding), the sdf-only dot product, output staging and the
//          per-point tail of the reverse pass are the code of the fp32 kernel; the two transposed GEMMs of the
//          reverse pass use the same split-fp16 MMAs with one 16-point m-tile per warp.
#include <cuda_fp16.h>

#include "common.cuh"
#include "mma_sync.cuh"
#include "sdf_common.cuh"

namespace o2345 {
namespace {
using namespace sdfk;

constexpr int LDP = TM + 8;                    // halves per plane row
constexpr int PLANE = IN1 * LDP;               // halves per plane (144 rows)
constexpr int REGION = 2 * PLANE * 2;          // bytes of a hi + lo plane pair = 78 336 >= 73 728 (an fp32 [144][128] block)
static_assert(REGION >= TM * 129 * 4, "the fp32 output staging must fit in the weight region");
constexpr int SMEM_TC_FWD = 2 * REGION + SM_MISC * 4;
constexpr int SMEM_TC_GRAD = 2 * REGION + SM_A0 * 4 + SM_MISC * 4;
constexpr int K0PAD = 48;                      // layer-0 K (39) padded to three k-blocks

__device__ __forceinline__ void split(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
__device__ __forceinline__ void ldsm4t(uint32_t (&r)[4], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void stsm4t(__half* p, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  __half2 h = __halves2half2(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// weights of one layer: fp32 [K][128] (k-major, as packed) -> hi / lo planes [KP][LDP]; rows K..KP-1 are zero
__device__ __forceinline__ void load_weight_planes(__half* sWh, __half* sWl, const float* __restrict__ g, int K, int KP) {
#pragma unroll 6   // several independent L2 loads in flight (18 trips for a 144-row layer)
  for (int i = threadIdx.x * 4; i < KP * HID; i += NT * 4) {
    const int k = i >> 7, c = i & 127;
    float4 v = k < K ? ldg4(g + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    __half h[4], l[4];
    split(v.x, h[0], l[0]), split(v.y, h[1], l[1]), split(v.z, h[2], l[2]), split(v.w, h[3], l[3]);
    *reinterpret_cast<uint2*>(sWh + k * LDP + c) = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
    *reinterpret_cast<uint2*>(sWl + k * LDP + c) = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
  }
}

// acc[2 m-tiles][8 n-tiles] += A[32 points x 16 KB] . W[16 KB x 64], split-fp16 (three MMAs per product)
template <int KB>
__device__ __forceinline__ void gemm_split(float (&acc)[2][8][4], const __half* sAh, const __half* sAl, const __half* sWh,
                                           const __half* sWl, int mw, int nw, int lane) {
  // ldmatrix.trans lane -> row / column offsets inside a 16 x 16 block of a k-major plane
  const int a_row = (lane & 7) + ((lane >> 4) & 1) * 8, a_col = ((lane >> 3) & 1) * 8;   // A: matrices (k lo, m lo), (k lo, m hi), (k hi, m lo), (k hi, m hi)
  const int b_row = (lane & 7) + ((lane >> 3) & 1) * 8, b_col = ((lane >> 4) & 1) * 8;   // B: (k lo, n lo), (k hi, n lo), (k lo, n hi), (k hi, n hi)
#pragma unroll 1
  for (int kb = 0; kb < KB; ++kb) {
    uint32_t ah[2][4], al[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int off = (16 * kb + a_row) * LDP + mw + 16 * mt + a_col;
      ldsm4t(ah[mt], sAh + off);
      ldsm4t(al[mt], sAl + off);
    }
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t bh[4], bl[4];
      const int off = (16 * kb + b_row) * LDP + nw + 16 * np + b_col;
      ldsm4t(bh, sWh + off);
      ldsm4t(bl, sWl + off);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma16816(acc[mt][2 * np], al[mt], bh[0], bh[1]);
        mma16816(acc[mt][2 * np], ah[mt], bl[0], bl[1]);
        mma16816(acc[mt][2 * np], ah[mt], bh[0], bh[1]);
        mma16816(acc[mt][2 * np + 1], al[mt], bh[2], bh[3]);
        mma16816(acc[mt][2 * np + 1], ah[mt], bl[2], bl[3]);
        mma16816(acc[mt][2 * np + 1], ah[mt], bh[2], bh[3]);
      }
    }
  }
}

// reverse-pass weights: fp32 [K][ncols] rows of length src_ld (k-major: W1 as [j][i], W0 as [n][i]) -> planes [K][LD]
__device__ __forceinline__ void load_planes_generic(__half* sWh, __half* sWl, const float* __restrict__ g, int K, int ncols, int src_ld,
                                                    int LD) {
  const int c4n = ncols >> 2;
#pragma unroll 4
  for (int i = threadIdx.x; i < K * c4n; i += NT) {
    const int k = i / c4n, c = (i - k * c4n) * 4;
    float4 v = ldg4(g + k * src_ld + c);
    __half h[4], l[4];
    split(v.x, h[0], l[0]), split(v.y, h[1], l[1]), split(v.z, h[2], l[2]), split(v.w, h[3], l[3]);
    *reinterpret_cast<uint2*>(sWh + k * LD + c) = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
    *reinterpret_cast<uint2*>(sWl + k * LD + c) = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
  }
}

// acc[NP pairs of n-tiles] += A[16 points (columns m0..m0+15 of the planes) x 128] . W[128 x 16 NP], split-fp16.
// One m-tile per warp: a warp reads and (in the callers) rewrites only ITS 16 point columns of the activation planes,
// so the reverse pass needs no CTA barrier around its in-place updates.
template <int NP>
__device__ __forceinline__ void gemm_split_rows(float (&acc)[2 * NP][4], const __half* sAh, const __half* sAl, const __half* sWh,
                                                const __half* sWl, int LDW, int m0, int lane) {
  const int a_row = (lane & 7) + ((lane >> 4) & 1) * 8, a_col = ((lane >> 3) & 1) * 8;
  const int b_row = (lane & 7) + ((lane >> 3) & 1) * 8, b_col = ((lane >> 4) & 1) * 8;
#pragma unroll 1
  for (int kb = 0; kb < HID / 16; ++kb) {
    uint32_t ah[4], al[4];
    const int offa = (16 * kb + a_row) * LDP + m0 + a_col;
    ldsm4t(ah, sAh + offa);
    ldsm4t(al, sAl + offa);
#pragma unroll
    for (int np = 0; np < NP; ++np) {
      uint32_t bh[4], bl[4];
      const int off = (16 * kb + b_row) * LDW + 16 * np + b_col;
      ldsm4t(bh, sWh + off);
      ldsm4t(bl, sWl + off);
      mma16816(acc[2 * np], al, bh[0], bh[1]);
      mma16816(acc[2 * np], ah, bl[0], bl[1]);
      mma16816(acc[2 * np], ah, bh[0], bh[1]);
      mma16816(acc[2 * np + 1], al, bh[2], bh[3]);
      mma16816(acc[2 * np + 1], ah, bl[2], bl[3]);
      mma16816(acc[2 * np + 1], ah, bh[2], bh[3]);
    }
  }
}

__device__ __forceinline__ void init_bias(float (&acc)[2][8][4], const float* __restrict__ b, int nw, int t) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float b0 = __ldg(b + nw + 8 * j + 2 * t), b1 = __ldg(b + nw + 8 * j + 2 * t + 1);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) acc[mt][j][0] = acc[mt][j][2] = b0, acc[mt][j][1] = acc[mt][j][3] = b1;
  }
}

// softplus on the accumulators, then back into the activation planes as rows n (= k of the next layer), columns m;
// sA0 != nullptr: also keep the fp32 activations [n][m] for the reverse pass
__device__ __forceinline__ void store_activations(float (&acc)[2][8][4], __half* sAh, __half* sAl, float* sA0, int mw, int nw,
                                                  int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {           // q = 2 * (n-tile of the pair) + (row half): blocks (m lo, n0), (m hi, n0), (m lo, n1), (m hi, n1)
        const int j = 2 * np + (q >> 1), r = q & 1;
        const float v0 = softplus100_fast(acc[mt][j][2 * r]), v1 = softplus100_fast(acc[mt][j][2 * r + 1]);
        if (sA0) {
          const int m = mw + 16 * mt + 8 * r + g, nn = nw + 8 * j + 2 * t;
          sA0[nn * TM + m] = v0, sA0[(nn + 1) * TM + m] = v1;
        }
        __half h0, l0, h1, l1;
        split(v0, h0, l0), split(v1, h1, l1);
        hi[q] = pack_h2(h0, h1), lo[q] = pack_h2(l0, l1);
      }
      // stmatrix.trans: lane l supplies the address of row (l & 7) of matrix (l >> 3); matrix q is the 8 x 8 block
      // (points mw + 16 mt + 8 (q & 1) .., outputs nw + 16 np + 8 (q >> 1) ..) stored as rows = outputs, columns = points
      const int q = lane >> 3;
      const int off = (nw + 16 * np + 8 * (q >> 1) + (lane & 7)) * LDP + mw + 16 * mt + 8 * (q & 1);
      stsm4t(sAh + off, hi[0], hi[1], hi[2], hi[3]);
      stsm4t(sAl + off, lo[0], lo[1], lo[2], lo[3]);
    }
}

// VOX: the points and latents come from VoxelSrc (o2345_sdf_voxels) instead of `src` + the trilinear fetch.
template <bool GRAD, bool VOX>
__global__ void __launch_bounds__(NT, 1)
sdf_query_tc_kernel(o2345_points src, int64_t n, const float* __restrict__ vol, int D, const float* __restrict__ wp,
                    const uint8_t* __restrict__ active, float inactive_sdf, float sign, float* __restrict__ o_sdf,
                    float* __restrict__ o_feat, float* __restrict__ o_lat, float* __restrict__ o_grad, VoxelSrc vx) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sAh = reinterpret_cast<__half*>(smem_raw);
  __half* sAl = sAh + PLANE;
  __half* sWh = reinterpret_cast<__half*>(smem_raw + REGION);
  __half* sWl = sWh + PLANE;
  float* sW = reinterpret_cast<float*>(smem_raw + REGION);     // fp32 view of the weight region (staging / reverse pass)
  float* sA0 = reinterpret_cast<float*>(smem_raw + 2 * REGION);
  float* sMisc = GRAD ? sA0 + SM_A0 : sA0;
  float* sPts = sMisc;
  float* sGp = sMisc + 3 * TM;
  int* sFlag = reinterpret_cast<int*>(sMisc + 6 * TM);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mw = (warp & 3) * 32, nw = (warp >> 2) * 64;
  const int pm = tid & (TM - 1), half = tid >> 7;
  const int64_t ntiles = (n + TM - 1) / TM;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t g0 = tile * TM;
    const int64_t gi = g0 + pm;
    // ---------------- stage 0: point, latent, embedding (as sdf_query_kernel, written as hi / lo halves) -----------
    bool act = gi < n && (VOX ? __ldg(vx.occ + gi) > 0.f : (active == nullptr || active[gi] != 0));
    int any = __syncthreads_or(act ? 1 : 0);
    if (!any) {
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
    auto put = [&](int k, float v) {
      __half h, l;
      split(v, h, l);
      sAh[k * LDP + pm] = h, sAl[k * LDP + pm] = l;
    };
    {
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
      for (int c = 0; c < 8; ++c) put(HID + 8 * half + c, lat[c]);
      if (o_lat && gi < n) {   // the latent is an output in full fp32 precision: written from registers
#pragma unroll
        for (int c = 0; c < 8; ++c) o_lat[gi * LAT + 8 * half + c] = act ? lat[c] : 0.f;
      }
      float p[3] = {px, py, pz};
      if (half == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) put(a, p[a]);
      } else {
        for (int k = PE; k < K0PAD; ++k) put(k, 0.f);   // zero rows of the padded layer-0 K range
      }
#pragma unroll
      for (int f = 0; f < 3; ++f) {
        int k = 3 * half + f;
        float fr = (float)(1 << k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          float s, c;
          sincosf(fr * p[a], &s, &c);
          put(3 + 6 * k + a, s);
          put(3 + 6 * k + 3 + a, c);
        }
      }
    }
    load_weight_planes(sWh, sWl, wp + OFF_W0T, PE, K0PAD);
    __syncthreads();

    float acc[2][8][4];
    // ---------------- layer 0: 39 -> 128, softplus ---------------------------------------------------------------
    init_bias(acc, wp + OFF_B0, nw, lane & 3);
    gemm_split<K0PAD / 16>(acc, sAh, sAl, sWh, sWl, mw, nw, lane);
    __syncthreads();
    store_activations(acc, sAh, sAl, GRAD ? sA0 : nullptr, mw, nw, lane);
    load_weight_planes(sWh, sWl, wp + OFF_W1T, IN1, IN1);
    __syncthreads();
    // ---------------- layer 1: 144 -> 128, softplus --------------------------------------------------------------
    init_bias(acc, wp + OFF_B1, nw, lane & 3);
    gemm_split<IN1 / 16>(acc, sAh, sAl, sWh, sWl, mw, nw, lane);
    __syncthreads();
    store_activations(acc, sAh, sAl, nullptr, mw, nw, lane);
    const bool need_feat = (o_feat != nullptr);
    if (need_feat) load_weight_planes(sWh, sWl, wp + OFF_W2T, IN1, IN1);
    __syncthreads();
    // ---------------- layer 2: 144 -> 128 (no activation) --------------------------------------------------------
    if (need_feat) {
      init_bias(acc, wp + OFF_B2, nw, lane & 3);
      gemm_split<IN1 / 16>(acc, sAh, sAl, sWh, sWl, mw, nw, lane);
      __syncthreads();  // everyone is done reading the weight planes -> reuse the region as fp32 staging [TM][129]
      {
        const int g = lane >> 2, t = lane & 3;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int m = mw + 16 * mt + 8 * r + g, nn = nw + 8 * j + 2 * t;
              sW[m * 129 + nn] = acc[mt][j][2 * r], sW[m * 129 + nn + 1] = acc[mt][j][2 * r + 1];
            }
      }
      __syncthreads();
      int64_t cnt = min((int64_t)TM, n - g0);
      for (int64_t e = tid; e < cnt * 127; e += NT) {
        int m = (int)(e / 127), c = (int)(e - (int64_t)m * 127);
        o_feat[g0 * 127 + e] = sFlag[m] ? sW[m * 129 + 1 + c] : 0.f;
      }
      if (half == 0 && gi < n && o_sdf) o_sdf[gi] = sFlag[pm] ? sign * sW[pm * 129] : inactive_sdf;
    } else if (half == 0) {
      // only the sdf column is needed: one fp32 dot product per point over [a1 | latent] (hi + lo) and column 0 of W2^T
      float s = __ldg(wp + OFF_B2);
#pragma unroll 8
      for (int k = 0; k < IN1; ++k)
        s = fmaf(__half2float(sAh[k * LDP + pm]) + __half2float(sAl[k * LDP + pm]), __ldg(wp + OFF_W2T + k * HID), s);
      if (gi < n && o_sdf) o_sdf[gi] = sFlag[pm] ? sign * s : inactive_sdf;
    }
    if (GRAD) {
      // ---------------- reverse pass on the tensor cores ----------------------------------------------------------
      // warp w owns points 16 w .. 16 w + 15 (ONE m-tile) for both transposed GEMMs: it transforms, reads and rewrites
      // only its own 16 columns of the activation planes / sA0, so only the weight planes need CTA barriers.
      constexpr int LDW1 = IN1 + 8, LDW0 = W0PAD + 8;          // 152 / 56 halves: conflict-free ldmatrix rows
      static_assert(HID * LDW1 <= PLANE, "W1 planes must fit in the weight region");
      const int m0w = 16 * warp, g = lane >> 2, t = lane & 3;
      __syncthreads();                                          // layer-1 planes complete, sdf dot products done
      load_planes_generic(sWh, sWl, wp + OFF_W1, HID, IN1, IN1, LDW1);
      // delta1[j][m] = W2[0][j] * softplus'(z1[j][m]) in place over a1 (own columns): lane -> (row j, 2 columns)
      for (int e = lane; e < HID * 8; e += 32) {
        const int j = e >> 3, c = m0w + 2 * (e & 7);
        const float w = __ldg(wp + OFF_W2T + j * HID);
        __half2 h = *reinterpret_cast<__half2*>(sAh + j * LDP + c), l = *reinterpret_cast<__half2*>(sAl + j * LDP + c);
        const float d0 = w * dsoftplus_from_act_fast(__low2float(h) + __low2float(l));
        const float d1 = w * dsoftplus_from_act_fast(__high2float(h) + __high2float(l));
        __half h0, l0, h1, l1;
        split(d0, h0, l0), split(d1, h1, l1);
        *reinterpret_cast<__half2*>(sAh + j * LDP + c) = __halves2half2(h0, h1);
        *reinterpret_cast<__half2*>(sAl + j * LDP + c) = __halves2half2(l0, l1);
      }
      __syncthreads();                                          // W1 planes complete (and this warp's delta1 visible)
      {
        // g[m][i] = sum_j delta1[j][m] W1[j][i], i = 0..143 (9 pairs of n-tiles)
        float acc1[18][4];
#pragma unroll
        for (int j = 0; j < 18; ++j) acc1[j][0] = acc1[j][1] = acc1[j][2] = acc1[j][3] = 0.f;
        gemm_split_rows<9>(acc1, sAh, sAl, sWh, sWl, LDW1, m0w, lane);
        __syncwarp();
        // i < 128: delta0 = g * softplus'(z0) back into the planes (rows i, own columns) through stmatrix.trans
#pragma unroll
        for (int np = 0; np < 8; ++np) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int j = 2 * np + (q >> 1), r = q & 1;
            const int m = m0w + 8 * r + g, nn = 8 * j + 2 * t;
            const float v0 = acc1[j][2 * r] * dsoftplus_from_act_fast(sA0[nn * TM + m]);
            const float v1 = acc1[j][2 * r + 1] * dsoftplus_from_act_fast(sA0[(nn + 1) * TM + m]);
            __half h0, l0, h1, l1;
            split(v0, h0, l0), split(v1, h1, l1);
            hi[q] = pack_h2(h0, h1), lo[q] = pack_h2(l0, l1);
          }
          const int q = lane >> 3;
          const int off = (16 * np + 8 * (q >> 1) + (lane & 7)) * LDP + m0w + 8 * (q & 1);
          stsm4t(sAh + off, hi[0], hi[1], hi[2], hi[3]);
          stsm4t(sAl + off, lo[0], lo[1], lo[2], lo[3]);
        }
        __syncwarp();   // every lane has read sA0 (layer-0 activations of the own columns): rows 48..63 may be reused
        // i = 128..143: gradient w.r.t. the latent = g + direct path through layer 2 -> sA0 rows 48..63 (fp32)
#pragma unroll
        for (int j = 16; j < 18; ++j)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int m = m0w + 8 * r + g, c = 8 * (j - 16) + 2 * t;
            sA0[(48 + c) * TM + m] = acc1[j][2 * r] + __ldg(wp + OFF_W2T + (HID + c) * HID);
            sA0[(48 + c + 1) * TM + m] = acc1[j][2 * r + 1] + __ldg(wp + OFF_W2T + (HID + c + 1) * HID);
          }
      }
      __syncthreads();                                          // every warp is done with the W1 planes
      load_planes_generic(sWh, sWl, wp + OFF_W0, HID, W0PAD, W0PAD, LDW0);
      __syncthreads();
      {
        // g_pe[m][i] = sum_n delta0[n][m] W0[n][i], i = 0..47 -> sA0 rows 0..47 (own columns)
        float acc0[6][4];
#pragma unroll
        for (int j = 0; j < 6; ++j) acc0[j][0] = acc0[j][1] = acc0[j][2] = acc0[j][3] = 0.f;
        gemm_split_rows<3>(acc0, sAh, sAl, sWh, sWl, LDW0, m0w, lane);
#pragma unroll
        for (int j = 0; j < 6; ++j)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int m = m0w + 8 * r + g, nn = 8 * j + 2 * t;
            sA0[nn * TM + m] = acc0[j][2 * r], sA0[(nn + 1) * TM + m] = acc0[j][2 * r + 1];
          }
      }
      __syncthreads();
      backward_point_tail(sA0, sA0 + 48 * TM, sPts, sGp, sFlag, vol, D, gi, n, o_grad);
    }
    __syncthreads();  // smem is reused by the next tile
  }
}

}  // namespace

// vx != nullptr: o2345_sdf_voxels (forward only; points and latents from *vx, `src` and `active` unused)
int launch_sdf_query_tc(const o2345_points* src, int64_t n, const float* vol_cl, int D, const float* wpack, const uint8_t* active,
                        float inactive_sdf, float sign, float* sdf, float* feat, float* latent, float* grad, cudaStream_t st,
                        const VoxelSrc* vx) {
  static PerDeviceOnce attr_done;
  if (attr_done.need()) {
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_tc_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TC_FWD));
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_tc_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TC_GRAD));
    O2345_CUDA(cudaFuncSetAttribute(sdf_query_tc_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TC_FWD));
  }
  int64_t tiles = (n + TM - 1) / TM;
  int grid = (int)(tiles < (int64_t)sm_count() ? tiles : (int64_t)sm_count());
  if (vx)
    sdf_query_tc_kernel<false, true><<<grid, NT, SMEM_TC_FWD, st>>>(*src, n, vol_cl, D, wpack, nullptr, inactive_sdf, sign, sdf, feat,
                                                                    latent, nullptr, *vx);
  else if (grad)
    sdf_query_tc_kernel<true, false><<<grid, NT, SMEM_TC_GRAD, st>>>(*src, n, vol_cl, D, wpack, active, inactive_sdf, sign, sdf, feat,
                                                                     latent, grad, VoxelSrc{});
  else
    sdf_query_tc_kernel<false, false><<<grid, NT, SMEM_TC_FWD, st>>>(*src, n, vol_cl, D, wpack, active, inactive_sdf, sign, sdf, feat,
                                                                     latent, grad, VoxelSrc{});
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

}  // namespace o2345
