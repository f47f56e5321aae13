// Path A glue kernels around the wgmma GEMM: everything in the Zero123 UNet / VAE that is not a matrix
// product.  Activations are channel-last fp16 ([B, H*W, C]); normalisation statistics, softmax and the
// DDIM update are computed in fp32, matching the reference's autocast policy (GroupNorm32 / LayerNorm /
// softmax in fp32: ldm/modules/diffusionmodules/util.py:214-216, SURVEY.md section 8 header).
//
//   groupnorm_stats      per (image, group) statistics -> per (image, channel) scale / shift   openaimodel.py:256-276 (GroupNorm32)
//   norm_act_im2col      GroupNorm apply (+SiLU) fused with the 3x3 / 1x1 patch gather (optionally behind a
//                        nearest x2 up-sampling or with stride 2) -> the K-major A operand of the conv GEMM
//   layernorm_rows       attention.py:214-218
//   softmax_rows         attention.py:189 (fp16 scores in, fp32 math, fp16 probabilities out)
//   geglu                attention.py:37-45
//   transpose_tokens     [B,N,C] -> [B,C,N] for the PV product
//   timestep_embedding   util.py:151-171
//   cfg_ddim_update      ddim.py:212-243 (classifier-free guidance + x0 / direction / noise update)
//   layout converters    NCHW fp32 <-> channel-last fp16, channel concat
//   clip_patches / clip_add_positions   CLIP image tower front end (encoders/modules.py:362-370): bicubic resize +
//                        normalisation + patch gather in one pass, class token and positional embeddings
#include <cuda_fp16.h>

#include "common.cuh"

namespace o2345 {
namespace {

__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }

// Per-group sums of a CTA in a FIXED order (no atomics, so a run is bit-reproducible): thread (prow, slot) holds the partial
// sums s[8] / sums of squares q[8] of channels slot * 8 .. slot * 8 + 7 over its pixels; the pixel rows are added channel by
// channel in row order into chan [2 C], then the channels of a group in channel order into out[2 g], out[2 g + 1].
// blockDim must be rows * C / 8; every thread calls it.
__device__ void block_group_sums(const float (&s)[8], const float (&q)[8], int slot, int prow, int rows, int C, int G,
                                 float* chan, float* out) {
  for (int r = 0; r < rows; ++r) {
    if (prow == r) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int c = slot * 8 + e;
        chan[2 * c] = (r ? chan[2 * c] : 0.f) + s[e];
        chan[2 * c + 1] = (r ? chan[2 * c + 1] : 0.f) + q[e];
      }
    }
    __syncthreads();
  }
  const int cg = C / G;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int c = g * cg; c < (g + 1) * cg; ++c) a += chan[2 * c], b += chan[2 * c + 1];
    out[2 * g] = a, out[2 * g + 1] = b;
  }
  __syncthreads();
}

// GroupNorm statistics folded into a per-(image, channel) affine: y = x * scale[b, c] + shift[b, c] with
// scale = rstd * gamma, shift = beta - mean * rstd * gamma.  x [B, HW, C] fp16 channel-last.
// grid (chunks, B): a CTA reads a slab of pixels with 16-byte loads (thread = fixed 8-channel slot, so the partial sums
// stay in registers), folds them into per-group sums (block_group_sums), stores those in its own slot of the scratch, and the
// LAST CTA of each image (ticket counter) adds the chunks' sums in chunk order, turns them into scale / shift and resets the
// ticket for the next call.  Scratch: B ticket ints, then [B][chunks][2 G] floats.
__global__ void groupnorm_stats_kernel(const __half* __restrict__ x, int HW, int C, int G, float eps,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       float* __restrict__ scratch, int B, int P,
                                       float* __restrict__ scale, float* __restrict__ shift) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float gsm[];           // [2 G] sums, then [2 G] mean / rstd, then [2 C] channel sums
  __shared__ int is_last;
  const int b = blockIdx.y, c8n = C >> 3, cg = C / G;
  const int slot = threadIdx.x % c8n, prow = threadIdx.x / c8n, rows = blockDim.x / c8n;
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = 0.f, q[e] = 0.f;
  const int p0 = blockIdx.x * P, p1 = min(HW, p0 + P);
  const __half* base = x + (int64_t)b * HW * C + slot * 8;
  if (prow < rows) {
    for (int pix = p0 + prow; pix < p1; pix += rows) {
      uint4 v = *reinterpret_cast<const uint4*>(base + (int64_t)pix * C);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h[e]);
        s[2 * e] += f.x, q[2 * e] = fmaf(f.x, f.x, q[2 * e]);
        s[2 * e + 1] += f.y, q[2 * e + 1] = fmaf(f.y, f.y, q[2 * e + 1]);
      }
    }
  }
  block_group_sums(s, q, slot, prow, rows, C, G, gsm + 4 * G, gsm);
  int* ticket = reinterpret_cast<int*>(scratch) + b;
  float* parts = scratch + B + (int64_t)b * gridDim.x * 2 * G;           // this image's [chunks][2 G]
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) parts[(int64_t)blockIdx.x * 2 * G + i] = gsm[i];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float ts = 0.f, tq = 0.f;
    for (int k = 0; k < (int)gridDim.x; ++k) ts += __ldcg(parts + (int64_t)k * 2 * G + 2 * g), tq += __ldcg(parts + (int64_t)k * 2 * G + 2 * g + 1);
    float n = (float)HW * cg, m = ts / n;
    float var = fmaxf(tq / n - m * m, 0.f);
    gsm[2 * g] = m, gsm[2 * g + 1] = rsqrtf(var + eps);
  }
  __syncthreads();
  if (threadIdx.x == 0) *ticket = 0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float m = gsm[2 * (c / cg)], r = gsm[2 * (c / cg) + 1];
    float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    scale[(int64_t)b * C + c] = r * ga, shift[(int64_t)b * C + c] = be - m * r * ga;
  }
}

// out[(b, oy, ox), (ky, kx, c)] = f(in[b, iy, ix, c]);  f = optional per-(image, channel) affine (GroupNorm) (+SiLU).
// KS in {1,3}; `up` doubles the input grid by nearest-neighbour replication before the convolution; zero padding.
__global__ void norm_act_im2col_kernel(const __half* __restrict__ x, int B, int H, int W, int C, int KS, int stride, int up,
                                       const float* __restrict__ scale, const float* __restrict__ shift, int act,
                                       __half* __restrict__ out, int Ho, int Wo, int pad) {
  pdl_wait();
  pdl_trigger();
  const int c8 = C >> 3;  // 8 channels (16 bytes) per thread
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = (int64_t)B * Ho * Wo * KS * KS * c8;
  if (idx >= total) return;
  int cc = (int)(idx % c8);
  int kk = (int)((idx / c8) % (KS * KS));
  int64_t pix = idx / ((int64_t)c8 * KS * KS);
  int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), b = (int)(pix / ((int64_t)Wo * Ho));
  int ky = kk / KS, kx = kk % KS;
  int Hin = up ? 2 * H : H, Win = up ? 2 * W : W;
  int iy = oy * stride + ky - pad, ix = ox * stride + kx - pad;
  uint4 o = make_uint4(0, 0, 0, 0);
  if (iy >= 0 && iy < Hin && ix >= 0 && ix < Win) {
    int sy = up ? iy >> 1 : iy, sx = up ? ix >> 1 : ix;
    uint4 v = *reinterpret_cast<const uint4*>(x + (((int64_t)b * H + sy) * W + sx) * C + cc * 8);
    if (scale) {
      const __half2* h = reinterpret_cast<const __half2*>(&v);
      const float4* sc = reinterpret_cast<const float4*>(scale + (int64_t)b * C + cc * 8);
      const float4* sh = reinterpret_cast<const float4*>(shift + (int64_t)b * C + cc * 8);
      float4 s0 = __ldg(sc), s1 = __ldg(sc + 1), t0 = __ldg(sh), t1 = __ldg(sh + 1);
      float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w}, tv[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
      __half2 r[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h[e]);
        f.x = fmaf(f.x, sv[2 * e], tv[2 * e]), f.y = fmaf(f.y, sv[2 * e + 1], tv[2 * e + 1]);
        if (act) f.x = silu(f.x), f.y = silu(f.y);
        r[e] = __floats2half2_rn(f.x, f.y);
      }
      o = *reinterpret_cast<uint4*>(r);
    } else {
      o = v;
    }
  }
  *reinterpret_cast<uint4*>(out + (pix * KS * KS + kk) * C + cc * 8) = o;
}

// KS = 1 without stride / up-sampling is a plain per-(image, channel) affine (+SiLU) over the activation -- most GroupNorm
// applications of the VAE, whose maps are too large for the one-kernel cluster GroupNorm.  grid (chunks, B); blockDim is a
// multiple of C / 8, so a thread keeps its 8-channel slot (scale / shift fetched once, no index divisions per element) and
// has four 16-byte loads in flight.  (The general gather above spends ~300 instructions per 16 bytes on 64-bit index
// arithmetic and table loads: 1.3 TB/s on the VAE's 67 MB maps.)
__global__ void norm_act_apply_kernel(const __half* __restrict__ x, int HW, int C, const float* __restrict__ scale,
                                      const float* __restrict__ shift, int act, __half* __restrict__ out, int P) {
  pdl_wait();
  pdl_trigger();
  constexpr int U = 4;
  const int b = blockIdx.y, c8n = C >> 3;
  const int slot = threadIdx.x % c8n, prow = threadIdx.x / c8n, rows = blockDim.x / c8n;
  float sv[8], tv[8];
  {
    const float4* sc = reinterpret_cast<const float4*>(scale + (int64_t)b * C + slot * 8);
    const float4* sh = reinterpret_cast<const float4*>(shift + (int64_t)b * C + slot * 8);
    const float4 s0 = __ldg(sc), s1 = __ldg(sc + 1), t0 = __ldg(sh), t1 = __ldg(sh + 1);
    sv[0] = s0.x, sv[1] = s0.y, sv[2] = s0.z, sv[3] = s0.w, sv[4] = s1.x, sv[5] = s1.y, sv[6] = s1.z, sv[7] = s1.w;
    tv[0] = t0.x, tv[1] = t0.y, tv[2] = t0.z, tv[3] = t0.w, tv[4] = t1.x, tv[5] = t1.y, tv[6] = t1.z, tv[7] = t1.w;
  }
  const int p0 = blockIdx.x * P, p1 = min(HW, p0 + P);
  const __half* base = x + (int64_t)b * HW * C + slot * 8;
  __half* obase = out + (int64_t)b * HW * C + slot * 8;
  for (int pix = p0 + prow; pix < p1; pix += U * rows) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (pix + u * rows < p1) v[u] = *reinterpret_cast<const uint4*>(base + (int64_t)(pix + u * rows) * C);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = pix + u * rows;
      if (pu >= p1) break;
      const __half2* h = reinterpret_cast<const __half2*>(&v[u]);
      __half2 r[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h[e]);
        f.x = fmaf(f.x, sv[2 * e], tv[2 * e]), f.y = fmaf(f.y, sv[2 * e + 1], tv[2 * e + 1]);
        if (act) f.x = silu(f.x), f.y = silu(f.y);
        r[e] = __floats2half2_rn(f.x, f.y);
      }
      *reinterpret_cast<uint4*>(obase + (int64_t)pu * C) = *reinterpret_cast<uint4*>(r);
    }
  }
}

// GroupNorm (+SiLU) of a whole activation in ONE kernel (ksize 1: the implicit-conv and transformer inputs, 55 of the 61 GroupNorms
// of a UNet pass): an image is handled by one thread-block CLUSTER of CL CTAs.  Pass 1: every CTA reads its slab of pixels
// ONCE (16-byte loads, four in flight per thread, a thread keeps its 8-channel slot), parks it in shared memory (KEEP) and sums
// it into per-group shared-memory sums; the CL partial sums are exchanged through distributed shared memory
// (ld.shared::cluster) around one cluster barrier; pass 2 normalises the parked slab and writes it: x is read once and y
// written once -- the traffic floor of the operation.  (Slabs over 200 KB per CTA -- not reached by the UNet / VAE shapes at
// the cluster sizes the launcher picks -- re-read x from L2 instead.)  Replaces groupnorm_stats (global atomics + ticket +
// last-CTA finalize) followed by norm_act_im2col: one launch instead of two, no global atomics, no scratch.
// Round-2 history: the first version read one 16-byte piece per thread and iteration in both passes and summed the 16 remote
// partials with dependent loads: 21-28 us per launch at the batched sampler sizes, a sixth of what the traffic needs.
template <bool KEEP>
__global__ void groupnorm_apply_cluster_kernel(const __half* __restrict__ x, int HW, int C, int G, float eps,
                                               const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                               __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) float gsm[];           // [2 G] this CTA's sums, [2 G] the image's sums, [2 C] channel sums,
                                                          // then (KEEP) the slab
  constexpr int U = 4;
  uint32_t rank, csize;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(csize));
  const int b = blockIdx.y, cg = C / G, c8n = C >> 3;
  const int slot = threadIdx.x % c8n, prow = threadIdx.x / c8n, rows = blockDim.x / c8n;   // blockDim is a multiple of c8n
  uint4* slab = reinterpret_cast<uint4*>(gsm + ((4 * G + 2 * C + 3) & ~3));
  const int P = (HW + (int)csize - 1) / (int)csize;
  const int p0 = (int)rank * P, p1 = min(HW, p0 + P);
  const __half* base = x + (int64_t)b * HW * C + slot * 8;
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = 0.f, q[e] = 0.f;
  for (int pix = p0 + prow; pix < p1; pix += U * rows) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      v[u] = pix + u * rows < p1 ? *reinterpret_cast<const uint4*>(base + (int64_t)(pix + u * rows) * C) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (KEEP && pix + u * rows < p1) slab[(pix + u * rows - p0) * c8n + slot] = v[u];
      const __half2* h = reinterpret_cast<const __half2*>(&v[u]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        s[2 * e] += f.x, q[2 * e] = fmaf(f.x, f.x, q[2 * e]);
        s[2 * e + 1] += f.y, q[2 * e + 1] = fmaf(f.y, f.y, q[2 * e + 1]);
      }
    }
  }
  block_group_sums(s, q, slot, prow, rows, C, G, gsm + 4 * G, gsm);
  // every CTA's partial sums become visible to the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {
    const uint32_t local = (uint32_t)__cvta_generic_to_shared(gsm + i);
    float part[16];                                        // the (up to 16) remote loads are independent: one round trip
#pragma unroll
    for (uint32_t r = 0; r < 16; ++r) {
      part[r] = 0.f;
      if (r < csize) {
        uint32_t remote;
        asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(r));
        asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(part[r]) : "r"(remote));
      }
    }
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) t += part[r];
    gsm[2 * G + i] = t;
  }
  __syncthreads();
  // no CTA may leave (or overwrite its sums) while a sibling still reads them
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  float sv[8], tv[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = slot * 8 + e, g = c / cg;
    const float n = (float)HW * (float)cg, m = gsm[2 * G + 2 * g] / n;
    const float r = rsqrtf(fmaxf(gsm[2 * G + 2 * g + 1] / n - m * m, 0.f) + eps);
    const float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    sv[e] = r * ga, tv[e] = be - m * r * ga;
  }
  __half* obase = out + (int64_t)b * HW * C + slot * 8;
  for (int pix = p0 + prow; pix < p1; pix += U * rows) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = pix + u * rows;
      if (pu < p1) v[u] = KEEP ? slab[(pu - p0) * c8n + slot] : *reinterpret_cast<const uint4*>(base + (int64_t)pu * C);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = pix + u * rows;
      if (pu >= p1) break;
      const __half2* h = reinterpret_cast<const __half2*>(&v[u]);
      __half2 r[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h[e]);
        f.x = fmaf(f.x, sv[2 * e], tv[2 * e]), f.y = fmaf(f.y, sv[2 * e + 1], tv[2 * e + 1]);
        if (act) f.x = silu(f.x), f.y = silu(f.y);
        r[e] = __floats2half2_rn(f.x, f.y);
      }
      *reinterpret_cast<uint4*>(obase + (int64_t)pu * C) = *reinterpret_cast<uint4*>(r);
    }
  }
}

// one warp per row: y = (x - mean) * rstd * gamma + beta, fp32 math.  The row is fetched ONCE with 16-byte loads (a lane keeps up to
// MAXJ chunks of 8 channels in registers between the statistics and the normalisation) and written with 16-byte stores.
// (The first version read single halves, twice, and stored single halves: 1.2 TB/s on the batch-64 UNet's 42-168 MB tensors.)
template <int MAXJ>
__global__ void layernorm_rows_vec_kernel(const __half* __restrict__ x, int64_t M, int C, float eps, const float* __restrict__ gamma,
                                          const float* __restrict__ beta, __half* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, nch = C >> 3;
  if (row >= M) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  uint4 v[MAXJ];
  float s = 0.f, q = 0.f;
#pragma unroll
  for (int j = 0; j < MAXJ; ++j) {
    const int ch = lane + 32 * j;
    if (ch < nch) {
      v[j] = xr[ch];
      const __half2* h = reinterpret_cast<const __half2*>(&v[j]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        s += f.x + f.y, q = fmaf(f.x, f.x, fmaf(f.y, f.y, q));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o), q += __shfl_xor_sync(0xffffffffu, q, o);
  const float m = s / C, r = rsqrtf(fmaxf(q / C - m * m, 0.f) + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int j = 0; j < MAXJ; ++j) {
    const int ch = lane + 32 * j;
    if (ch < nch) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + 8 * ch)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + 8 * ch + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + 8 * ch)), b1 = __ldg(reinterpret_cast<const float4*>(beta + 8 * ch + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      const __half2* h = reinterpret_cast<const __half2*>(&v[j]);
      __half2 o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        o[e] = __floats2half2_rn((f.x - m) * r * gg[2 * e] + bb[2 * e], (f.y - m) * r * gg[2 * e + 1] + bb[2 * e + 1]);
      }
      yr[ch] = *reinterpret_cast<uint4*>(o);
    }
  }
}

// any C (scalar accesses): the fallback for rows that are not whole 16-byte chunks
__global__ void layernorm_rows_kernel(const __half* __restrict__ x, int64_t M, int C, float eps,
                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                      __half* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= M) return;
  const __half* xr = x + row * C;
  float s = 0.f, q = 0.f;
  for (int c = lane; c < C; c += 32) { float v = __half2float(xr[c]); s += v, q = fmaf(v, v, q); }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o), q += __shfl_xor_sync(0xffffffffu, q, o);
  float m = s / C, r = rsqrtf(fmaxf(q / C - m * m, 0.f) + eps);
  for (int c = lane; c < C; c += 32) y[row * C + c] = __float2half_rn((__half2float(xr[c]) - m) * r * gamma[c] + beta[c]);
}

// one warp per row of length n (<= 1024): probabilities in fp16
__global__ void softmax_rows_kernel(const __half* __restrict__ s, int64_t rows, int n, __half* __restrict__ p) {
  pdl_wait();
  pdl_trigger();
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const __half* sr = s + row * n;
  float v[32];
  float mx = -3.4e38f;
  int cnt = (n + 31) / 32;
  for (int i = 0; i < cnt; ++i) {
    int c = lane + 32 * i;
    v[i] = c < n ? __half2float(sr[c]) : -3.4e38f;
    mx = fmaxf(mx, v[i]);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int i = 0; i < cnt; ++i) { v[i] = (lane + 32 * i < n) ? expf(v[i] - mx) : 0.f; sum += v[i]; }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  float inv = 1.f / sum;
  for (int i = 0; i < cnt; ++i) { int c = lane + 32 * i; if (c < n) p[row * n + c] = __float2half_rn(v[i] * inv); }
}

__global__ void geglu_kernel(const __half* __restrict__ x, int64_t M, int I, __half* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  const int i8 = I >> 3;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * i8) return;
  int64_t r = i / i8;
  int c = (int)(i - r * i8) * 8;
  uint4 va = *reinterpret_cast<const uint4*>(x + r * 2 * I + c), vg = *reinterpret_cast<const uint4*>(x + r * 2 * I + I + c);
  const __half* a = reinterpret_cast<const __half*>(&va);
  const __half* g = reinterpret_cast<const __half*>(&vg);
  __half o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float gf = __half2float(g[e]);
    o[e] = __float2half_rn(__half2float(a[e]) * (0.5f * gf * (1.f + erff(gf * 0.70710678118654752f))));
  }
  *reinterpret_cast<uint4*>(y + r * I + c) = *reinterpret_cast<uint4*>(o);
}

__global__ void silu_kernel(const __half* __restrict__ x, int64_t n, __half* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __float2half_rn(silu(__half2float(x[i])));
}

// [B, N, C] -> [B, C, N]
__global__ void transpose_tokens_kernel(const __half* __restrict__ x, int N, int C, __half* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  __shared__ __half tile[32][33];
  int b = blockIdx.z, n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int n = n0 + j, c = c0 + threadIdx.x;
    if (n < N && c < C) tile[j][threadIdx.x] = x[((int64_t)b * N + n) * C + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int c = c0 + j, n = n0 + threadIdx.x;
    if (n < N && c < C) y[((int64_t)b * C + c) * N + n] = tile[threadIdx.x][j];
  }
}

// timestep_embedding(t, dim): [cos(t * f_i) | sin(t * f_i)], f_i = exp(-ln(10000) * i / half)   (util.py:151-171)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B, int dim, __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int half_dim = dim / 2;
  if (i >= B * half_dim) return;
  int b = i / half_dim, k = i % half_dim;
  float f = expf(-logf(10000.f) * (float)k / (float)half_dim);
  float a = t[b] * f;
  out[b * dim + k] = __float2half_rn(cosf(a));
  out[b * dim + half_dim + k] = __float2half_rn(sinf(a));
}

// y[b, p, c] += e[b, c]   (ResBlock: h + emb_out[..., None, None], openaimodel.py:271)
__global__ void add_channel_bias_kernel(__half* __restrict__ y, const __half* __restrict__ e, int HW, int C, int lde, int64_t total) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int c = (int)(i % C);
  int64_t b = i / ((int64_t)HW * C);
  y[i] = __float2half_rn(__half2float(y[i]) + __half2float(e[b * lde + c]));
}

// dst[:, off:off+C] = src  (channel concat on channel-last rows)
__global__ void copy_channels_kernel(const __half* __restrict__ src, int64_t M, int C, __half* __restrict__ dst, int ldd, int off) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int c8 = C >> 3;
  if (i >= M * c8) return;
  int64_t r = i / c8;
  int c = (int)(i - r * c8) * 8;
  *reinterpret_cast<uint4*>(dst + r * ldd + off + c) = *reinterpret_cast<const uint4*>(src + r * C + c);
}

__global__ void nchw_f32_to_cl_f16_kernel(const float* __restrict__ x, int B, int C, int HW, __half* __restrict__ y, int ldy, int off) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * C * HW) return;
  int p = (int)(i % HW), c = (int)((i / HW) % C);
  int64_t b = i / ((int64_t)HW * C);
  y[(b * HW + p) * ldy + off + c] = __float2half_rn(x[i]);
}

__global__ void cl_f16_to_nchw_f32_kernel(const __half* __restrict__ x, int B, int C, int HW, int ldx, float* __restrict__ y) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * C * HW) return;
  int p = (int)(i % HW), c = (int)((i / HW) % C);
  int64_t b = i / ((int64_t)HW * C);
  y[i] = __half2float(x[(b * HW + p) * ldx + c]);
}

// e_t = e_uc + s (e_c - e_uc); pred_x0 = (x - sqrt(1-a) e_t)/sqrt(a); x_prev = sqrt(a') pred_x0 + sqrt(1-a'-sigma^2) e_t
// + sigma * noise.  eps holds [uncond batch | cond batch] (ddim.py:196-243); all fp32.
__global__ void cfg_ddim_update_kernel(const float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ noise,
                                       int64_t n, float scale, float a_t, float a_prev, float sigma_t, float sqrt_1m_at,
                                       float* __restrict__ x_prev, float* __restrict__ pred_x0) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float eu = eps[i], ec = eps[n + i];
  float e = eu + scale * (ec - eu);
  float p0 = (x[i] - sqrt_1m_at * e) / sqrtf(a_t);
  float dir = sqrtf(1.f - a_prev - sigma_t * sigma_t) * e;
  float nz = sigma_t * (noise ? noise[i] : 0.f);
  x_prev[i] = sqrtf(a_prev) * p0 + dir + nz;
  if (pred_x0) pred_x0[i] = p0;
}

// ---- CLIP image tower front end (reference ldm/modules/encoders/modules.py:362-370 + the patch embedding's im2col)
// bicubic weights of torch's upsample_bicubic2d (A = -0.75) for the taps at offsets -1, 0, 1, 2
__device__ __forceinline__ void cubic_w(float t, float (&w)[4]) {
  const float A = -0.75f;
  float x = t + 1.f;
  w[0] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
  w[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
  x = 1.f - t;
  w[2] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
  x = 2.f - t;
  w[3] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
}
// x [B,3,H,W] fp32 in [-1,1] -> rows (b, py, px) x columns (c, ky, kx) of the res x res bicubic resize (align_corners),
// mapped to [0,1] and normalised with the CLIP mean / std; fp16; columns 3 P^2 .. kp-1 are zero padding
__global__ void clip_patches_kernel(const float* __restrict__ x, int B, int H, int W, int res, int P, float m0, float m1, float m2,
                                    float s0, float s1, float s2, int kp, __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int g = res / P, kk = 3 * P * P;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * g * g * kp) return;
  const int col = (int)(i % kp);
  const int64_t row = i / kp;
  if (col >= kk) { out[i] = __float2half(0.f); return; }
  const int c = col / (P * P), ky = (col / P) % P, kx = col % P;
  const int px = (int)(row % g), py = (int)((row / g) % g), b = (int)(row / (g * g));
  const int oy = py * P + ky, ox = px * P + kx;
  const float sy = (float)oy * (float)(H - 1) / (float)(res - 1), sx = (float)ox * (float)(W - 1) / (float)(res - 1);
  const float fy = floorf(sy), fx = floorf(sx);
  float wy[4], wx[4];
  cubic_w(sy - fy, wy), cubic_w(sx - fx, wx);
  const float* src = x + ((int64_t)b * 3 + c) * H * W;
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int yy = min(max((int)fy - 1 + j, 0), H - 1);
    float r = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) r = fmaf(__ldg(src + (int64_t)yy * W + min(max((int)fx - 1 + k, 0), W - 1)), wx[k], r);
    acc = fmaf(r, wy[j], acc);
  }
  const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
  out[i] = __float2half_rn(((acc + 1.f) * 0.5f - mean) / sd);
}

// tok [B*N, d] fp16: row n = 0 of every image becomes class_embedding + pos[0]; rows n >= 1 (patch embeddings) += pos[n]
__global__ void clip_add_positions_kernel(__half* __restrict__ tok, const float* __restrict__ cls, const float* __restrict__ pos, int B,
                                          int N, int d) {
  pdl_wait();
  pdl_trigger();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * N * d) return;
  const int c = (int)(i % d), n = (int)((i / d) % N);
  const float v = n == 0 ? cls[c] : __half2float(tok[i]);
  tok[i] = __float2half_rn(v + pos[(int64_t)n * d + c]);
}

}  // namespace
}  // namespace o2345

using namespace o2345;
#define ST ((cudaStream_t)stream)

// B ticket ints, then [B][chunks][2 G] per-CTA sums; o2345_groupnorm_stats launches at most cdiv(2 * SMs, B) chunks per image
extern "C" int64_t o2345_groupnorm_scratch_floats(int B, int G) { return (int64_t)B + (int64_t)B * cdiv(2 * sm_count(), B) * 2 * G; }

extern "C" int o2345_groupnorm_stats(const void* x, int B, int HW, int C, int G, float eps, const float* gamma,
                                     const float* beta, float* scratch, float* scale, float* shift, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && scratch && scale && shift && B > 0 && HW > 0 && G > 0 && C % G == 0, "bad arguments");
  O2345_CHECK_ARG((C % 8) == 0 && C / 8 <= 1024 && ((uintptr_t)x % 16) == 0, "C must be a multiple of 8 (<= 8192), x 16-byte aligned");
  const int c8n = C / 8;
  const int rows = c8n >= 256 ? 1 : 256 / c8n;
  const int threads = c8n * rows;
  int chunks = cdiv(2 * sm_count(), B);
  if (chunks > HW / (2 * rows)) chunks = HW / (2 * rows);
  if (chunks < 1) chunks = 1;
  const int P = cdiv(HW, chunks);
  chunks = cdiv(HW, P);
  const size_t smem = (size_t)(4 * G + 2 * C) * sizeof(float);
  static PerDeviceOnce attr;
  if (attr.need()) O2345_CUDA(cudaFuncSetAttribute(groupnorm_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (4 * 256 + 2 * 8192)));
  O2345_CUDA(launch_pdl(groupnorm_stats_kernel, dim3(dim3(chunks, B)), dim3(threads), smem, ST, (const __half*)x, HW, C, G, eps, gamma, beta,
                                                                                  scratch, B, P, scale, shift));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

static int g_gn_cluster = 0;   // tuning hook: CTAs per image of the one-kernel GroupNorm (0: the launcher's rule)
extern "C" void o2345_debug_groupnorm_cluster(int cl) { g_gn_cluster = cl; }

extern "C" int o2345_groupnorm_apply(const void* x, int B, int HW, int C, int G, float eps, const float* gamma, const float* beta,
                                     int act, void* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && out && B > 0 && HW > 0 && G > 0 && G <= 256 && C % G == 0, "bad arguments");
  O2345_CHECK_ARG((C % 8) == 0 && C / 8 <= 1024 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 16) == 0,
                  "C must be a multiple of 8 (<= 8192), x and out 16-byte aligned");
  const int c8n = C / 8;
  const int rows = c8n >= 512 ? 1 : 512 / c8n;
  const int threads = c8n * rows;
  // CTAs per image = cluster size (a power of two <= 8, the portable size: a cluster of CTAs that park up to 200 KB each
  // must fit one GPC).  The rule aims at about ONE CTA per SM for the whole launch (tools/gn_bench.py sweeps it), except
  // that slabs beyond ~400 KB per CTA want one more doubling.  Never more CTAs than the image has pixel rows.
  int cl = 1;
  while (cl < 8 && (int64_t)2 * cl * B <= (int64_t)sm_count()) cl <<= 1;
  if (cl < 8 && (int64_t)HW * C * 2 / cl > 400 * 1024) cl <<= 1;
  while (cl > 1 && HW < cl * rows) cl >>= 1;
  if (g_gn_cluster > 0) {
    cl = g_gn_cluster < 8 ? g_gn_cluster : 8;
    while (cl > 1 && HW < cl * rows) cl >>= 1;
  }
  const size_t sums = (size_t)((4 * G + 2 * C + 3) & ~3) * sizeof(float);
  const size_t slab = (size_t)cdiv(HW, cl) * C * 2;
  const bool keep = sums + slab <= 200 * 1024;
  static PerDeviceOnce attr;
  if (attr.need()) {
    O2345_CUDA(cudaFuncSetAttribute(groupnorm_apply_cluster_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    O2345_CUDA(cudaFuncSetAttribute(groupnorm_apply_cluster_kernel<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    O2345_CUDA(cudaFuncSetAttribute(groupnorm_apply_cluster_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 201 * 1024));
    O2345_CUDA(cudaFuncSetAttribute(groupnorm_apply_cluster_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 201 * 1024));
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(cl, B), cfg.blockDim = dim3(threads), cfg.dynamicSmemBytes = sums + (keep ? slab : 0), cfg.stream = ST;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  at[1].id = cudaLaunchAttributeClusterDimension;
  at[1].val.clusterDim.x = cl, at[1].val.clusterDim.y = 1, at[1].val.clusterDim.z = 1;
  cfg.attrs = at, cfg.numAttrs = 2;
  if (keep)
    O2345_CUDA(cudaLaunchKernelEx(&cfg, groupnorm_apply_cluster_kernel<true>, (const __half*)x, HW, C, G, eps, gamma, beta, act, (__half*)out));
  else
    O2345_CUDA(cudaLaunchKernelEx(&cfg, groupnorm_apply_cluster_kernel<false>, (const __half*)x, HW, C, G, eps, gamma, beta, act, (__half*)out));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_norm_act_im2col(const void* x, int B, int H, int W, int C, int ksize, int stride, int upsample, int pad_lo,
                                     const float* scale, const float* shift, int act, void* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && out && (C % 8) == 0 && (ksize == 1 || ksize == 3) && (stride == 1 || stride == 2), "bad arguments");
  O2345_CHECK_ARG(!scale == !shift, "scale and shift come together");
  int Hin = upsample ? 2 * H : H, Win = upsample ? 2 * W : W;
  int pad_hi = ksize / 2, pad = pad_lo < 0 ? ksize / 2 : pad_lo;   // pad_lo = 0: the VAE's (0,1,0,1) down-sampling pad
  int Ho = (Hin + pad + pad_hi - ksize) / stride + 1, Wo = (Win + pad + pad_hi - ksize) / stride + 1;
  if (ksize == 1 && stride == 1 && !upsample && scale && C / 8 <= 512 && (int64_t)H * W < (1 << 30)) {
    const int c8 = C / 8, threads = (512 / c8) * c8, rows = threads / c8, HW = H * W;
    int chunks = cdiv(4 * sm_count(), B);
    if (chunks > HW / (4 * rows)) chunks = HW / (4 * rows);
    if (chunks < 1) chunks = 1;
    const int P = cdiv(HW, chunks);
    O2345_CUDA(launch_pdl(norm_act_apply_kernel, dim3(cdiv(HW, P), B), dim3(threads), (size_t)(0), ST, (const __half*)x, HW, C, scale, shift, act,
                          (__half*)out, P));
    O2345_LAUNCH_CHECK();
    return O2345_OK;
  }
  int64_t total = (int64_t)B * Ho * Wo * ksize * ksize * (C / 8);
  O2345_CUDA(launch_pdl(norm_act_im2col_kernel, dim3(cdiv(total, 256)), dim3(256), (size_t)(0), ST, (const __half*)x, B, H, W, C, ksize, stride, upsample, scale, shift,
                                                           act, (__half*)out, Ho, Wo, pad));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_layernorm_rows(const void* x, int64_t M, int C, float eps, const float* gamma, const float* beta, void* y,
                                    o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y && gamma && beta, "null pointer");
  const bool vec = (C % 8) == 0 && C / 8 <= 160 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)gamma % 16) == 0 &&
                   ((uintptr_t)beta % 16) == 0;
  if (vec && C / 8 <= 64)
    O2345_CUDA(launch_pdl(layernorm_rows_vec_kernel<2>, dim3(cdiv(M, 8)), dim3(256), (size_t)(0), ST, (const __half*)x, M, C, eps, gamma, beta, (__half*)y));
  else if (vec && C / 8 <= 96)
    O2345_CUDA(launch_pdl(layernorm_rows_vec_kernel<3>, dim3(cdiv(M, 8)), dim3(256), (size_t)(0), ST, (const __half*)x, M, C, eps, gamma, beta, (__half*)y));
  else if (vec)
    O2345_CUDA(launch_pdl(layernorm_rows_vec_kernel<5>, dim3(cdiv(M, 8)), dim3(256), (size_t)(0), ST, (const __half*)x, M, C, eps, gamma, beta, (__half*)y));
  else
    O2345_CUDA(launch_pdl(layernorm_rows_kernel, dim3(cdiv(M, 8)), dim3(256), (size_t)(0), ST, (const __half*)x, M, C, eps, gamma, beta, (__half*)y));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_softmax_rows(const void* s, int64_t rows, int n, void* p, o2345_stream_t stream) {
  O2345_CHECK_ARG(s && p && n >= 1 && n <= 1024, "row length must be 1..1024");
  O2345_CUDA(launch_pdl(softmax_rows_kernel, dim3(cdiv(rows, 8)), dim3(256), (size_t)(0), ST, (const __half*)s, rows, n, (__half*)p));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_geglu(const void* x, int64_t M, int I, void* y, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y && (I % 8) == 0, "null pointer / I must be a multiple of 8");
  O2345_CUDA(launch_pdl(geglu_kernel, dim3(cdiv(M * (I / 8), 256)), dim3(256), (size_t)(0), ST, (const __half*)x, M, I, (__half*)y));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_silu(const void* x, int64_t n, void* y, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y, "null pointer");
  O2345_CUDA(launch_pdl(silu_kernel, dim3(cdiv(n, 256)), dim3(256), (size_t)(0), ST, (const __half*)x, n, (__half*)y));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_transpose_tokens(const void* x, int B, int N, int C, void* y, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y, "null pointer");
  O2345_CUDA(launch_pdl(transpose_tokens_kernel, dim3(dim3(cdiv(N, 32), cdiv(C, 32), B)), dim3(dim3(32, 8)), (size_t)(0), ST, (const __half*)x, N, C, (__half*)y));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_timestep_embedding(const float* t, int B, int dim, void* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(t && out && dim % 2 == 0, "bad arguments");
  O2345_CUDA(launch_pdl(timestep_embedding_kernel, dim3(cdiv(B * dim / 2, 128)), dim3(128), (size_t)(0), ST, t, B, dim, (__half*)out));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_add_channel_bias(void* y, const void* e, int B, int HW, int C, int lde, o2345_stream_t stream) {
  O2345_CHECK_ARG(y && e, "null pointer");
  int64_t total = (int64_t)B * HW * C;
  O2345_CUDA(launch_pdl(add_channel_bias_kernel, dim3(cdiv(total, 256)), dim3(256), (size_t)(0), ST, (__half*)y, (const __half*)e, HW, C, lde, total));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_copy_channels(const void* src, int64_t M, int C, void* dst, int ldd, int off, o2345_stream_t stream) {
  O2345_CHECK_ARG(src && dst && (C % 8) == 0 && (ldd % 8) == 0 && (off % 8) == 0, "channels must be multiples of 8");
  O2345_CUDA(launch_pdl(copy_channels_kernel, dim3(cdiv(M * (C / 8), 256)), dim3(256), (size_t)(0), ST, (const __half*)src, M, C, (__half*)dst, ldd, off));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_nchw_f32_to_cl_f16(const float* x, int B, int C, int HW, void* y, int ldy, int off, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y, "null pointer");
  O2345_CUDA(launch_pdl(nchw_f32_to_cl_f16_kernel, dim3(cdiv((int64_t)B * C * HW, 256)), dim3(256), (size_t)(0), ST, x, B, C, HW, (__half*)y, ldy, off));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_cl_f16_to_nchw_f32(const void* x, int B, int C, int HW, int ldx, float* y, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && y, "null pointer");
  O2345_CUDA(launch_pdl(cl_f16_to_nchw_f32_kernel, dim3(cdiv((int64_t)B * C * HW, 256)), dim3(256), (size_t)(0), ST, (const __half*)x, B, C, HW, ldx, y));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_cfg_ddim_update(const float* x, const float* eps, const float* noise, int64_t n, float scale, float a_t,
                                     float a_prev, float sigma_t, float sqrt_one_minus_at, float* x_prev, float* pred_x0,
                                     o2345_stream_t stream) {
  O2345_CHECK_ARG(x && eps && x_prev, "null pointer");
  O2345_CUDA(launch_pdl(cfg_ddim_update_kernel, dim3(cdiv(n, 256)), dim3(256), (size_t)(0), ST, x, eps, noise, n, scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, x_prev, pred_x0));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_clip_patches(const float* x, int B, int H, int W, int res, int patch, const float* mean3, const float* std3, int kp,
                                  void* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && mean3 && std3 && out, "null pointer");
  O2345_CHECK_ARG(B > 0 && H > 1 && W > 1 && res > 1 && patch > 0 && res % patch == 0 && kp >= 3 * patch * patch && (kp % 8) == 0,
                  "bad sizes (res must be a multiple of patch, kp a multiple of 8 >= 3 patch^2)");
  const int g = res / patch;
  const int64_t total = (int64_t)B * g * g * kp;
  O2345_CUDA(launch_pdl(clip_patches_kernel, dim3(cdiv(total, 256)), dim3(256), (size_t)0, ST, x, B, H, W, res, patch, mean3[0], mean3[1],
                        mean3[2], std3[0], std3[1], std3[2], kp, (__half*)out));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_clip_add_positions(void* tok, const float* cls, const float* pos, int B, int N, int d, o2345_stream_t stream) {
  O2345_CHECK_ARG(tok && cls && pos && B > 0 && N > 0 && d > 0, "bad arguments");
  O2345_CUDA(launch_pdl(clip_add_positions_kernel, dim3(cdiv((int64_t)B * N * d, 256)), dim3(256), (size_t)0, ST, (__half*)tok, cls, pos,
                        B, N, d));
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
