// FeatureNet (FPN) + compress layer primitives: direct conv2d, batch-statistics InPlaceABN,
// bilinear x2/x4 upsampling with fused add / channel concat.  Rows B1/B2 of SURVEY.md section 8.
// Replaces cuDNN conv2d + inplace_abn + F.interpolate call sites in reference
// models/featurenet.py:12-91, trainer_generic.py:1104-1125, sparse_sdf_network.py:171-173,311-315.
//
// The whole network is bandwidth-bound (2.2 GFLOP / image against ~20 MB of activations per
// image), so the kernels are organised around traffic: a 16x16 output tile of ALL output
// channels per CTA (input patch staged once in shared memory, weights broadcast as float4s),
// the batch statistics of the following InPlaceABN reduced in the conv epilogue (no extra
// read pass), and a strided output view so that normalised results land directly in the
// channel-last / concatenated layout the next stage gathers from.
#include "common.cuh"

namespace o2345 {
namespace {

constexpr int TILE = 16;
constexpr int CCH = 4;  // input channels staged per iteration

template <int COUT, int K, int S>
__global__ void __launch_bounds__(TILE * TILE)
conv2d_kernel(const float* __restrict__ in, int Cin, int H, int W, const float* __restrict__ wgt,
              const float* __restrict__ bias, int Ho, int Wo, int pad, float* __restrict__ out,
              double* __restrict__ stats) {
  constexpr int PT = (TILE - 1) * S + K;  // input patch side
  __shared__ float sIn[CCH][PT][PT + 1];
  __shared__ __align__(16) float sWt[CCH][K * K][COUT];
  __shared__ float sRed[2][TILE * TILE / 32][COUT];   // per-warp channel sums, added in warp order
  const int tx = threadIdx.x % TILE, ty = threadIdx.x / TILE;
  const int n = blockIdx.z;
  const int ox = blockIdx.x * TILE + tx, oy = blockIdx.y * TILE + ty;
  const int ix0 = blockIdx.x * TILE * S - pad, iy0 = blockIdx.y * TILE * S - pad;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = bias ? __ldg(bias + c) : 0.f;
  const float* inN = in + (int64_t)n * Cin * H * W;
  for (int c0 = 0; c0 < Cin; c0 += CCH) {
    for (int e = threadIdx.x; e < CCH * PT * PT; e += TILE * TILE) {
      int ci = e / (PT * PT), r = (e / PT) % PT, c = e % PT;
      int iy = iy0 + r, ix = ix0 + c;
      float v = 0.f;
      if (c0 + ci < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(inN + ((int64_t)(c0 + ci) * H + iy) * W + ix);
      sIn[ci][r][c] = v;
    }
    for (int e = threadIdx.x; e < CCH * K * K * COUT; e += TILE * TILE) {
      int ci = e / (K * K * COUT), kk = (e / COUT) % (K * K), co = e % COUT;
      sWt[ci][kk][co] = (c0 + ci < Cin) ? __ldg(wgt + ((int64_t)co * Cin + c0 + ci) * K * K + kk) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < CCH; ++ci)
#pragma unroll
      for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          float v = sIn[ci][ty * S + ky][tx * S + kx];
#pragma unroll
          for (int c4 = 0; c4 < COUT / 4; ++c4) {
            float4 w = *reinterpret_cast<const float4*>(&sWt[ci][ky * K + kx][4 * c4]);
            acc[4 * c4 + 0] = fmaf(v, w.x, acc[4 * c4 + 0]);
            acc[4 * c4 + 1] = fmaf(v, w.y, acc[4 * c4 + 1]);
            acc[4 * c4 + 2] = fmaf(v, w.z, acc[4 * c4 + 2]);
            acc[4 * c4 + 3] = fmaf(v, w.w, acc[4 * c4 + 3]);
          }
        }
    __syncthreads();
  }
  const bool valid = ox < Wo && oy < Ho;
  if (valid) {
    float* o = out + ((int64_t)n * COUT * Ho + oy) * Wo + ox;
#pragma unroll
    for (int c = 0; c < COUT; ++c) o[(int64_t)c * Ho * Wo] = acc[c];
  }
  if (stats) {
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
      float s = valid ? acc[c] : 0.f, q = s * s;
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o), q += __shfl_xor_sync(0xffffffffu, q, o);
      if ((threadIdx.x & 31) == 0) sRed[0][threadIdx.x >> 5][c] = s, sRed[1][threadIdx.x >> 5][c] = q;
    }
    __syncthreads();
    if (threadIdx.x < COUT) {   // fixed-order CTA sum; the CTAs' fp32 sums are added in fp64 (exact in practice)
      float s = 0.f, q = 0.f;
      for (int w = 0; w < TILE * TILE / 32; ++w) s += sRed[0][w][threadIdx.x], q += sRed[1][w][threadIdx.x];
      atomicAdd(stats + threadIdx.x, (double)s);
      atomicAdd(stats + COUT + threadIdx.x, (double)q);
    }
  }
}

// InPlaceABN, training mode: (x-mean)/sqrt(var+eps)*(|gamma|+eps)+beta, leaky-ReLU.
__global__ void abn_apply_kernel(const float* __restrict__ x, int N, int C, int H, int W,
                                 const double* __restrict__ stats, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, float slope, o2345_view4 out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = (int64_t)N * C * H * W;
  if (i >= total) return;
  int w = (int)(i % W), h = (int)((i / W) % H), c = (int)((i / ((int64_t)W * H)) % C), n = (int)(i / ((int64_t)W * H * C));
  double cnt = (double)N * H * W;
  double mean = stats[c] / cnt;
  double var = fmax(stats[C + c] / cnt - mean * mean, 0.0);
  float inv = (float)(1.0 / sqrt(var + (double)eps));
  float y = (x[i] - (float)mean) * inv * (fabsf(gamma[c]) + eps) + beta[c];
  y = y > 0.f ? y : y * slope;
  out.ptr[n * out.sn + (c + out.c0) * out.sc + h * out.sh + w * out.sw] = y;
}

// F.interpolate(scale_factor=f, mode='bilinear', align_corners=True) (+ optional add), NCHW in.
__global__ void upsample_kernel(const float* __restrict__ x, int N, int C, int H, int W, int f,
                                const float* __restrict__ add, o2345_view4 out) {
  int Ho = H * f, Wo = W * f;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = (int64_t)N * C * Ho * Wo;
  if (i >= total) return;
  int w = (int)(i % Wo), h = (int)((i / Wo) % Ho), c = (int)((i / ((int64_t)Wo * Ho)) % C), n = (int)(i / ((int64_t)Wo * Ho * C));
  float sh = (float)(H - 1) / (float)(Ho - 1), sw = (float)(W - 1) / (float)(Wo - 1);
  float fy = sh * h, fx = sw * w;
  int y0 = (int)fy, x0 = (int)fx;
  int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float* p = x + ((int64_t)n * C + c) * H * W;
  float v = hy * (hx * p[y0 * W + x0] + lx * p[y0 * W + x1]) + ly * (hx * p[y1 * W + x0] + lx * p[y1 * W + x1]);
  if (add) v += add[i];
  out.ptr[n * out.sn + (c + out.c0) * out.sc + h * out.sh + w * out.sw] = v;
}

__global__ void copy_view_kernel(const float* __restrict__ x, int N, int C, int H, int W, o2345_view4 out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = (int64_t)N * C * H * W;
  if (i >= total) return;
  int w = (int)(i % W), h = (int)((i / W) % H), c = (int)((i / ((int64_t)W * H)) % C), n = (int)(i / ((int64_t)W * H * C));
  out.ptr[n * out.sn + (c + out.c0) * out.sc + h * out.sh + w * out.sw] = x[i];
}

}  // namespace
}  // namespace o2345

using namespace o2345;

template <int COUT, int K, int S>
static void launch_conv2d(const float* in, int N, int Cin, int H, int W, const float* w, const float* b, int Ho,
                          int Wo, int pad, float* out, double* stats, cudaStream_t st) {
  dim3 grid(cdiv(Wo, TILE), cdiv(Ho, TILE), N);
  conv2d_kernel<COUT, K, S><<<grid, TILE * TILE, 0, st>>>(in, Cin, H, W, w, b, Ho, Wo, pad, out, stats);
}

extern "C" int o2345_conv2d(const float* in, int N, int Cin, int H, int W, const float* weight, const float* bias,
                            int Cout, int K, int stride, int pad, float* out, double* stats,
                            o2345_stream_t stream) {
  O2345_CHECK_ARG(in && weight && out, "null pointer");
  O2345_CHECK_ARG(N > 0 && N <= 65535 && Cin > 0 && H > 0 && W > 0, "bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  int Ho = (H + 2 * pad - K) / stride + 1, Wo = (W + 2 * pad - K) / stride + 1;
  if (stats) O2345_CUDA(cudaMemsetAsync(stats, 0, 2 * Cout * sizeof(double), st));
#define O2345_C2D(CO, KK, SS)                                                                        \
  if (Cout == CO && K == KK && stride == SS) {                                                       \
    launch_conv2d<CO, KK, SS>(in, N, Cin, H, W, weight, bias, Ho, Wo, pad, out, stats, st);          \
    O2345_LAUNCH_CHECK();                                                                            \
    return O2345_OK;                                                                                 \
  }
  O2345_C2D(8, 3, 1)
  O2345_C2D(16, 3, 1)
  O2345_C2D(32, 3, 1)
  O2345_C2D(16, 5, 2)
  O2345_C2D(32, 5, 2)
  O2345_C2D(32, 1, 1)
#undef O2345_C2D
  set_error("o2345_conv2d: unsupported (Cout=%d, K=%d, stride=%d)", Cout, K, stride);
  return O2345_EUNSUPPORTED;
}

extern "C" int o2345_abn_apply(const float* x, int N, int C, int H, int W, const double* stats, const float* gamma,
                               const float* beta, float eps, float slope, const o2345_view4* out,
                               o2345_stream_t stream) {
  O2345_CHECK_ARG(x && stats && gamma && beta && out && out->ptr, "null pointer");
  int64_t total = (int64_t)N * C * H * W;
  abn_apply_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, N, C, H, W, stats, gamma, beta, eps, slope, *out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_upsample_bilinear(const float* x, int N, int C, int H, int W, int factor, const float* add,
                                       const o2345_view4* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(x && out && out->ptr, "null pointer");
  O2345_CHECK_ARG(factor >= 1 && H > 1 && W > 1, "bad sizes");
  int64_t total = (int64_t)N * C * H * W * factor * factor;
  if (factor == 1 && !add)
    copy_view_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, N, C, H, W, *out);
  else
    upsample_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, N, C, H, W, factor, add, *out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
