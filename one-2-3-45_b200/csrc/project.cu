// Projection of the input photo onto a mesh (o2345/mesh_texture.py, run.py --project_input): for every query point (a
// vertex or the surface point behind a texel) whether the photo's camera sees it, how squarely, and the photo's colour
// there, blended into the reconstruction's colour.  One thread per point; the rules and constants are in include/o2345.h
// (o2345_project_view).
//
// Every float operation is an explicit round-to-nearest intrinsic in the order oracle/project_oracle.py repeats with
// numpy float32 (no FMA contraction), so weights and colours are bit-identical to the oracle and bit-reproducible.
#include <cfloat>

#include "mesh_common.cuh"

namespace o2345 {
namespace {

constexpr float kCosLo = O2345_PROJECT_COS_LO, kCosHi = O2345_PROJECT_COS_HI, kTauPix = O2345_PROJECT_TAU_PIX;

// Bilinear sample of channel c of a uint8 [H, W, C] image at (x, y) in [0, W-1] x [0, H-1] (pixel i's centre at i, the
// projector's align_corners=True rule), in pixel units (0 .. 255): taps nw, ne, sw, se summed in that order.  A tap past
// the last row or column has weight 0 and reads the last one instead.
__device__ __forceinline__ float bilinear(const uint8_t* __restrict__ img, int W, int H, int C, int c, float x, float y) {
  float x0 = floorf(x), y0 = floorf(y), x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f);
  float wnw = __fmul_rn(__fsub_rn(x1, x), __fsub_rn(y1, y)), wne = __fmul_rn(__fsub_rn(x, x0), __fsub_rn(y1, y));
  float wsw = __fmul_rn(__fsub_rn(x1, x), __fsub_rn(y, y0)), wse = __fmul_rn(__fsub_rn(x, x0), __fsub_rn(y, y0));
  int ix = (int)x0, iy = (int)y0, jx = min(ix + 1, W - 1), jy = min(iy + 1, H - 1);
  auto at = [&](int r, int q) { return (float)__ldg(img + ((int64_t)r * W + q) * C + c); };
  float acc = __fmul_rn(at(iy, ix), wnw);
  acc = __fadd_rn(acc, __fmul_rn(at(iy, jx), wne));
  acc = __fadd_rn(acc, __fmul_rn(at(jy, ix), wsw));
  return __fadd_rn(acc, __fmul_rn(at(jy, jx), wse));
}

__global__ void project_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, const float* __restrict__ base,
                               int64_t n, const float* __restrict__ M, float fx, float fy, float cx, float cy, float near,
                               const uint8_t* __restrict__ photo, const uint8_t* __restrict__ alpha, int W, int H,
                               const float* __restrict__ depth, int s, float* __restrict__ out, float* __restrict__ weight) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]}, q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    q[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[4 * r], p[0]), __fmul_rn(M[4 * r + 1], p[1])),
                               __fmul_rn(M[4 * r + 2], p[2])), M[4 * r + 3]);
  float w = 0.f, x = 0.f, y = 0.f;
  // a finite q.z means a finite point: an infinite coordinate gives an infinite or NaN q.z
  if (q[2] > near && q[2] <= FLT_MAX) {
    x = __fadd_rn(__fdiv_rn(__fmul_rn(fx, q[0]), q[2]), cx);
    y = __fadd_rn(__fdiv_rn(__fmul_rn(fy, q[1]), q[2]), cy);
    float nv[3] = {nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]};
    float nl = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nv[0], nv[0]), __fmul_rn(nv[1], nv[1])), __fmul_rn(nv[2], nv[2])));
    if (x >= 0.f && x <= (float)(W - 1) && y >= 0.f && y <= (float)(H - 1) && nl > 0.f && nl <= FLT_MAX) {
      float d[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {   // camera centre -R^T t, minus the point
        float ck = -__fadd_rn(__fadd_rn(__fmul_rn(M[k], M[3]), __fmul_rn(M[4 + k], M[7])), __fmul_rn(M[8 + k], M[11]));
        d[k] = __fsub_rn(ck, p[k]);
      }
      float dl = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
      float cs = __fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(nv[0], nl), __fdiv_rn(d[0], dl)),
                                     __fmul_rn(__fdiv_rn(nv[1], nl), __fdiv_rn(d[1], dl))),
                           __fmul_rn(__fdiv_rn(nv[2], nl), __fdiv_rn(d[2], dl)));
      float t = __fdiv_rn(__fsub_rn(cs, kCosLo), __fsub_rn(kCosHi, kCosLo));
      float wa = t > 0.f ? (t < 1.f ? t : 1.f) : 0.f;   // NaN -> 0
      if (wa > 0.f) {
        // image coordinate x lies in buffer pixel floor(s (x + 0.5)) of a buffer rendered with s fx, s (cx + 0.5)
        int j = min((int)floorf(__fmul_rn((float)s, __fadd_rn(x, 0.5f))), s * W - 1);
        int k = min((int)floorf(__fmul_rn((float)s, __fadd_rn(y, 0.5f))), s * H - 1);
        float D = __ldg(depth + (int64_t)k * s * W + j);
        float tau = __fdiv_rn(__fdiv_rn(__fmul_rn(kTauPix, q[2]), __fmul_rn((float)s, fx)), fmaxf(cs, kCosLo));
        if (D <= 0.f || __fsub_rn(q[2], D) <= tau) {   // the rasterizer's background (depth 0) counts as seen
          // the taps' weights may sum to 1 + ulp: the alpha is capped at 1 so the weight never exceeds it
          float a = alpha ? fminf(__fdiv_rn(bilinear(alpha, W, H, 1, 0, x, y), 255.f), 1.f) : 1.f;
          w = __fmul_rn(wa, a);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float b = base[3 * i + c];
    out[3 * i + c] = w > 0.f ? __fadd_rn(b, __fmul_rn(w, __fsub_rn(__fdiv_rn(bilinear(photo, W, H, 3, c, x, y), 255.f), b))) : b;
  }
  weight[i] = w;
}

// One thread per entry: the unit normal of face face_index[i], (B - A) x (C - A) normalised in fp64 and rounded once;
// (0, 0, 0) for an index out of range, a corner out of range or a face without area.
__global__ void face_normal_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                                   const int32_t* __restrict__ face_index, int64_t n, float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t f = face_index[i];
  int c[3] = {-1, -1, -1};
  if (f >= 0 && f < nf) c[0] = F[3 * f], c[1] = F[3 * f + 1], c[2] = F[3 * f + 2];
  D3 r = {0.0, 0.0, 0.0};
  if (face_ok(c, nv)) unit3(cross3(vert(V, c[0]), vert(V, c[1]), vert(V, c[2])), r);
  out[3 * i] = __double2float_rn(r.x), out[3 * i + 1] = __double2float_rn(r.y), out[3 * i + 2] = __double2float_rn(r.z);
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int o2345_project_view(const float* points, const float* normals, const float* base, int64_t n, const float* w2c,
                                  float fx, float fy, float cx, float cy, float near, const uint8_t* photo,
                                  const uint8_t* alpha, int W, int H, const float* depth, int scale, float* out,
                                  float* weight, o2345_stream_t stream) {
  O2345_CHECK_ARG(points && normals && base && w2c && photo && depth && out && weight,
                  "points, normals, base, w2c, photo, depth, out and weight are required");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX, "need 1 <= n <= 2^31-1");
  O2345_CHECK_ARG(W >= 1 && H >= 1 && scale >= 1 && (int64_t)scale * W <= 16384 && (int64_t)scale * H <= 16384,
                  "need W, H, scale >= 1 and scale * W, scale * H <= 16384");
  O2345_CHECK_ARG(fx > 0.f && fy > 0.f && fx <= FLT_MAX && fy <= FLT_MAX, "fx and fy must be positive and finite");
  O2345_CHECK_ARG(cx >= -FLT_MAX && cx <= FLT_MAX && cy >= -FLT_MAX && cy <= FLT_MAX, "cx and cy must be finite");
  O2345_CHECK_ARG(near > 0.f, "near must be > 0");
  cudaStream_t s = (cudaStream_t)stream;
  project_kernel<<<cdiv(n, 256), 256, 0, s>>>(points, normals, base, n, w2c, fx, fy, cx, cy, near, photo, alpha, W, H, depth,
                                              scale, out, weight);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_face_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const int32_t* face_index,
                                  int64_t n, float* normals, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && face_index && normals, "verts, faces, face_index and normals are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX, "need 1 <= n <= 2^31-1");
  cudaStream_t s = (cudaStream_t)stream;
  face_normal_kernel<<<cdiv(n, 256), 256, 0, s>>>(verts, nv, faces, nf, face_index, n, normals);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
