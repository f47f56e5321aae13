// Ambient occlusion (ops.ambient_occlusion, o2345/mesh_texture.py, run.py / simplify_mesh.py --ambient_occlusion): the share
// of fixed directions in a point's hemisphere along which the mesh is open within a distance.  The rule is in
// include/o2345.h (o2345_ambient_occlusion).
//
//   LBVH        over the occluder's faces, padded face boxes (lbvh.cuh);
//   AO         one warp per point, lane l tracing directions l, l + 32, ...: a stack traversal that stops at the first
//               face hit, the rays' misses counted per lane and summed over the warp (integers: the order is immaterial).
//
// Every float operation of the frame, the box test and the triangle test is an explicit round-to-nearest intrinsic in the
// order of the header, which oracle/ao_oracle.py repeats with numpy float32 / float64.  A node box contains the padded
// boxes of every face below it and the box test is monotone in its bounds under rounding, so the traversal skips no face
// whose own box test passes, and the result equals the oracle's search over all faces bit for bit.
#include <cfloat>

#include "lbvh.cuh"

namespace o2345 {
namespace {

enum { kErr = 0 };
constexpr float kPadScale = 0x1p-13f;   // face boxes grow by the diagonal times this (see the header)

__device__ __forceinline__ float comp(float3 v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : v.z); }

struct Ray {
  float3 p, inv;      // origin; 1 / w per axis
  bool fin[3];        // 1 / w_c is finite
  int kx, ky, kz;
  float Sx, Sy, Sz;
};

// The box test of the header on the segment [0, t_max].
__device__ __forceinline__ bool box_pass(const Ray& r, float4 lo, float4 hi, float t_max) {
  float tn = 0.f, tf = t_max;
  const float L[3] = {lo.x, lo.y, lo.z}, H[3] = {hi.x, hi.y, hi.z}, P[3] = {r.p.x, r.p.y, r.p.z}, I[3] = {r.inv.x, r.inv.y, r.inv.z};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (r.fin[c]) {
      const float t1 = __fmul_rn(__fsub_rn(L[c], P[c]), I[c]), t2 = __fmul_rn(__fsub_rn(H[c], P[c]), I[c]);
      tn = fmaxf(tn, fminf(t1, t2));
      tf = fminf(tf, fmaxf(t1, t2));
    } else if (!(L[c] <= P[c] && P[c] <= H[c])) {
      return false;
    }
  }
  return tn <= tf;
}

__device__ __forceinline__ float edge64(float ax, float by, float ay, float bx) {
  return __double2float_rn(__dsub_rn(__dmul_rn((double)ax, (double)by), __dmul_rn((double)ay, (double)bx)));
}

// The watertight ray-triangle test of Woop, Benthin and Wald (2013), without culling, on [t_min, t_max] (see the header).
__device__ __forceinline__ bool tri_hit(const Ray& r, const float* __restrict__ t9, float t_min, float t_max) {
  float3 P[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    P[j] = make_float3(__fsub_rn(__ldg(t9 + 3 * j), r.p.x), __fsub_rn(__ldg(t9 + 3 * j + 1), r.p.y),
                       __fsub_rn(__ldg(t9 + 3 * j + 2), r.p.z));
  float x[3], y[3], z[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    z[j] = comp(P[j], r.kz);
    x[j] = __fsub_rn(comp(P[j], r.kx), __fmul_rn(r.Sx, z[j]));
    y[j] = __fsub_rn(comp(P[j], r.ky), __fmul_rn(r.Sy, z[j]));
  }
  float U = __fsub_rn(__fmul_rn(x[2], y[1]), __fmul_rn(y[2], x[1]));
  float V = __fsub_rn(__fmul_rn(x[0], y[2]), __fmul_rn(y[0], x[2]));
  float W = __fsub_rn(__fmul_rn(x[1], y[0]), __fmul_rn(y[1], x[0]));
  if (U == 0.f || V == 0.f || W == 0.f) {
    U = edge64(x[2], y[1], y[2], x[1]);
    V = edge64(x[0], y[2], y[0], x[2]);
    W = edge64(x[1], y[0], y[1], x[0]);
  }
  if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) return false;
  float det = __fadd_rn(__fadd_rn(U, V), W);
  if (det == 0.f) return false;
  float T = __fadd_rn(__fadd_rn(__fmul_rn(U, __fmul_rn(r.Sz, z[0])), __fmul_rn(V, __fmul_rn(r.Sz, z[1]))),
                      __fmul_rn(W, __fmul_rn(r.Sz, z[2])));
  if (det < 0.f) T = -T, det = -det;
  return __fmul_rn(t_min, det) <= T && T <= __fmul_rn(t_max, det);
}

// any face hit on [t_min, t_max]: a stack traversal from the root that stops at the first hit
__device__ bool any_hit(const Ray& r, int64_t nf, const int2* __restrict__ child, const float4* __restrict__ box,
                        const float* __restrict__ tri, float t_min, float t_max) {
  const int first_leaf = (int)(nf - 1);
  int node = 0;
  if (!box_pass(r, __ldg(box), __ldg(box + 1), t_max)) return false;
  int stack[kLbvhStack];
  int sp = 0;
  while (true) {
    if (node >= first_leaf) {
      if (tri_hit(r, tri + 9 * (int64_t)(node - first_leaf), t_min, t_max)) return true;
    } else {
      const int2 c = __ldg(child + node);
      const bool h0 = box_pass(r, __ldg(box + 2 * c.x), __ldg(box + 2 * c.x + 1), t_max);
      const bool h1 = box_pass(r, __ldg(box + 2 * c.y), __ldg(box + 2 * c.y + 1), t_max);
      if (h0 || h1) {
        if (h0 && h1) stack[sp++] = c.y;
        node = h0 ? c.x : c.y;
        continue;
      }
    }
    if (sp == 0) return false;
    node = stack[--sp];
  }
}

// One warp per point: lane l traces directions l, l + 32, ... < k; out[i] = (misses) / k.
__global__ void __launch_bounds__(256) ao_kernel(const float* __restrict__ points, const float* __restrict__ normals,
                                                 int64_t n, const float* __restrict__ dirs, int k, float t_min, float t_max,
                                                 int64_t nf, const int2* __restrict__ child, const float4* __restrict__ box,
                                                 const float* __restrict__ tri, float* __restrict__ out) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const float px = points[3 * i], py = points[3 * i + 1], pz = points[3 * i + 2];
  const float nx = normals[3 * i], ny = normals[3 * i + 1], nz = normals[3 * i + 2];
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
  if (!(len > 0.f && len <= FLT_MAX) || !isfinite(px) || !isfinite(py) || !isfinite(pz)) {
    if (lane == 0) out[i] = 1.f;
    return;
  }
  // Duff et al. 2017
  const float ux = __fdiv_rn(nx, len), uy = __fdiv_rn(ny, len), uz = __fdiv_rn(nz, len);
  const float s = copysignf(1.f, uz);
  const float a = __fdiv_rn(-1.f, __fadd_rn(s, uz));
  const float b = __fmul_rn(__fmul_rn(ux, uy), a);
  const float3 T = make_float3(__fadd_rn(1.f, __fmul_rn(__fmul_rn(__fmul_rn(s, ux), ux), a)), __fmul_rn(s, b), -__fmul_rn(s, ux));
  const float3 B = make_float3(b, __fadd_rn(s, __fmul_rn(__fmul_rn(uy, uy), a)), -uy);
  int misses = 0;
  for (int j = lane; j < k; j += 32) {
    const float dx = dirs[3 * j], dy = dirs[3 * j + 1], dz = dirs[3 * j + 2];
    const float w[3] = {__fadd_rn(__fadd_rn(__fmul_rn(dx, T.x), __fmul_rn(dy, B.x)), __fmul_rn(dz, ux)),
                        __fadd_rn(__fadd_rn(__fmul_rn(dx, T.y), __fmul_rn(dy, B.y)), __fmul_rn(dz, uy)),
                        __fadd_rn(__fadd_rn(__fmul_rn(dx, T.z), __fmul_rn(dy, B.z)), __fmul_rn(dz, uz))};
    Ray r;
    r.p = make_float3(px, py, pz);
    float inv[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      inv[c] = __frcp_rn(w[c]);
      r.fin[c] = isfinite(inv[c]);
    }
    r.inv = make_float3(inv[0], inv[1], inv[2]);
    int kz = 0;
    if (fabsf(w[1]) > fabsf(w[0])) kz = 1;
    if (fabsf(w[2]) > fabsf(w[kz])) kz = 2;
    int kx = kz == 2 ? 0 : kz + 1, ky = kx == 2 ? 0 : kx + 1;
    if (w[kz] < 0.f) {
      const int t = kx;
      kx = ky, ky = t;
    }
    r.kx = kx, r.ky = ky, r.kz = kz;
    r.Sx = __fdiv_rn(w[kx], w[kz]);
    r.Sy = __fdiv_rn(w[ky], w[kz]);
    r.Sz = __frcp_rn(w[kz]);
    misses += !any_hit(r, nf, child, box, tri, t_min, t_max);
  }
  misses = __reduce_add_sync(0xffffffffu, misses);
  if (lane == 0) out[i] = __fdiv_rn((float)misses, (float)k);
}

__global__ void fill_one_kernel(float* __restrict__ out, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = 1.f;
}

// The scratch of o2345_ambient_occlusion, carved in this order (a Carver without a base only measures it).
struct AoScratch {
  int64_t nv, nf;
  Carver c;
  Lbvh bvh{c, nf};
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_ambient_occlusion_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 0 || nv > INT32_MAX - 1 || nf < 0 || nf > (1 << 29)) return -1;
  return AoScratch{nv, nf, {}}.c.bytes;
}

extern "C" int o2345_ambient_occlusion(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* points,
                                       const float* normals, int64_t n, const float* dirs, int k, float t_min, float t_max,
                                       void* scratch, int64_t scratch_bytes, float* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(nv >= 0 && nv <= INT32_MAX - 1 && nf >= 0 && nf <= (1 << 29) && n >= 0 && n <= INT32_MAX,
                  "need 0 <= nv < 2^31-1, 0 <= nf <= 2^29 and 0 <= n < 2^31");
  O2345_CHECK_ARG(k >= 1 && k <= (1 << 20), "need 1 <= k <= 2^20 directions");
  O2345_CHECK_ARG(t_min >= 0.f && t_min <= t_max && t_max <= FLT_MAX, "need 0 <= t_min <= t_max, both finite");
  O2345_CHECK_ARG((verts || nv == 0) && (faces || nf == 0) && (points && normals && dirs && out || n == 0),
                  "verts, faces, points, normals, dirs and out are required");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_ambient_occlusion_scratch_bytes(nv, nf),
                  "scratch smaller than o2345_ambient_occlusion_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  if (n == 0) return O2345_OK;
  cudaStream_t s = (cudaStream_t)stream;
  AoScratch S{nv, nf, {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.bvh.ctr, 0, 4 * 8, s));
  if (nv > 0 || nf > 0) {
    int32_t err = 0;
    O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.bvh.ctr + kErr, s));
    O2345_CUDA(cudaMemcpyAsync(&err, S.bvh.ctr + kErr, 4, cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    O2345_TRY(mesh_check_status(err, __func__));
  }
  if (nf == 0) {
    fill_one_kernel<<<cdiv(n, 256), 256, 0, s>>>(out, n);
    O2345_LAUNCH_CHECK();
    return O2345_OK;
  }

  O2345_TRY(S.bvh.build(verts, nv, faces, nf, kPadScale, s));
  ao_kernel<<<cdiv(n * 32, 256), 256, 0, s>>>(points, normals, n, dirs, k, t_min, t_max, nf, S.bvh.child, S.bvh.box, S.bvh.tri, out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
