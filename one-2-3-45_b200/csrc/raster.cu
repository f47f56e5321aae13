// Deterministic triangle rasterizer: many views of one mesh per call (render_eval.py, o2345/mesh_raster.py).
//
//   vertices   one thread per (view, vertex): camera space (OpenCV), projection, snap to 8 subpixel bits;
//   triangles  one thread per (view, triangle): int64 edge functions, top-left rule, one sample at every pixel centre,
//              64-bit atomicMin of (float bits of the perspective-correct camera z) << 32 | triangle id.  A triangle whose
//              clipped bounding box holds more than `split` pixels is queued and walked by a warp instead;
//   resolve    one thread per (view, pixel): the winner's perspective-correct barycentrics -> colour, alpha, depth,
//              camera-facing world normal (the face's, or its normal map's in the interpolated tangent frame), triangle id.
//
// Every float operation of the vertex, depth and resolve stages is an explicit round-to-nearest intrinsic in the order
// oracle/raster_oracle.py repeats with numpy float32 (no FMA contraction), so the triangle ids are bit-identical to the
// oracle and every output is bit-reproducible (atomicMin does not depend on arrival order).
#include "common.cuh"

namespace o2345 {
namespace {

constexpr int kSub = 256;                    // 8 subpixel bits
constexpr float kMaxFixed = 536870912.0f;    // |fixed coordinate| < 2^29: edge functions stay below 2^61
constexpr int kInvalid = INT32_MIN;          // vertex at z <= near or projecting outside the fixed-point range
constexpr int kDefaultSplit = 64;            // tools/time_raster.py: bbox pixels above which a warp takes the triangle

int g_split = 0;

struct Tri {
  int64_t x[3], y[3], area;
  float r[3];   // 1 / camera z of the vertex in each slot
  int idx[3];   // mesh vertex of each slot (slots 1 and 2 are swapped for a clockwise triangle)
};

// Loads and orients triangle t of view v; false if it is dropped (bad index, vertex behind near / out of range, zero area).
__device__ __forceinline__ bool tri_setup(const int32_t* __restrict__ faces, int64_t nv, int64_t t, int v,
                                          const int2* __restrict__ xy, const float* __restrict__ zc, Tri& T) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int i = __ldg(faces + 3 * t + k);
    if (i < 0 || i >= nv) return false;
    int64_t g = (int64_t)v * nv + i;
    int2 p = xy[g];
    if (p.x == kInvalid) return false;
    T.x[k] = p.x, T.y[k] = p.y, T.r[k] = __fdiv_rn(1.0f, zc[g]), T.idx[k] = i;
  }
  int64_t a = (T.x[1] - T.x[0]) * (T.y[2] - T.y[0]) - (T.y[1] - T.y[0]) * (T.x[2] - T.x[0]);
  if (a == 0) return false;
  if (a < 0) {
    int64_t tx = T.x[1], ty = T.y[1];
    float tr = T.r[1];
    int ti = T.idx[1];
    T.x[1] = T.x[2], T.y[1] = T.y[2], T.r[1] = T.r[2], T.idx[1] = T.idx[2];
    T.x[2] = tx, T.y[2] = ty, T.r[2] = tr, T.idx[2] = ti;
    a = -a;
  }
  T.area = a;
  return true;
}

// Edge function of edge a->b at (sx, sy); positive inside a counter-clockwise (area > 0) triangle of the y-down frame.
__device__ __forceinline__ int64_t edge(int64_t xa, int64_t ya, int64_t xb, int64_t yb, int64_t sx, int64_t sy) {
  return (xb - xa) * (sy - ya) - (yb - ya) * (sx - xa);
}

// Top-left rule: an edge owns the samples on it iff it is a left edge (dy < 0) or a top edge (dy == 0, dx > 0).
__device__ __forceinline__ bool covers(int64_t w, int64_t xa, int64_t ya, int64_t xb, int64_t yb) {
  return w > 0 || (w == 0 && (yb - ya < 0 || (yb == ya && xb - xa > 0)));
}

// Barycentric weights of pixel (px, py) (w[k]: edge opposite slot k) and whether the pixel centre is covered.
__device__ __forceinline__ bool tri_weights(const Tri& T, int px, int py, int64_t w[3]) {
  int64_t sx = (int64_t)px * kSub + kSub / 2, sy = (int64_t)py * kSub + kSub / 2;
  w[0] = edge(T.x[1], T.y[1], T.x[2], T.y[2], sx, sy);
  w[1] = edge(T.x[2], T.y[2], T.x[0], T.y[0], sx, sy);
  w[2] = edge(T.x[0], T.y[0], T.x[1], T.y[1], sx, sy);
  return covers(w[0], T.x[1], T.y[1], T.x[2], T.y[2]) && covers(w[1], T.x[2], T.y[2], T.x[0], T.y[0]) &&
         covers(w[2], T.x[0], T.y[0], T.x[1], T.y[1]);
}

// Screen barycentrics b = w / area, interpolated 1/z, camera z = 1 / (1/z).
__device__ __forceinline__ float tri_depth(const Tri& T, const int64_t w[3], float b[3], float& iz) {
  float fa = __ll2float_rn(T.area);
#pragma unroll
  for (int k = 0; k < 3; ++k) b[k] = __fdiv_rn(__ll2float_rn(w[k]), fa);
  iz = __fadd_rn(__fadd_rn(__fmul_rn(b[0], T.r[0]), __fmul_rn(b[1], T.r[1])), __fmul_rn(b[2], T.r[2]));
  return __fdiv_rn(1.0f, iz);
}

// Pixel range [lo, hi] of the centres inside fixed-point [a, b] (centre of pixel i: 256 i + 128), clipped to [0, n).
__device__ __forceinline__ void span(int64_t a, int64_t b, int n, int& lo, int& hi) {
  int64_t l = (a - kSub / 2 + kSub - 1) >> 8, h = (b - kSub / 2) >> 8;
  lo = (int)max(l, (int64_t)0), hi = (int)min(h, (int64_t)n - 1);
}

__device__ __forceinline__ void bbox(const Tri& T, int W, int H, int& x0, int& x1, int& y0, int& y1) {
  span(min(T.x[0], min(T.x[1], T.x[2])), max(T.x[0], max(T.x[1], T.x[2])), W, x0, x1);
  span(min(T.y[0], min(T.y[1], T.y[2])), max(T.y[0], max(T.y[1], T.y[2])), H, y0, y1);
}

__device__ __forceinline__ void shade_pixel(const Tri& T, int px, int py, uint32_t id, unsigned long long* zrow) {
  int64_t w[3];
  if (!tri_weights(T, px, py, w)) return;
  float b[3], iz;
  float z = tri_depth(T, w, b, iz);
  atomicMin(zrow + px, ((unsigned long long)__float_as_uint(z) << 32) | id);
}

__global__ void raster_vertices_kernel(const float* __restrict__ verts, int64_t nv, int V, const float* __restrict__ w2c,
                                       const float* __restrict__ intr, float near, int2* __restrict__ xy,
                                       float* __restrict__ zc) {
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (int64_t)V * nv) return;
  int v = (int)(g / nv);
  int64_t i = g - (int64_t)v * nv;
  const float* M = w2c + 12 * v;
  float p[3] = {verts[3 * i], verts[3 * i + 1], verts[3 * i + 2]}, c[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    c[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[4 * r], p[0]), __fmul_rn(M[4 * r + 1], p[1])),
                               __fmul_rn(M[4 * r + 2], p[2])), M[4 * r + 3]);
  const float* K = intr + 4 * v;   // fx fy cx cy
  float sx = __fmul_rn(__fadd_rn(__fdiv_rn(__fmul_rn(K[0], c[0]), c[2]), K[2]), (float)kSub);
  float sy = __fmul_rn(__fadd_rn(__fdiv_rn(__fmul_rn(K[1], c[1]), c[2]), K[3]), (float)kSub);
  bool ok = c[2] > near && fabsf(sx) < kMaxFixed && fabsf(sy) < kMaxFixed;   // NaN fails every comparison
  xy[g] = ok ? make_int2(__float2int_rn(sx), __float2int_rn(sy)) : make_int2(kInvalid, kInvalid);
  zc[g] = c[2];
}

__global__ void raster_triangles_kernel(const int32_t* __restrict__ faces, int64_t nv, int64_t nf, int V, int W, int H,
                                        const int2* __restrict__ xy, const float* __restrict__ zc, int split,
                                        unsigned long long* __restrict__ zbuf, int64_t* __restrict__ queue, int64_t qcap,
                                        int* __restrict__ qcount) {
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (int64_t)V * nf) return;
  int v = (int)(g / nf);
  int64_t t = g - (int64_t)v * nf;
  Tri T;
  if (!tri_setup(faces, nv, t, v, xy, zc, T)) return;
  int x0, x1, y0, y1;
  bbox(T, W, H, x0, x1, y0, y1);
  if (x0 > x1 || y0 > y1) return;
  if ((int64_t)(x1 - x0 + 1) * (y1 - y0 + 1) > split) {
    int slot = atomicAdd(qcount, 1);
    if (slot < qcap) {
      queue[slot] = g;
      return;
    }   // queue full: this thread walks the triangle itself (same result, atomicMin is order-free)
  }
  for (int py = y0; py <= y1; ++py) {
    unsigned long long* zrow = zbuf + ((int64_t)v * H + py) * W;
    for (int px = x0; px <= x1; ++px) shade_pixel(T, px, py, (uint32_t)t, zrow);
  }
}

// One warp per queued triangle; the lanes stride over its bounding box.
__global__ void raster_big_kernel(const int32_t* __restrict__ faces, int64_t nv, int64_t nf, int W, int H,
                                  const int2* __restrict__ xy, const float* __restrict__ zc,
                                  unsigned long long* __restrict__ zbuf, const int64_t* __restrict__ queue, int64_t qcap,
                                  const int* __restrict__ qcount) {
  int lane = threadIdx.x & 31;
  int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  int64_t n = min((int64_t)*qcount, qcap);
  for (int64_t q = warp; q < n; q += nwarps) {
    int64_t g = queue[q];
    int v = (int)(g / nf);
    int64_t t = g - (int64_t)v * nf;
    Tri T;
    if (!tri_setup(faces, nv, t, v, xy, zc, T)) continue;
    int x0, x1, y0, y1;
    bbox(T, W, H, x0, x1, y0, y1);
    int bw = x1 - x0 + 1;
    int64_t cnt = (int64_t)bw * (y1 - y0 + 1);
    for (int64_t k = lane; k < cnt; k += 32) {
      int py = y0 + (int)(k / bw), px = x0 + (int)(k % bw);
      shade_pixel(T, px, py, (uint32_t)t, zbuf + ((int64_t)v * H + py) * W);
    }
  }
}

__device__ __forceinline__ int wrap(int i, int n, int mode) {
  if (mode == 1) return min(max(i, 0), n - 1);
  if (mode == 2) {
    int m = ((i % (2 * n)) + 2 * n) % (2 * n);
    return m < n ? m : 2 * n - 1 - m;
  }
  return ((i % n) + n) % n;
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) {
  return __fadd_rn(__fmul_rn(a, __fsub_rn(1.0f, t)), __fmul_rn(b, t));
}

// Bilinear sample of texture `tex` at uv (glTF: texel centres at (i + 0.5) / w, v down), RGB in [0, 1].
__device__ void sample_texture(const uint8_t* __restrict__ texels, const int32_t* __restrict__ info, float u, float v,
                               float rgb[3]) {
  int64_t base = info[0];
  int w = info[1], h = info[2];
  float fx = fminf(fmaxf(__fsub_rn(__fmul_rn(u, (float)w), 0.5f), -16777216.0f), 16777216.0f);
  float fy = fminf(fmaxf(__fsub_rn(__fmul_rn(v, (float)h), 0.5f), -16777216.0f), 16777216.0f);
  float flx = floorf(fx), fly = floorf(fy);
  float ax = __fsub_rn(fx, flx), ay = __fsub_rn(fy, fly);
  int ix = (int)flx, iy = (int)fly;
  int xa = wrap(ix, w, info[3]), xb = wrap(ix + 1, w, info[3]), ya = wrap(iy, h, info[4]), yb = wrap(iy + 1, h, info[4]);
  const uint8_t* t00 = texels + 4 * (base + (int64_t)ya * w + xa);
  const uint8_t* t10 = texels + 4 * (base + (int64_t)ya * w + xb);
  const uint8_t* t01 = texels + 4 * (base + (int64_t)yb * w + xa);
  const uint8_t* t11 = texels + 4 * (base + (int64_t)yb * w + xb);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float top = lerp_rn(__fdiv_rn((float)t00[c], 255.0f), __fdiv_rn((float)t10[c], 255.0f), ax);
    float bot = lerp_rn(__fdiv_rn((float)t01[c], 255.0f), __fdiv_rn((float)t11[c], 255.0f), ax);
    rgb[c] = lerp_rn(top, bot, ay);
  }
}

__device__ __forceinline__ float interp(const float p[3], float a, float b, float c) {
  return __fadd_rn(__fadd_rn(__fmul_rn(p[0], a), __fmul_rn(p[1], b)), __fmul_rn(p[2], c));
}

// v := v / |v| in fp32; false (v unchanged) when |v| is not a positive finite number
__device__ __forceinline__ bool normalize3(float v[3]) {
  float l = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
  if (!(l > 0.f && l < INFINITY)) return false;
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(v[c], l);
  return true;
}

// The normal-mapped normal at perspective-correct weights p: N = normalize(interpolated normal), T = normalize(interpolated
// tangent xyz), B = (N x T) * w (w the sign of the interpolated tangent w), t = 2 * texel - 1, n = normalize((t.x T +
// t.y B) + t.z N).  False when N, T or n has no direction (the face normal is kept).
__device__ bool mapped_normal(const o2345_raster_mesh& m, const float p[3], int i0, int i1, int i2, int ntex, float u,
                              float v, float n[3]) {
  float N[3], T[3], t[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    N[c] = interp(p, m.normals[3 * i0 + c], m.normals[3 * i1 + c], m.normals[3 * i2 + c]);
    T[c] = interp(p, m.tangents[4 * i0 + c], m.tangents[4 * i1 + c], m.tangents[4 * i2 + c]);
  }
  if (!normalize3(N) || !normalize3(T)) return false;
  float w = interp(p, m.tangents[4 * i0 + 3], m.tangents[4 * i1 + 3], m.tangents[4 * i2 + 3]) < 0.f ? -1.f : 1.f;
  float B[3] = {__fmul_rn(__fsub_rn(__fmul_rn(N[1], T[2]), __fmul_rn(N[2], T[1])), w),
                __fmul_rn(__fsub_rn(__fmul_rn(N[2], T[0]), __fmul_rn(N[0], T[2])), w),
                __fmul_rn(__fsub_rn(__fmul_rn(N[0], T[1]), __fmul_rn(N[1], T[0])), w)};
  sample_texture(m.texels, m.tex_info + 5 * ntex, u, v, t);
#pragma unroll
  for (int c = 0; c < 3; ++c) t[c] = __fsub_rn(__fmul_rn(2.0f, t[c]), 1.0f);
#pragma unroll
  for (int c = 0; c < 3; ++c) n[c] = __fadd_rn(__fadd_rn(__fmul_rn(t[0], T[c]), __fmul_rn(t[1], B[c])), __fmul_rn(t[2], N[c]));
  return normalize3(n);
}

__global__ void raster_resolve_kernel(o2345_raster_mesh m, int V, const float* __restrict__ w2c, int W, int H,
                                      const int2* __restrict__ xy, const float* __restrict__ zc, int shading,
                                      const unsigned long long* __restrict__ zbuf, float* __restrict__ color,
                                      float* __restrict__ alpha, float* __restrict__ depth, float* __restrict__ normal,
                                      int32_t* __restrict__ tri) {
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t hw = (int64_t)H * W;
  if (g >= (int64_t)V * hw) return;
  int v = (int)(g / hw);
  int64_t pix = g - (int64_t)v * hw;
  int py = (int)(pix / W), px = (int)(pix % W);
  unsigned long long key = zbuf[g];
  float rgb[3] = {0.f, 0.f, 0.f}, nrm[3] = {0.f, 0.f, 0.f}, a = 0.f, z = 0.f;
  int32_t id = -1;
  Tri T;
  if (key != ~0ull && tri_setup(m.faces, m.nv, (int64_t)(uint32_t)key, v, xy, zc, T)) {
    id = (int32_t)(uint32_t)key;
    z = __uint_as_float((uint32_t)(key >> 32));
    a = 1.f;
    int64_t w[3];
    tri_weights(T, px, py, w);
    float b[3], iz, p[3];
    tri_depth(T, w, b, iz);
#pragma unroll
    for (int k = 0; k < 3; ++k) p[k] = __fdiv_rn(__fmul_rn(b[k], T.r[k]), iz);
    const int i0 = T.idx[0], i1 = T.idx[1], i2 = T.idx[2];
    if (m.colors) {
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = interp(p, m.colors[3 * i0 + c], m.colors[3 * i1 + c], m.colors[3 * i2 + c]);
    } else {
      rgb[0] = rgb[1] = rgb[2] = 1.f;
    }
    int tex = m.face_tex ? m.face_tex[id] : -1;
    int ntex = m.face_ntex && m.normals && m.tangents ? m.face_ntex[id] : -1;
    float u = 0.f, vv = 0.f;
    if ((tex >= 0 && tex < m.n_tex) || (ntex >= 0 && ntex < m.n_tex)) {
      u = interp(p, m.uvs[2 * i0], m.uvs[2 * i1], m.uvs[2 * i2]);
      vv = interp(p, m.uvs[2 * i0 + 1], m.uvs[2 * i1 + 1], m.uvs[2 * i2 + 1]);
    }
    if (tex >= 0 && tex < m.n_tex) {
      float t[3];
      sample_texture(m.texels, m.tex_info + 5 * tex, u, vv, t);
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = __fmul_rn(rgb[c], t[c]);
    }
    // world-space face normal, turned toward the camera centre C = -R^T t
    const float* P0 = m.verts + 3 * i0;
    const float* P1 = m.verts + 3 * i1;
    const float* P2 = m.verts + 3 * i2;
    float e1[3], e2[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) e1[c] = __fsub_rn(P1[c], P0[c]), e2[c] = __fsub_rn(P2[c], P0[c]);
    float n[3] = {__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1])),
                  __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2])),
                  __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]))};
    float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
    const float* M = w2c + 12 * v;
    float face = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float cc = -__fadd_rn(__fadd_rn(__fmul_rn(M[c], M[3]), __fmul_rn(M[4 + c], M[7])), __fmul_rn(M[8 + c], M[11]));
      face = __fadd_rn(face, __fmul_rn(n[c], __fsub_rn(cc, P0[c])));
    }
    float s = len > 0.f ? (face < 0.f ? -1.f : 1.f) : 0.f;
    float nm[3];
    if (len > 0.f && ntex >= 0 && ntex < m.n_tex && mapped_normal(m, p, i0, i1, i2, ntex, u, vv, nm)) {
      // s turns the slot-ordered normal toward the camera; the map's normal takes the sign of the face's own winding
      float sf = i1 == m.faces[3 * (int64_t)id + 1] ? s : -s;
#pragma unroll
      for (int c = 0; c < 3; ++c) nrm[c] = __fmul_rn(sf, nm[c]);
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) nrm[c] = len > 0.f ? __fdiv_rn(__fmul_rn(s, n[c]), len) : 0.f;
    }
    if (shading == O2345_SHADE_LAMBERT) {
      float l = __fadd_rn(0.4f, __fmul_rn(0.6f, fmaxf(nrm[2], 0.f)));
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = __fmul_rn(rgb[c], l);
    }
  }
  if (color) color[3 * g] = rgb[0], color[3 * g + 1] = rgb[1], color[3 * g + 2] = rgb[2];
  if (normal) normal[3 * g] = nrm[0], normal[3 * g + 1] = nrm[1], normal[3 * g + 2] = nrm[2];
  if (alpha) alpha[g] = a;
  if (depth) depth[g] = z;
  if (tri) tri[g] = id;
}

int64_t queue_cap(int64_t nf, int V) { return min((int64_t)V * nf, (int64_t)1 << 22); }

// The scratch of o2345_raster, carved in this order (a Carver without a base only measures it).
struct Scratch {
  int64_t npix, nvv, qcap;   // V * H * W, V * nv, queue_cap
  Carver c;
  unsigned long long* zbuf = c.take<unsigned long long>(npix);
  int2* xy = c.take<int2>(nvv);
  int64_t* queue = c.take<int64_t>(qcap);
  float* zc = c.take<float>(nvv);
  int* qcount = c.take<int>(1);
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_raster_scratch_bytes(int64_t nv, int64_t nf, int V, int W, int H) {
  if (nv < 0 || nf < 0 || V < 1 || W < 1 || H < 1) return -1;
  return Scratch{(int64_t)V * H * W, (int64_t)V * nv, queue_cap(nf, V), {}}.c.bytes;
}

extern "C" void o2345_debug_raster_split(int pixels) { g_split = pixels > 0 ? pixels : 0; }

extern "C" int o2345_raster(const o2345_raster_mesh* mesh, int V, const float* w2c, const float* intr, int W, int H,
                            float near, int shading, void* scratch, int64_t scratch_bytes, float* color, float* alpha,
                            float* depth, float* normal, int32_t* tri, o2345_stream_t stream) {
  O2345_CHECK_ARG(mesh && mesh->verts && mesh->faces, "mesh, its vertices and its faces are required");
  const o2345_raster_mesh& m = *mesh;
  O2345_CHECK_ARG(m.nv >= 1 && m.nv <= INT32_MAX && m.nf >= 0 && m.nf <= INT32_MAX - 1,
                  "need 1 <= nv <= 2^31-1 and 0 <= nf < 2^31-1");
  O2345_CHECK_ARG(V >= 1 && W >= 1 && H >= 1 && W <= 16384 && H <= 16384, "need V >= 1 and 1 <= W, H <= 16384");
  O2345_CHECK_ARG(w2c && intr, "w2c [V,3,4] and intr [V,4] are required");
  O2345_CHECK_ARG(near > 0.f, "near must be > 0");
  O2345_CHECK_ARG(shading == O2345_SHADE_UNLIT || shading == O2345_SHADE_LAMBERT, "unknown shading mode");
  O2345_CHECK_ARG(!m.face_tex || (m.uvs && m.texels && m.tex_info && m.n_tex >= 1), "face_tex needs uvs, texels and tex_info");
  O2345_CHECK_ARG(!m.face_ntex || (m.uvs && m.texels && m.tex_info && m.n_tex >= 1), "face_ntex needs uvs, texels and tex_info");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_raster_scratch_bytes(m.nv, m.nf, V, W, H),
                  "scratch smaller than o2345_raster_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");   // 64-bit atomics, int2 stores
  cudaStream_t s = (cudaStream_t)stream;
  Scratch S{(int64_t)V * H * W, (int64_t)V * m.nv, queue_cap(m.nf, V), {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.zbuf, 0xff, 8 * S.npix, s));
  O2345_CUDA(cudaMemsetAsync(S.qcount, 0, sizeof(int), s));
  raster_vertices_kernel<<<cdiv(S.nvv, 256), 256, 0, s>>>(m.verts, m.nv, V, w2c, intr, near, S.xy, S.zc);
  O2345_LAUNCH_CHECK();
  if (m.nf > 0) {
    raster_triangles_kernel<<<cdiv((int64_t)V * m.nf, 256), 256, 0, s>>>(m.faces, m.nv, m.nf, V, W, H, S.xy, S.zc,
                                                                         g_split ? g_split : kDefaultSplit, S.zbuf, S.queue,
                                                                         S.qcap, S.qcount);
    O2345_LAUNCH_CHECK();
    raster_big_kernel<<<sm_count() * 8, 256, 0, s>>>(m.faces, m.nv, m.nf, W, H, S.xy, S.zc, S.zbuf, S.queue, S.qcap, S.qcount);
    O2345_LAUNCH_CHECK();
  }
  raster_resolve_kernel<<<cdiv(S.npix, 256), 256, 0, s>>>(m, V, w2c, W, H, S.xy, S.zc, shading, S.zbuf, color, alpha, depth,
                                                          normal, tri);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
