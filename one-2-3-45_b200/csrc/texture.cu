// Texture baking (ops.texture_atlas / texel_points / texture_fill / transfer_colors / tangent_normals / normal_quantise /
// vertex_normals, o2345/mesh_texture.py): one isometric chart per face, packed on shelves into an N x N atlas, the surface
// point behind every texel of a chart, push-pull fill of the texels no chart owns, the colour of a point taken from the
// nearest face of a source mesh, and normal maps: world normals in each face's tangent frame, quantised to uint8.
//
//   atlas         one thread per face: the chart (base = the longest edge by fp32 squared length, first on ties; L, d, h in
//                 fp64 rounded once to fp32) and L * h in fp64; the sum of L * h in a fixed order (cumsum_f64_chunked, scan.cu:
//                 sequential inside chunks of 1024 faces, then over the chunk totals); rho0 = sqrt(0.5 N^2 / sum) on the host;
//                 per trial of the ladder rho_j = rho0 * j / 64 (a binary search over j in [1, 256]): the boxes (one
//                 thread per face) and next-fit shelf packing in one warp (stable counting sort by height descending, then
//                 the shelves in sorted order, 32 boxes per step through shuffles); the fit flag is read on the host;
//                 finally the uv of every corner (one thread per face) and the owner map (one block per box);
//   texel points  ordered compaction of the owned texels (o2345_compact), one thread per owned texel: the closest point of
//                 its chart's triangle to the texel centre (the 7-region test in fp64) and the surface point it maps to;
//   fill          the owned texels' colours scattered into the texture, a pull pyramid of weighted 2 x 2 means and a push
//                 pass that hands every empty texel its parent's value;
//   transfer      one thread per point: the closest point of the source face behind the point's nearest surface sample
//                 and the face's vertex colours interpolated there;
//   tangent       one thread per owned texel: the face's frame (T, B, N) from its corners and uv in fp64 and the world
//                 normal's coordinates in it; quantise: one thread per texel, renormalised in fp32 and coded to uint8;
//   vertex normal vertex -> face adjacency (vertex_faces, mesh_common.cu), then one thread per vertex: the sum of its
//                 faces' (B - A) x (C - A) in ascending face order in fp64, normalised, rounded once to fp32.
//   chart atlas   multi-face charts (include/o2345.h): per face its normal's dominant axis and sign and the projected
//                 corners; edges of two faces through vertex_faces; components by hooking; per round the chart buckets,
//                 extents, the pairwise separating-axis test inside each chart and the median cut of overlapping charts;
//                 then the same boxes, shelves and ladder as the atlas, uv, and the owner by 64-bit atomicMin of
//                 (fp32 squared distance, face) over each face's grown uv box.
//
// Every floating-point operation is an explicit round-to-nearest intrinsic in the order oracle/texture_oracle.py repeats
// with numpy (no FMA contraction), so every output is bit-identical to the oracle and independent of thread scheduling.
#include <math.h>

#include "mesh_common.cuh"

namespace o2345 {
namespace {

constexpr int kPad = 2;        // texels of padding on every side of a chart's box
constexpr int kMinN = 64, kMaxN = 8192;
constexpr int kRungs = 256, kRungDen = 64;   // rho_j = rho0 * j / 64, j in [1, 256]
enum { kErr = 0, kFits = 1, kChanged = 2, kFlagged = 3, kCtr = 4 };

// The corner that starts the longest edge of the three (v0v1, v1v2, v2v0) by fp32 squared length, the first on ties.
__device__ __forceinline__ int base_corner(const float* __restrict__ V, const int c[3]) {
  float best = -1.f;
  int k0 = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = V + 3 * (int64_t)c[k];
    const float* q = V + 3 * (int64_t)c[(k + 1) % 3];
    float dx = __fsub_rn(__ldg(q), __ldg(p)), dy = __fsub_rn(__ldg(q + 1), __ldg(p + 1)), dz = __fsub_rn(__ldg(q + 2), __ldg(p + 2));
    float l2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    if (l2 > best) best = l2, k0 = k;
  }
  return k0;
}

// (la * A + lb * B) + lc * C per component in fp32, the weights rounded to fp32 first
__device__ __forceinline__ void blend3(const Bary& l, const float* A, const float* B, const float* C, float* out) {
  float la = __double2float_rn(l.a), lb = __double2float_rn(l.b), lc = __double2float_rn(l.c);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = __fadd_rn(__fadd_rn(__fmul_rn(la, A[k]), __fmul_rn(lb, B[k])), __fmul_rn(lc, C[k]));
}

// ----------------------------------------------------------------------------- atlas
// chart[f] = (L, d, h, base corner bits), lh[f] = L * h in fp64 (exact: two fp32 factors)
__global__ void chart_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                             float4* __restrict__ chart, double* __restrict__ lh) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  int c[3] = {F[3 * f], F[3 * f + 1], F[3 * f + 2]};
  if (!face_ok(c, nv)) {   // refused on the host
    chart[f] = make_float4(0.f, 0.f, 0.f, 0.f), lh[f] = 0.0;
    return;
  }
  int k0 = base_corner(V, c);
  D3 a = vert(V, c[k0]), b = vert(V, c[(k0 + 1) % 3]), q = vert(V, c[(k0 + 2) % 3]);
  D3 e1 = sub3(b, a), e2 = sub3(q, a);
  double L = __dsqrt_rn(dot3(e1, e1)), d = 0.0, h = 0.0;
  if (L > 0.0) {
    D3 n = cross3(a, b, q);
    d = __ddiv_rn(dot3(e2, e1), L);
    h = __ddiv_rn(__dsqrt_rn(dot3(n, n)), L);
  }
  float Lf = __double2float_rn(L), df = __double2float_rn(d), hf = __double2float_rn(h);
  df = fminf(fmaxf(df, 0.f), Lf);   // 0 <= d <= L up to rounding: clamped so the chart stays inside its box
  chart[f] = make_float4(Lf, df, hf, __int_as_float(k0));
  lh[f] = __dmul_rn((double)Lf, (double)hf);
}

// box side of a chart extent e at scale rho: ceil(e * rho) + 2P (anything wider than N is N + 1: it cannot fit)
__device__ __forceinline__ int box_side(float e, double rho, int N) {
  double s = ceil(__dmul_rn((double)e, rho));
  return s > (double)N ? N + 1 : (int)s + 2 * kPad;
}

// boxes[f] = (x, y, w, hgt): w and hgt at scale rho (x and y come from the packing)
__global__ void box_kernel(const float4* __restrict__ chart, int64_t nf, double rho, int N, int32_t* __restrict__ boxes) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  float4 ch = chart[f];
  boxes[4 * f + 2] = box_side(ch.x, rho, N);
  boxes[4 * f + 3] = box_side(ch.z, rho, N);
}

// One warp.  Stable counting sort of the boxes by height descending (order), then next-fit shelves: a box goes at the
// cursor unless it would cross x = N, in which case a new shelf opens below the tallest box (the first) of the current
// one.  *fits = every box lies inside N x N; boxes[f].x, .y are written up to the first box that does not fit.
__global__ void __launch_bounds__(32) pack_kernel(int32_t* __restrict__ boxes, int nf, int N, int32_t* __restrict__ order,
                                                  int32_t* __restrict__ fits) {
  __shared__ int start[kMaxN + 2];
  const int lane = threadIdx.x;
  for (int i = lane; i <= N; i += 32) start[i] = 0;
  __syncwarp();
  bool over = false;
  for (int f = lane; f < nf; f += 32) {
    int w = boxes[4 * f + 2], h = boxes[4 * f + 3];
    if (w > N || h > N) over = true;
    else atomicAdd(start + h, 1);
  }
  __syncwarp();
  if (__any_sync(0xffffffffu, over)) {
    if (lane == 0) *fits = 0;
    return;
  }
  // exclusive start of every height, heights descending: lane l scans the rank chunk [l c, (l + 1) c) of r = N - h
  const int c = (N + 1 + 31) / 32, r0 = min(lane * c, N + 1), r1 = min(r0 + c, N + 1);
  int sum = 0;
  for (int r = r0; r < r1; ++r) sum += start[N - r];
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  __syncwarp();
  int run = incl - sum;
  for (int r = r0; r < r1; ++r) {
    int n = start[N - r];
    start[N - r] = run;
    run += n;
  }
  __syncwarp();
  const unsigned lt = (1u << lane) - 1u;
  for (int base = 0; base < nf; base += 32) {   // scatter in face order: stable
    int f = base + lane;
    int h = f < nf ? boxes[4 * f + 3] : -1;
    unsigned m = __match_any_sync(0xffffffffu, h);
    int pos = f < nf ? start[h] + __popc(m & lt) : 0;
    __syncwarp();
    if (f < nf) {
      order[pos] = f;
      if (lane == 31 - __clz(m)) start[h] += __popc(m);
    }
    __syncwarp();
  }
  int cx = 0, cy = 0, sh = 0;
  bool ok = true;
  for (int base = 0; base < nf && ok; base += 32) {
    int i = base + lane, f = i < nf ? order[i] : 0;
    int w = i < nf ? boxes[4 * f + 2] : 0, h = i < nf ? boxes[4 * f + 3] : 0, x = 0, y = 0;
    int n = min(32, nf - base);
    for (int k = 0; k < n; ++k) {
      int wk = __shfl_sync(0xffffffffu, w, k), hk = __shfl_sync(0xffffffffu, h, k);
      if (cx > 0 && cx + wk > N) cy += sh, cx = 0, sh = 0;
      if (cx + wk > N || cy + hk > N) {
        ok = false;
        n = k;
        break;
      }
      if (lane == k) x = cx, y = cy;
      cx += wk, sh = max(sh, hk);
    }
    if (lane < n) boxes[4 * f] = x, boxes[4 * f + 1] = y;
  }
  if (lane == 0) *fits = ok ? 1 : 0;
}

// uv[f][k] of corner k: a at (x + P, y + P), b at (x + P + L rho, y + P), c at (x + P + d rho, y + P + h rho), / N
__global__ void uv_kernel(const int32_t* __restrict__ F, const float4* __restrict__ chart, const int32_t* __restrict__ boxes,
                          int64_t nf, double rho, int N, float* __restrict__ uv) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  float4 ch = chart[f];
  int k0 = __float_as_int(ch.w);
  double x = (double)(boxes[4 * f] + kPad), y = (double)(boxes[4 * f + 1] + kPad), n = (double)N;
  double px[3] = {x, __dadd_rn(x, __dmul_rn((double)ch.x, rho)), __dadd_rn(x, __dmul_rn((double)ch.y, rho))};
  double py[3] = {y, y, __dadd_rn(y, __dmul_rn((double)ch.z, rho))};
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    int k = (k0 + j) % 3;
    uv[6 * f + 2 * k] = __double2float_rn(__ddiv_rn(px[j], n));
    uv[6 * f + 2 * k + 1] = __double2float_rn(__ddiv_rn(py[j], n));
  }
}

// one block per face: owner[texel] = f for every texel of its box
__global__ void owner_kernel(const int32_t* __restrict__ boxes, int N, int32_t* __restrict__ owner) {
  const int f = blockIdx.x;
  const int x = boxes[4 * f], y = boxes[4 * f + 1], w = boxes[4 * f + 2], h = boxes[4 * f + 3];
  for (int t = threadIdx.x; t < w * h; t += blockDim.x) owner[(int64_t)(y + t / w) * N + x + t % w] = f;
}

// The scratch of o2345_texture_atlas, carved in this order (a Carver without a base only measures it).
struct AtlasScratch {
  int64_t nf;
  Carver c;
  float4* chart = c.take<float4>(nf);
  double* lh = c.take<double>(nf);
  double* tot = c.take<double>(sum_chunks(nf) + 1);
  int32_t* order = c.take<int32_t>(nf);
  int32_t* ctr = c.take<int32_t>(kCtr);
};

bool valid_size(int N) { return N >= kMinN && N <= kMaxN && (N & (N - 1)) == 0; }

// The scratch of o2345_texel_points: the owned flags and the compaction's scratch.
struct TexelScratch {
  int64_t n;
  Carver c;
  uint8_t* flags = c.take<uint8_t>(n);
  int32_t* cscratch = c.take<int32_t>(o2345_compact_scratch_ints(n));
};

// The scratch of o2345_texture_fill: the push-pull levels N/2 .. 1 (rgb, weight), finest first.
struct FillScratch {
  Carver c;
  float4* lvl[16];
  int levels = 0;
  FillScratch(char* base, int N) : c{base} {
    for (int m = N / 2; m >= 1; m /= 2) lvl[levels++] = c.take<float4>((int64_t)m * m);
  }
};

// ----------------------------------------------------------------------------- texel points
__global__ void owned_kernel(const int32_t* __restrict__ owner, int64_t n, uint8_t* __restrict__ flags) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = owner[i] >= 0;
}

// One thread per owned texel (the compacted list): the chart's triangle is its face's uv times N (exact), the base corner
// as in chart_kernel; the closest point of it to the texel centre maps to la A + lb B + lc C.
__global__ void texel_points_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                                    const float* __restrict__ uv, const int32_t* __restrict__ owner, int N,
                                    const int32_t* __restrict__ texel_index, const int32_t* __restrict__ count,
                                    float* __restrict__ points, int32_t* __restrict__ texel_face) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  int t = texel_index[i], f = owner[t];
  texel_face[i] = f;
  int c[3] = {-1, -1, -1};
  if (f >= 0 && f < nf) c[0] = F[3 * (int64_t)f], c[1] = F[3 * (int64_t)f + 1], c[2] = F[3 * (int64_t)f + 2];
  if (!face_ok(c, nv)) {   // not a face the atlas accepted
    points[3 * i] = points[3 * i + 1] = points[3 * i + 2] = __int_as_float(0x7fc00000);
    return;
  }
  int k0 = base_corner(V, c);
  int ka = k0, kb = (k0 + 1) % 3, kc = (k0 + 2) % 3;
  const float n = (float)N;
  auto corner = [&](int k) {
    return D3{(double)__fmul_rn(uv[6 * (int64_t)f + 2 * k], n), (double)__fmul_rn(uv[6 * (int64_t)f + 2 * k + 1], n), 0.0};
  };
  D3 q = {__dadd_rn((double)(t % N), 0.5), __dadd_rn((double)(t / N), 0.5), 0.0};
  Bary l = closest_point(q, corner(ka), corner(kb), corner(kc));
  blend3(l, V + 3 * (int64_t)c[ka], V + 3 * (int64_t)c[kb], V + 3 * (int64_t)c[kc], points + 3 * i);
}

// ----------------------------------------------------------------------------- fill
__global__ void scatter_kernel(const int32_t* __restrict__ texel_index, const int32_t* __restrict__ count,
                               const float* __restrict__ rgb, float* __restrict__ tex) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  int64_t t = texel_index[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) tex[3 * t + k] = rgb[3 * i + k];
}

// level n (n x n, rgb + weight) from its 2n x 2n children: weights summed, rgb the weight-normalised mean (0 without
// weight).  The finest children are the texture itself with weight 1 where owned.
__device__ __forceinline__ float4 child(const float4* __restrict__ lvl, const float* __restrict__ tex,
                                        const int32_t* __restrict__ owner, int64_t j) {
  if (lvl) return lvl[j];
  return make_float4(tex[3 * j], tex[3 * j + 1], tex[3 * j + 2], owner[j] >= 0 ? 1.f : 0.f);
}

__global__ void pull_kernel(const float4* __restrict__ fine, const float* __restrict__ tex, const int32_t* __restrict__ owner,
                            int n, float4* __restrict__ coarse) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * n) return;
  int64_t y = i / n, x = i % n, w2 = 2 * (int64_t)n;
  float4 c[4] = {child(fine, tex, owner, 2 * y * w2 + 2 * x), child(fine, tex, owner, 2 * y * w2 + 2 * x + 1),
                 child(fine, tex, owner, (2 * y + 1) * w2 + 2 * x), child(fine, tex, owner, (2 * y + 1) * w2 + 2 * x + 1)};
  float sw = __fadd_rn(__fadd_rn(__fadd_rn(c[0].w, c[1].w), c[2].w), c[3].w);
  float4 o = make_float4(0.f, 0.f, 0.f, sw);
  if (sw > 0.f) {
    float s[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float v0 = k == 0 ? c[0].x : k == 1 ? c[0].y : c[0].z, v1 = k == 0 ? c[1].x : k == 1 ? c[1].y : c[1].z;
      float v2 = k == 0 ? c[2].x : k == 1 ? c[2].y : c[2].z, v3 = k == 0 ? c[3].x : k == 1 ? c[3].y : c[3].z;
      s[k] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c[0].w, v0), __fmul_rn(c[1].w, v1)), __fmul_rn(c[2].w, v2)),
                                 __fmul_rn(c[3].w, v3)),
                       sw);
    }
    o.x = s[0], o.y = s[1], o.z = s[2];
  }
  coarse[i] = o;
}

// every empty texel of an n x n level (the texture itself when lvl is null) takes its parent's rgb
__global__ void push_kernel(float4* __restrict__ lvl, float* __restrict__ tex, const int32_t* __restrict__ owner, int n,
                            const float4* __restrict__ parent) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * n) return;
  float4 p = parent[(i / n / 2) * (n / 2) + (i % n) / 2];
  if (lvl) {
    if (lvl[i].w == 0.f) lvl[i] = make_float4(p.x, p.y, p.z, 0.f);
  } else if (owner[i] < 0) {
    tex[3 * i] = p.x, tex[3 * i + 1] = p.y, tex[3 * i + 2] = p.z;
  }
}

// ----------------------------------------------------------------------------- transfer
__global__ void transfer_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                                const float* __restrict__ colors, const float* __restrict__ pts, int64_t n,
                                const int32_t* __restrict__ nn_index, const int32_t* __restrict__ sample_face,
                                int64_t n_samples, float* __restrict__ rgb) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int s = nn_index[i], f = s >= 0 && s < n_samples ? sample_face[s] : -1;
  int c[3] = {-1, -1, -1};
  if (f >= 0 && f < nf) c[0] = F[3 * (int64_t)f], c[1] = F[3 * (int64_t)f + 1], c[2] = F[3 * (int64_t)f + 2];
  if (!face_ok(c, nv)) {
    rgb[3 * i] = rgb[3 * i + 1] = rgb[3 * i + 2] = __int_as_float(0x7fc00000);
    return;
  }
  D3 p = {(double)pts[3 * i], (double)pts[3 * i + 1], (double)pts[3 * i + 2]};
  Bary l = closest_point(p, vert(V, c[0]), vert(V, c[1]), vert(V, c[2]));
  blend3(l, colors + 3 * (int64_t)c[0], colors + 3 * (int64_t)c[1], colors + 3 * (int64_t)c[2], rgb + 3 * i);
}

// ----------------------------------------------------------------------------- normal maps
__device__ __forceinline__ D3 scale3(D3 a, double s) { return {__dmul_rn(a.x, s), __dmul_rn(a.y, s), __dmul_rn(a.z, s)}; }

// One thread per texel: the tangent-space coordinates of world normal nw[i] in the frame of face texel_face[i] (rule in
// include/o2345.h): T = dp/du, B = -dp/dv, N = e1 x e2, each normalised; (0, 0, 1) for a degenerate face or a zero or
// non-finite normal, NaN for a face index out of range.  kDecoded: B = w (N x T), w = sign((N x T) . -dp/dv) (+1 on 0),
// the frame a decoder builds from NORMAL and TANGENT (T, w) when dp/du and dp/dv are not orthogonal.
template <bool kDecoded>
__global__ void tangent_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                               const float* __restrict__ uv, const int32_t* __restrict__ texel_face,
                               const float* __restrict__ nw, int64_t n, float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t f = texel_face[i];
  int c[3] = {-1, -1, -1};
  if (f >= 0 && f < nf) c[0] = F[3 * f], c[1] = F[3 * f + 1], c[2] = F[3 * f + 2];
  if (!face_ok(c, nv)) {
    out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = __int_as_float(0x7fc00000);
    return;
  }
  float t[3] = {0.f, 0.f, 1.f};
  D3 P0 = vert(V, c[0]), P1 = vert(V, c[1]), P2 = vert(V, c[2]), e1 = sub3(P1, P0), e2 = sub3(P2, P0);
  const float* q = uv + 6 * f;
  double du1 = __dsub_rn((double)q[2], (double)q[0]), dv1 = __dsub_rn((double)q[3], (double)q[1]);
  double du2 = __dsub_rn((double)q[4], (double)q[0]), dv2 = __dsub_rn((double)q[5], (double)q[1]);
  double det = __dsub_rn(__dmul_rn(du1, dv2), __dmul_rn(du2, dv1));
  D3 w = {(double)nw[3 * i], (double)nw[3 * i + 1], (double)nw[3 * i + 2]};
  double ln = __dsqrt_rn(dot3(w, w));
  D3 T, B, N;
  if (fabs(det) > 0.0 && ln > 0.0 && ln < INFINITY) {
    D3 dpdu = sub3(scale3(e1, dv2), scale3(e2, dv1)), dpdv = sub3(scale3(e2, du1), scale3(e1, du2));
    dpdu = {__ddiv_rn(dpdu.x, det), __ddiv_rn(dpdu.y, det), __ddiv_rn(dpdu.z, det)};
    dpdv = {__ddiv_rn(-dpdv.x, det), __ddiv_rn(-dpdv.y, det), __ddiv_rn(-dpdv.z, det)};
    bool ok = unit3(dpdu, T) && unit3(dpdv, B) && unit3(cross3(P0, P1, P2), N);
    if (kDecoded && ok) {
      D3 C = cross3({0.0, 0.0, 0.0}, N, T);   // N x T
      B = dot3(C, dpdv) < 0.0 ? D3{-C.x, -C.y, -C.z} : C;
    }
    if (ok) {
      t[0] = __double2float_rn(__ddiv_rn(dot3(w, T), ln));
      t[1] = __double2float_rn(__ddiv_rn(dot3(w, B), ln));
      t[2] = __double2float_rn(__ddiv_rn(dot3(w, N), ln));
    }
  }
  out[3 * i] = t[0], out[3 * i + 1] = t[1], out[3 * i + 2] = t[2];
}

// One thread per texel: v / |v| in fp32 ((0, 0, 1) when |v| is zero or not finite), each component coded as
// round_half_even((c + 1) * 127.5).
__global__ void quantise_kernel(const float* __restrict__ tex, int64_t n, uint8_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v[3] = {tex[3 * i], tex[3 * i + 1], tex[3 * i + 2]};
  float l = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
  bool ok = l > 0.f && l < INFINITY;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float c = ok ? __fdiv_rn(v[k], l) : (k == 2 ? 1.f : 0.f);
    int b = __float2int_rn(__fmul_rn(__fadd_rn(c, 1.f), 127.5f));
    out[3 * i + k] = (uint8_t)min(max(b, 0), 255);
  }
}

// One thread per vertex: the sum of its faces' (B - A) x (C - A) in ascending face order (fp64), normalised, rounded to
// fp32; (0, 0, 0) for a zero sum.
__global__ void vertex_normal_kernel(const float* __restrict__ V, const int32_t* __restrict__ F,
                                     const int32_t* __restrict__ off, const int32_t* __restrict__ adj, int64_t nv,
                                     float* __restrict__ out) {
  int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  D3 r = vertex_normal(V, F, adj + off[u], off[u + 1] - off[u]);
  out[3 * u] = __double2float_rn(r.x), out[3 * u + 1] = __double2float_rn(r.y), out[3 * u + 2] = __double2float_rn(r.z);
}

// The scratch of o2345_vertex_normals, carved in this order (a Carver without a base only measures it).
struct NormalScratch {
  int64_t nv, nf;
  Carver c;
  int32_t* off = c.take<int32_t>(nv + 1);
  int32_t* sums = c.take<int32_t>(scan_blocks(nv + 1));
  int32_t* cursor = c.take<int32_t>(nv);
  int32_t* adj = c.take<int32_t>(3 * nf);
  int32_t* err = c.take<int32_t>(1);
};

// ----------------------------------------------------------------------------- chart atlas
constexpr int kOwnLabel = 6;   // a face with a zero or non-finite normal: a chart of its own

// (b - a) x (p - a) in 2D, fp64: (bx - ax)(py - ay) - (by - ay)(px - ax)
__device__ __forceinline__ double orient2(double ax, double ay, double bx, double by, double px, double py) {
  return __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(py, ay)), __dmul_rn(__dsub_rn(by, ay), __dsub_rn(px, ax)));
}

// Separating-axis test of two projected triangles p, q (u0 v0 u1 v1 u2 v2): true when their interiors share a point.
// Axis k of a triangle t is its edge t_k t_k+1; s = orient(t_k, t_k+1, t_k+2) and the other triangle's three orients
// o_j; they are separated when max o_j <= min(0, s) or min o_j >= max(0, s) (touching does not count).  A triangle of
// zero area has no interior.
__device__ bool tri_overlap(const float* p, const float* q) {
  const float* t[2] = {p, q};
  for (int side = 0; side < 2; ++side) {
    const float* a = t[side];
    const float* b = t[1 - side];
    if (orient2(a[0], a[1], a[2], a[3], a[4], a[5]) == 0.0) return false;
    for (int k = 0; k < 3; ++k) {
      int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
      double ax = a[2 * k], ay = a[2 * k + 1], bx = a[2 * k1], by = a[2 * k1 + 1];
      double s = orient2(ax, ay, bx, by, a[2 * k2], a[2 * k2 + 1]);
      double lo = fmin(0.0, s), hi = fmax(0.0, s), omin = INFINITY, omax = -INFINITY;
      for (int j = 0; j < 3; ++j) {
        double o = orient2(ax, ay, bx, by, b[2 * j], b[2 * j + 1]);
        omin = fmin(omin, o), omax = fmax(omax, o);
      }
      if (omax <= lo || omin >= hi) return false;
    }
  }
  return true;
}

// One thread per face: n = (P1 - P0) x (P2 - P0) in fp64; axis a = the largest |n_a| (the lower axis on ties), label
// 2a + (n_a < 0), or kOwnLabel for a zero or non-finite n; projection (u, v) = (p[a+1], p[a+2]) (axes mod 3), u negated
// when n_a < 0, so every face of a label has positive uv area.  An own-label face projects along z.  key: the label,
// kOwnLabel + f for an own-label face (no face shares it).
__global__ void label_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                             int32_t* __restrict__ label, float* __restrict__ puv, int32_t* __restrict__ key) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  int c[3] = {F[3 * f], F[3 * f + 1], F[3 * f + 2]};
  D3 n = cross3(vert(V, c[0]), vert(V, c[1]), vert(V, c[2]));
  int a = 0;
  double na = n.x;
  if (fabs(n.y) > fabs(na)) a = 1, na = n.y;
  if (fabs(n.z) > fabs(na)) a = 2, na = n.z;
  bool ok = fabs(na) > 0.0 && isfinite(n.x) && isfinite(n.y) && isfinite(n.z);
  if (!ok) a = 2;
  bool neg = ok && na < 0.0;
  int lab = ok ? 2 * a + (neg ? 1 : 0) : kOwnLabel;
  label[f] = lab;
  key[f] = ok ? lab : kOwnLabel + (int32_t)f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = V + 3 * (int64_t)c[k];
    float u = p[(a + 1) % 3], v = p[(a + 2) % 3];
    puv[6 * f + 2 * k] = neg ? -u : u;
    puv[6 * f + 2 * k + 1] = v;
  }
}

// One thread per face edge (a, b) = (c_k, c_k+1): the edge's uses are the (face, edge) slots of any face with the same
// unordered pair (a != b), found through a's face list; nbr[3f + k] = the other face when there are exactly two uses
// and they belong to two faces, else -1 (boundary, non-manifold and degenerate edges cut).
__global__ void edge_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ off,
                            const int32_t* __restrict__ adj, int32_t* __restrict__ nbr) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * nf) return;
  const int64_t f = i / 3;
  const int k = (int)(i % 3);
  const int a = F[i], b = F[3 * f + (k + 1) % 3];
  int uses = 0, other = -1;
  if (a != b) {
    for (int j = off[a]; j < off[a + 1]; ++j) {
      int g = adj[j];
      if (j > off[a] && adj[j - 1] == g) continue;   // a face that holds a twice is listed twice
      for (int kk = 0; kk < 3; ++kk) {
        int x = F[3 * (int64_t)g + kk], y = F[3 * (int64_t)g + (kk + 1) % 3];
        if ((x == a && y == b) || (x == b && y == a)) {
          ++uses;
          if (g != f) other = g;
        }
      }
    }
  }
  nbr[i] = uses == 2 && other >= 0 ? other : -1;
}

// One thread per face: every neighbour g > f with the same key is joined with f (unite, mesh_common.cuh: each component
// ends rooted at its least face).
__global__ void hook_kernel(const int32_t* __restrict__ nbr, const int32_t* __restrict__ key, int64_t nf,
                            int32_t* parent, int32_t* __restrict__ changed) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int kf = key[f];
  for (int k = 0; k < 3; ++k) {
    int g = nbr[3 * f + k];
    if (g <= f || key[g] != kf) continue;
    unite(parent, (int)f, g, changed);
  }
}

// Chart buckets: cnt[root] counts its faces, then (after the scan) list[off[root] ..) holds them in scheduling order;
// every consumer of a bucket is independent of that order.  root flags for the ordered list of charts.
__global__ void bucket_count_kernel(const int32_t* __restrict__ parent, int64_t nf, int32_t* __restrict__ cnt,
                                    uint8_t* __restrict__ is_root) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  atomicAdd(cnt + parent[f], 1);
  is_root[f] = parent[f] == f;
}

__global__ void bucket_fill_kernel(const int32_t* __restrict__ parent, int64_t nf, const int32_t* __restrict__ off,
                                   int32_t* __restrict__ cursor, int32_t* __restrict__ list) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  int r = parent[f];
  list[off[r] + atomicAdd(cursor + r, 1)] = (int32_t)f;
}

// One block per chart i (root roots[i]): lo[i] = (min u, min v) of its corners; ext[i] = (max - min) in fp64 rounded up
// to fp32 in .x (u) and .z (v), the layout box_kernel reads; area[i] = ext_u ext_v in fp64.
__global__ void __launch_bounds__(128) extent_kernel(const int32_t* __restrict__ roots, const int32_t* __restrict__ off,
                                                     const int32_t* __restrict__ list, const float* __restrict__ puv,
                                                     float2* __restrict__ lo, float4* __restrict__ ext,
                                                     double* __restrict__ area) {
  __shared__ float red[4][128];
  const int r = roots[blockIdx.x];
  float m[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};   // min u, min v, max u, max v
  for (int j = off[r] + threadIdx.x; j < off[r + 1]; j += blockDim.x) {
    const float* p = puv + 6 * (int64_t)list[j];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      m[0] = fminf(m[0], p[2 * k]), m[1] = fminf(m[1], p[2 * k + 1]);
      m[2] = fmaxf(m[2], p[2 * k]), m[3] = fmaxf(m[3], p[2 * k + 1]);
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) red[q][threadIdx.x] = m[q];
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      red[0][threadIdx.x] = fminf(red[0][threadIdx.x], red[0][threadIdx.x + s]);
      red[1][threadIdx.x] = fminf(red[1][threadIdx.x], red[1][threadIdx.x + s]);
      red[2][threadIdx.x] = fmaxf(red[2][threadIdx.x], red[2][threadIdx.x + s]);
      red[3][threadIdx.x] = fmaxf(red[3][threadIdx.x], red[3][threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float eu = __double2float_ru(__dsub_rn((double)red[2][0], (double)red[0][0]));
    float ev = __double2float_ru(__dsub_rn((double)red[3][0], (double)red[1][0]));
    lo[blockIdx.x] = make_float2(red[0][0], red[1][0]);
    ext[blockIdx.x] = make_float4(eu, 0.f, ev, 0.f);
    area[blockIdx.x] = __dmul_rn((double)eu, (double)ev);
  }
}

// One thread per face f: the faces g > f of its chart are tested against it (uv boxes that overlap with positive area,
// then tri_overlap); any overlap flags the chart (flag[root] = 1, *any = 1).  A thread stops once its chart is flagged.
__global__ void overlap_kernel(const float* __restrict__ puv, const int32_t* __restrict__ parent, int64_t nf,
                               const int32_t* __restrict__ off, const int32_t* __restrict__ list, uint8_t* flag,
                               int32_t* __restrict__ any) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int r = parent[f];
  if (off[r + 1] - off[r] < 2) return;
  float p[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) p[k] = puv[6 * f + k];
  const float u0 = fminf(fminf(p[0], p[2]), p[4]), u1 = fmaxf(fmaxf(p[0], p[2]), p[4]);
  const float v0 = fminf(fminf(p[1], p[3]), p[5]), v1 = fmaxf(fmaxf(p[1], p[3]), p[5]);
  volatile uint8_t* vflag = flag;
  for (int j = off[r]; j < off[r + 1]; ++j) {
    if ((j & 63) == 0 && vflag[r]) return;
    int g = list[j];
    if (g <= f) continue;
    const float* q = puv + 6 * (int64_t)g;
    if (fmaxf(fmaxf(q[0], q[2]), q[4]) <= u0 || fminf(fminf(q[0], q[2]), q[4]) >= u1 ||
        fmaxf(fmaxf(q[1], q[3]), q[5]) <= v0 || fminf(fminf(q[1], q[3]), q[5]) >= v1)
      continue;
    float t[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) t[k] = q[k];
    if (tri_overlap(p, t)) {
      vflag[r] = 1;
      *any = 1;
      return;
    }
  }
}

// One thread per face: the key of the next round.  A face of a flagged chart of m faces is ranked by its centroid
// coordinate c = (x0 + x1) + x2 (fp64) along the chart's longer extent (u on ties), ties by face index; the first m / 2
// go to side 0, the rest to side 1.  key = 2 root + side (side 0 for a chart that was not flagged).
__global__ void cut_kernel(const float* __restrict__ puv, const int32_t* __restrict__ parent, int64_t nf,
                           const int32_t* __restrict__ off, const int32_t* __restrict__ list, const int32_t* __restrict__ pos,
                           const float4* __restrict__ ext, const uint8_t* __restrict__ flag, int32_t* __restrict__ key) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int r = parent[f];
  int side = 0;
  if (flag[r]) {
    float4 e = ext[pos[r]];
    const int ax = e.x >= e.z ? 0 : 1;
    auto centroid = [&](int64_t g) {
      const float* q = puv + 6 * g + ax;
      return __dadd_rn(__dadd_rn((double)q[0], (double)q[2]), (double)q[4]);
    };
    const double cf = centroid(f);
    int rank = 0;
    for (int j = off[r]; j < off[r + 1]; ++j) {
      int g = list[j];
      double cg = centroid(g);
      rank += cg < cf || (cg == cf && g < f);
    }
    side = rank >= (off[r + 1] - off[r]) / 2;
  }
  key[f] = 2 * r + side;
}

// One thread per face: uv of corner k = (box origin + P + (p_k - chart min) rho) / N in fp64, rounded to fp32; boxes[f]
// = its chart's box; chart[f] = its chart's id (least face).
__global__ void chart_uv_kernel(const float* __restrict__ puv, const int32_t* __restrict__ parent, int64_t nf,
                                const int32_t* __restrict__ pos, const float2* __restrict__ lo,
                                const int32_t* __restrict__ cboxes, double rho, int N, float* __restrict__ uv,
                                int32_t* __restrict__ boxes, int32_t* __restrict__ chart) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int r = parent[f], i = pos[r];
  const int32_t* b = cboxes + 4 * (int64_t)i;
  const double x = (double)(b[0] + kPad), y = (double)(b[1] + kPad), n = (double)N;
  const float2 m = lo[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double u = __dadd_rn(x, __dmul_rn(__dsub_rn((double)puv[6 * f + 2 * k], (double)m.x), rho));
    double v = __dadd_rn(y, __dmul_rn(__dsub_rn((double)puv[6 * f + 2 * k + 1], (double)m.y), rho));
    uv[6 * f + 2 * k] = __double2float_rn(__ddiv_rn(u, n));
    uv[6 * f + 2 * k + 1] = __double2float_rn(__ddiv_rn(v, n));
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) boxes[4 * f + k] = b[k];
  chart[f] = r;
}

// Squared distance (fp64) of q to the triangle abc: 0 when q lies inside or on it (orients of the three edges all >= 0
// or all <= 0, the triangle of non-zero area), else |q - ((la a + lb b) + lc c)|^2 with the 7-region barycentrics.
__device__ __forceinline__ double tri_dist2(D3 q, D3 a, D3 b, D3 c) {
  double w0 = orient2(b.x, b.y, c.x, c.y, q.x, q.y), w1 = orient2(c.x, c.y, a.x, a.y, q.x, q.y);
  double w2 = orient2(a.x, a.y, b.x, b.y, q.x, q.y), ar = orient2(a.x, a.y, b.x, b.y, c.x, c.y);
  if (ar != 0.0 && ((w0 >= 0.0 && w1 >= 0.0 && w2 >= 0.0) || (w0 <= 0.0 && w1 <= 0.0 && w2 <= 0.0))) return 0.0;
  Bary l = closest_point(q, a, b, c);
  double x = __dadd_rn(__dadd_rn(__dmul_rn(l.a, a.x), __dmul_rn(l.b, b.x)), __dmul_rn(l.c, c.x));
  double y = __dadd_rn(__dadd_rn(__dmul_rn(l.a, a.y), __dmul_rn(l.b, b.y)), __dmul_rn(l.c, c.y));
  double dx = __dsub_rn(q.x, x), dy = __dsub_rn(q.y, y);
  return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
}

// One block per face: every texel of its chart's box whose centre lies in the face's uv bounding box (uv * N in fp32)
// grown by P: key = (fp32 of tri_dist2) << 32 | f, the least kept by a 64-bit atomicMin.
__global__ void chart_owner_kernel(const float* __restrict__ uv, const int32_t* __restrict__ boxes, int N,
                                   unsigned long long* __restrict__ keys) {
  const int64_t f = blockIdx.x;
  const float n = (float)N;
  D3 t[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    t[k] = {(double)__fmul_rn(uv[6 * f + 2 * k], n), (double)__fmul_rn(uv[6 * f + 2 * k + 1], n), 0.0};
  const int bx = boxes[4 * f], by = boxes[4 * f + 1], bw = boxes[4 * f + 2], bh = boxes[4 * f + 3];
  const double g = (double)kPad + 0.5;
  const int x0 = max(bx, (int)ceil(__dsub_rn(fmin(fmin(t[0].x, t[1].x), t[2].x), g)));
  const int x1 = min(bx + bw - 1, (int)floor(__dadd_rn(fmax(fmax(t[0].x, t[1].x), t[2].x), (double)kPad - 0.5)));
  const int y0 = max(by, (int)ceil(__dsub_rn(fmin(fmin(t[0].y, t[1].y), t[2].y), g)));
  const int y1 = min(by + bh - 1, (int)floor(__dadd_rn(fmax(fmax(t[0].y, t[1].y), t[2].y), (double)kPad - 0.5)));
  const int w = x1 - x0 + 1, h = y1 - y0 + 1;
  if (w <= 0 || h <= 0) return;
  for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
    const int tx = x0 + i % w, ty = y0 + i / w;
    D3 q = {__dadd_rn((double)tx, 0.5), __dadd_rn((double)ty, 0.5), 0.0};
    float d = __double2float_rn(tri_dist2(q, t[0], t[1], t[2]));
    atomicMin(keys + (int64_t)ty * N + tx, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)f);
  }
}

__global__ void owner_from_keys_kernel(const unsigned long long* __restrict__ keys, int64_t n, int32_t* __restrict__ owner) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long k = keys[i];
  owner[i] = k == ~0ull ? -1 : (int32_t)(k & 0xffffffffull);
}

// The scratch of o2345_chart_atlas, carved in this order (a Carver without a base only measures it).
struct ChartScratch {
  int64_t nv, nf, N;
  Carver c;
  int32_t* ctr = c.take<int32_t>(kCtr);
  float* puv = c.take<float>(6 * nf);
  int32_t* key = c.take<int32_t>(nf);
  int32_t* nbr = c.take<int32_t>(3 * nf);
  int32_t* voff = c.take<int32_t>(nv + 1);            // vertex -> face adjacency (edge_kernel)
  int32_t* vsums = c.take<int32_t>(scan_blocks(nv + 1));
  int32_t* vcursor = c.take<int32_t>(nv);
  int32_t* vadj = c.take<int32_t>(3 * nf);
  int32_t* parent = c.take<int32_t>(nf);
  int32_t* off = c.take<int32_t>(nf + 1);             // chart buckets
  int32_t* sums = c.take<int32_t>(scan_blocks(nf + 1));
  int32_t* cursor = c.take<int32_t>(nf);
  int32_t* list = c.take<int32_t>(nf);
  uint8_t* is_root = c.take<uint8_t>(nf);
  uint8_t* flag = c.take<uint8_t>(nf);
  int32_t* roots = c.take<int32_t>(nf);
  int32_t* pos = c.take<int32_t>(nf);
  int32_t* count = c.take<int32_t>(1);
  int32_t* cscratch = c.take<int32_t>(o2345_compact_scratch_ints(nf));
  float2* lo = c.take<float2>(nf);
  float4* ext = c.take<float4>(nf);
  double* area = c.take<double>(nf);
  double* tot = c.take<double>(sum_chunks(nf) + 1);
  int32_t* cboxes = c.take<int32_t>(4 * nf);
  int32_t* order = c.take<int32_t>(nf);
  unsigned long long* keys = c.take<unsigned long long>(N * N);
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_texture_atlas_scratch_bytes(int64_t nf) {
  if (nf < 1 || nf > INT32_MAX / 3) return -1;
  return AtlasScratch{nf, {}}.c.bytes;
}

extern "C" int o2345_texture_atlas(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int N, void* scratch,
                                   int64_t scratch_bytes, float* uv, int32_t* boxes, int32_t* owner, int32_t* rung_host,
                                   double* rho_host, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && uv && boxes && owner, "verts, faces, uv, boxes and owner are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(valid_size(N), "N must be a power of two in [64, 8192]");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_texture_atlas_scratch_bytes(nf),
                  "scratch smaller than o2345_texture_atlas_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  AtlasScratch S{nf, {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.ctr, 0, 4 * kCtr, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.ctr + kErr, s));
  chart_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, nv, faces, nf, S.chart, S.lh);
  O2345_LAUNCH_CHECK();
  O2345_TRY(cumsum_f64_chunked(S.lh, nf, S.tot, s));   // lh becomes its prefix sums: only the total is used
  int32_t err = 0;
  double sum = 0.0;   // host reads: the input checks and the sum, then one fit flag per trial
  O2345_CUDA(cudaMemcpyAsync(&err, S.ctr + kErr, 4, cudaMemcpyDeviceToHost, s));
  O2345_CUDA(cudaMemcpyAsync(&sum, S.tot + sum_chunks(nf), 8, cudaMemcpyDeviceToHost, s));
  O2345_CUDA(cudaStreamSynchronize(s));
  O2345_TRY(mesh_check_status(err, __func__));
  if (!(sum > 0.0)) {
    set_error("%s: the faces have no area", __func__);
    return O2345_EINVAL;
  }
  const double rho0 = sqrt(0.5 * ((double)N * (double)N) / sum);
  auto rho_of = [&](int j) { return rho0 * (double)j / (double)kRungDen; };
  auto trial = [&](int j, int32_t& fits) {
    box_kernel<<<cdiv(nf, 256), 256, 0, s>>>(S.chart, nf, rho_of(j), N, boxes);
    pack_kernel<<<1, 32, 0, s>>>(boxes, (int)nf, N, S.order, S.ctr + kFits);
    O2345_LAUNCH_CHECK();
    O2345_CUDA(cudaMemcpyAsync(&fits, S.ctr + kFits, 4, cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };
  int32_t fits = 0;
  O2345_TRY(trial(1, fits));
  if (!fits) {
    set_error("%s: %d^2 texels cannot hold %lld charts", __func__, N, (long long)nf);
    return O2345_EINVAL;
  }
  int lo = 1, hi = kRungs + 1, last = 1;
  while (hi - lo > 1) {
    int mid = (lo + hi) / 2;
    O2345_TRY(trial(mid, fits));
    last = mid;
    if (fits) lo = mid;
    else hi = mid;
  }
  if (last != lo) O2345_TRY(trial(lo, fits));   // the boxes of the chosen rung
  const double rho = rho_of(lo);
  uv_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, S.chart, boxes, nf, rho, N, uv);
  O2345_CUDA(cudaMemsetAsync(owner, 0xff, 4 * (int64_t)N * N, s));
  owner_kernel<<<(unsigned)nf, 128, 0, s>>>(boxes, N, owner);
  O2345_LAUNCH_CHECK();
  if (rung_host) *rung_host = lo;
  if (rho_host) *rho_host = rho;
  return O2345_OK;
}

extern "C" int64_t o2345_texel_points_scratch_bytes(int N) {
  if (!valid_size(N)) return -1;
  return TexelScratch{(int64_t)N * N, {}}.c.bytes;
}

extern "C" int o2345_texel_points(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                                  const int32_t* owner, int N, void* scratch, int64_t scratch_bytes, int32_t* texel_index,
                                  float* points, int32_t* texel_face, int32_t* count, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && uv && owner && texel_index && points && texel_face && count,
                  "verts, faces, uv, owner, texel_index, points, texel_face and count are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(valid_size(N), "N must be a power of two in [64, 8192]");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_texel_points_scratch_bytes(N), "scratch smaller than o2345_texel_points_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = (int64_t)N * N;
  TexelScratch S{n, {(char*)scratch}};
  owned_kernel<<<cdiv(n, 256), 256, 0, s>>>(owner, n, S.flags);
  O2345_LAUNCH_CHECK();
  O2345_TRY(o2345_compact(S.flags, n, texel_index, nullptr, count, S.cscratch, stream));
  texel_points_kernel<<<cdiv(n, 128), 128, 0, s>>>(verts, nv, faces, nf, uv, owner, N, texel_index, count, points, texel_face);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int64_t o2345_texture_fill_scratch_bytes(int N) {
  if (!valid_size(N)) return -1;
  return FillScratch(nullptr, N).c.bytes;
}

extern "C" int o2345_texture_fill(const int32_t* texel_index, const int32_t* count, const float* rgb, const int32_t* owner,
                                  int N, void* scratch, int64_t scratch_bytes, float* texture, o2345_stream_t stream) {
  O2345_CHECK_ARG(texel_index && count && rgb && owner && texture, "texel_index, count, rgb, owner and texture are required");
  O2345_CHECK_ARG(valid_size(N), "N must be a power of two in [64, 8192]");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_texture_fill_scratch_bytes(N), "scratch smaller than o2345_texture_fill_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = (int64_t)N * N;
  FillScratch S((char*)scratch, N);
  O2345_CUDA(cudaMemsetAsync(texture, 0, 12 * n, s));
  scatter_kernel<<<cdiv(n, 256), 256, 0, s>>>(texel_index, count, rgb, texture);
  for (int l = 0; l < S.levels; ++l) {   // pull: level l + 1 of the pyramid (N >> (l + 1) texels a side)
    int m = N >> (l + 1);
    pull_kernel<<<cdiv((int64_t)m * m, 256), 256, 0, s>>>(l ? S.lvl[l - 1] : nullptr, texture, owner, m, S.lvl[l]);
  }
  for (int l = S.levels - 2; l >= -1; --l) {   // push: coarse to fine, the texture last
    int m = N >> (l + 1);
    push_kernel<<<cdiv((int64_t)m * m, 256), 256, 0, s>>>(l >= 0 ? S.lvl[l] : nullptr, texture, owner, m, S.lvl[l + 1]);
  }
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_transfer_colors(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* colors,
                                     const float* points, int64_t n, const int32_t* nn_index, const int32_t* sample_face,
                                     int64_t n_samples, float* rgb, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && colors && points && nn_index && sample_face && rgb,
                  "verts, faces, colors, points, nn_index, sample_face and rgb are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX && n_samples >= 1 && n_samples <= INT32_MAX, "need 1 <= n, n_samples <= 2^31-1");
  cudaStream_t s = (cudaStream_t)stream;
  transfer_kernel<<<cdiv(n, 128), 128, 0, s>>>(verts, nv, faces, nf, colors, points, n, nn_index, sample_face, n_samples, rgb);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_tangent_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                                     const int32_t* texel_face, const float* normals, int64_t n, float* out,
                                     o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && uv && texel_face && normals && out, "verts, faces, uv, texel_face, normals and out are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX, "need 1 <= n <= 2^31-1");
  cudaStream_t s = (cudaStream_t)stream;
  tangent_kernel<false><<<cdiv(n, 128), 128, 0, s>>>(verts, nv, faces, nf, uv, texel_face, normals, n, out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_tangent_normals_decoded(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                                             const int32_t* texel_face, const float* normals, int64_t n, float* out,
                                             o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && uv && texel_face && normals && out, "verts, faces, uv, texel_face, normals and out are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv <= 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX, "need 1 <= n <= 2^31-1");
  cudaStream_t s = (cudaStream_t)stream;
  tangent_kernel<true><<<cdiv(n, 128), 128, 0, s>>>(verts, nv, faces, nf, uv, texel_face, normals, n, out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_normal_quantise(const float* texture, int64_t n, uint8_t* out, o2345_stream_t stream) {
  O2345_CHECK_ARG(texture && out, "texture and out are required");
  O2345_CHECK_ARG(n >= 1 && n <= (int64_t)kMaxN * kMaxN, "need 1 <= n <= 8192^2");
  cudaStream_t s = (cudaStream_t)stream;
  quantise_kernel<<<cdiv(n, 256), 256, 0, s>>>(texture, n, out);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int64_t o2345_vertex_normals_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 1 || nv > INT32_MAX - 1 || nf < 1 || nf > INT32_MAX / 3) return -1;
  return NormalScratch{nv, nf, {}}.c.bytes;
}

extern "C" int o2345_vertex_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, void* scratch,
                                    int64_t scratch_bytes, float* normals, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && normals, "verts, faces and normals are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX - 1 && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv < 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_vertex_normals_scratch_bytes(nv, nf),
                  "scratch smaller than o2345_vertex_normals_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  NormalScratch S{nv, nf, {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.err, 0, 4, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.err, s));
  int32_t err = 0;   // the adjacency scatters through the face indices: they are checked on the host first
  O2345_CUDA(cudaMemcpyAsync(&err, S.err, 4, cudaMemcpyDeviceToHost, s));
  O2345_CUDA(cudaStreamSynchronize(s));
  O2345_TRY(mesh_check_status(err, __func__));
  O2345_TRY(vertex_faces(faces, nf, nv, S.off, S.sums, S.cursor, S.adj, s));
  vertex_normal_kernel<<<cdiv(nv, 128), 128, 0, s>>>(verts, faces, S.off, S.adj, nv, normals);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int64_t o2345_chart_atlas_scratch_bytes(int64_t nv, int64_t nf, int N) {
  if (nv < 1 || nv > INT32_MAX - 1 || nf < 1 || nf > INT32_MAX / 3 || !valid_size(N)) return -1;
  return ChartScratch{nv, nf, N, {}}.c.bytes;
}

extern "C" int o2345_chart_atlas(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int N, void* scratch,
                                 int64_t scratch_bytes, float* uv, int32_t* boxes, int32_t* owner, int32_t* labels,
                                 int32_t* chart, int32_t* rung_host, double* rho_host, int32_t* rounds_host,
                                 int32_t* charts_host, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && uv && boxes && owner && labels && chart,
                  "verts, faces, uv, boxes, owner, labels and chart are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX - 1 && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv < 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(valid_size(N), "N must be a power of two in [64, 8192]");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_chart_atlas_scratch_bytes(nv, nf, N),
                  "scratch smaller than o2345_chart_atlas_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  ChartScratch S{nv, nf, N, {(char*)scratch}};
  auto read = [&](const int32_t* d, int32_t& h) {
    O2345_CUDA(cudaMemcpyAsync(&h, d, 4, cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };
  O2345_CUDA(cudaMemsetAsync(S.ctr, 0, 4 * kCtr, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.ctr + kErr, s));
  int32_t err = 0;   // the adjacency scatters through the face indices: they are checked on the host first
  O2345_TRY(read(S.ctr + kErr, err));
  O2345_TRY(mesh_check_status(err, __func__));
  label_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, faces, nf, labels, S.puv, S.key);
  O2345_LAUNCH_CHECK();
  O2345_TRY(vertex_faces(faces, nf, nv, S.voff, S.vsums, S.vcursor, S.vadj, s));
  edge_kernel<<<cdiv(3 * nf, 256), 256, 0, s>>>(faces, nf, S.voff, S.vadj, S.nbr);
  O2345_LAUNCH_CHECK();
  int32_t rounds = 0, nc = 0;
  for (;;) {
    // connected components of the faces joined by an edge of two uses and the same key, rooted at their least face
    O2345_TRY(union_find(S.parent, nf, S.ctr + kChanged, [&] {
      hook_kernel<<<cdiv(nf, 256), 256, 0, s>>>(S.nbr, S.key, nf, S.parent, S.ctr + kChanged);
      O2345_LAUNCH_CHECK();
      return O2345_OK;
    }, s));
    O2345_CUDA(cudaMemsetAsync(S.off, 0, 4 * (nf + 1), s));
    O2345_CUDA(cudaMemsetAsync(S.cursor, 0, 4 * nf, s));
    bucket_count_kernel<<<cdiv(nf, 256), 256, 0, s>>>(S.parent, nf, S.off, S.is_root);
    O2345_LAUNCH_CHECK();
    O2345_TRY(scan_i32(S.off, nf + 1, S.sums, nullptr, s));
    bucket_fill_kernel<<<cdiv(nf, 256), 256, 0, s>>>(S.parent, nf, S.off, S.cursor, S.list);
    O2345_LAUNCH_CHECK();
    O2345_TRY(o2345_compact(S.is_root, nf, S.roots, S.pos, S.count, S.cscratch, stream));
    O2345_TRY(read(S.count, nc));
    extent_kernel<<<(unsigned)nc, 128, 0, s>>>(S.roots, S.off, S.list, S.puv, S.lo, S.ext, S.area);
    O2345_CUDA(cudaMemsetAsync(S.flag, 0, nf, s));
    O2345_CUDA(cudaMemsetAsync(S.ctr + kFlagged, 0, 4, s));
    overlap_kernel<<<cdiv(nf, 128), 128, 0, s>>>(S.puv, S.parent, nf, S.off, S.list, S.flag, S.ctr + kFlagged);
    O2345_LAUNCH_CHECK();
    int32_t flagged = 0;
    O2345_TRY(read(S.ctr + kFlagged, flagged));
    if (!flagged) break;
    ++rounds;   // every flagged chart has two or more faces and splits: the loop ends
    cut_kernel<<<cdiv(nf, 128), 128, 0, s>>>(S.puv, S.parent, nf, S.off, S.list, S.pos, S.ext, S.flag, S.key);
    O2345_LAUNCH_CHECK();
  }
  O2345_TRY(cumsum_f64_chunked(S.area, nc, S.tot, s));   // area becomes its prefix sums: only the total is used
  double sum = 0.0;
  O2345_CUDA(cudaMemcpyAsync(&sum, S.tot + sum_chunks(nc), 8, cudaMemcpyDeviceToHost, s));
  O2345_CUDA(cudaStreamSynchronize(s));
  if (!(sum > 0.0)) {
    set_error("%s: the charts have no area", __func__);
    return O2345_EINVAL;
  }
  const double rho0 = sqrt(0.5 * ((double)N * (double)N) / sum);
  auto rho_of = [&](int j) { return rho0 * (double)j / (double)kRungDen; };
  auto trial = [&](int j, int32_t& fits) {
    box_kernel<<<cdiv(nc, 256), 256, 0, s>>>(S.ext, nc, rho_of(j), N, S.cboxes);
    pack_kernel<<<1, 32, 0, s>>>(S.cboxes, nc, N, S.order, S.ctr + kFits);
    O2345_LAUNCH_CHECK();
    return read(S.ctr + kFits, fits);
  };
  int32_t fits = 0;
  O2345_TRY(trial(1, fits));
  if (!fits) {
    set_error("%s: %d^2 texels cannot hold %d charts", __func__, N, nc);
    return O2345_EINVAL;
  }
  int lo = 1, hi = kRungs + 1, last = 1;
  while (hi - lo > 1) {
    int mid = (lo + hi) / 2;
    O2345_TRY(trial(mid, fits));
    last = mid;
    if (fits) lo = mid;
    else hi = mid;
  }
  if (last != lo) O2345_TRY(trial(lo, fits));   // the boxes of the chosen rung
  const double rho = rho_of(lo);
  chart_uv_kernel<<<cdiv(nf, 256), 256, 0, s>>>(S.puv, S.parent, nf, S.pos, S.lo, S.cboxes, rho, N, uv, boxes, chart);
  O2345_CUDA(cudaMemsetAsync(S.keys, 0xff, 8 * (int64_t)N * N, s));
  chart_owner_kernel<<<(unsigned)nf, 64, 0, s>>>(uv, boxes, N, S.keys);
  owner_from_keys_kernel<<<cdiv((int64_t)N * N, 256), 256, 0, s>>>(S.keys, (int64_t)N * N, owner);
  O2345_LAUNCH_CHECK();
  if (rung_host) *rung_host = lo;
  if (rho_host) *rho_host = rho;
  if (rounds_host) *rounds_host = rounds;
  if (charts_host) *charts_host = nc;
  return O2345_OK;
}
