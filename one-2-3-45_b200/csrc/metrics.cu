// Mesh scoring (o2345/mesh_metrics.py, eval_mesh.py): area-uniform surface samples and an exact fp32 nearest neighbour.
//
//   surface sample  face weights = twice the area in fp64 (one thread per face), cumulative sums in a fixed order
//                   (cumsum_f64_chunked, scan.cu), one thread per sample: three splitmix64 uniforms, an upper-bound search
//                   of the CDF, the barycentric point in fp64 rounded once;
//   nearest         uniform grid of cubic cells over the reference points (bbox reduction, count, scan, scatter), one
//                   thread per query visiting rows of cells ring by ring around it until a conservative lower bound on
//                   the distance of every unvisited cell exceeds the best distance found.
//
// Every floating-point operation is an explicit round-to-nearest intrinsic in the order oracle/metrics_oracle.py repeats
// with numpy (no FMA contraction), so samples, neighbour indices and squared distances are bit-identical to the oracle
// and do not depend on thread scheduling (ties go to the lower reference index).
#include "mesh_common.cuh"

namespace o2345 {
namespace {

constexpr int kMaxSide = 256;       // cells per grid axis at most: 2^24 cells, 64 MiB of cell offsets
constexpr int kPtsPerCell = 4;      // target points per occupied cell of a surface: side ~ sqrt(n_ref / 4)
constexpr float kCellSlack = 1e-3f; // cells: bound on the rounding of a coordinate's cell position (binning and bound)
constexpr float kBoundSlack = 0.999996f;   // relative: rounding of the squared bound and of a computed distance

// ----------------------------------------------------------------------------- surface sampling
__device__ __forceinline__ uint64_t splitmix64(uint64_t seed, uint64_t c) {
  uint64_t z = seed + (c + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// uniform in [0, 1): the top 53 bits of output c of splitmix64 seeded with `seed`
__device__ __forceinline__ double uniform(uint64_t seed, uint64_t c) {
  return __dmul_rn((double)(splitmix64(seed, c) >> 11), 0x1.0p-53);
}

// cdf[t] := twice the area of face t (0 for an index outside [0, nv) and for a non-finite value)
__global__ void face_weights_kernel(const float* __restrict__ verts, int64_t nv, const int32_t* __restrict__ faces, int64_t nf,
                                    double* __restrict__ cdf) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nf) return;
  int i[3] = {__ldg(faces + 3 * t), __ldg(faces + 3 * t + 1), __ldg(faces + 3 * t + 2)};
  double w = 0.0;
  if (face_ok(i, nv)) {
    D3 n = cross3(vert(verts, i[0]), vert(verts, i[1]), vert(verts, i[2]));
    w = __dsqrt_rn(dot3(n, n));
    if (!isfinite(w)) w = 0.0;
  }
  cdf[t] = w;
}

__global__ void sample_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, const double* __restrict__ cdf,
                              int64_t nf, double total, int64_t n, uint64_t seed, float* __restrict__ pts,
                              int32_t* __restrict__ face_id) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double u0 = uniform(seed, 3 * (uint64_t)i), u1 = uniform(seed, 3 * (uint64_t)i + 1), u2 = uniform(seed, 3 * (uint64_t)i + 2);
  double target = __dmul_rn(u0, total);
  int64_t lo = 0, hi = nf;   // first face whose CDF exceeds the target: zero-weight faces are never chosen
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > target) hi = mid; else lo = mid + 1;
  }
  if (lo == nf) {            // u0 * total rounded up to the total: the first face that reaches it
    lo = 0, hi = nf;
    while (lo < hi) {
      int64_t mid = (lo + hi) >> 1;
      if (cdf[mid] >= total) hi = mid; else lo = mid + 1;
    }
  }
  double s = __dsqrt_rn(u1);
  double wa = __dsub_rn(1.0, s), wb = __dmul_rn(s, __dsub_rn(1.0, u2)), wc = __dmul_rn(s, u2);
  const int32_t* f = faces + 3 * lo;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double p = __dadd_rn(__dadd_rn(__dmul_rn(wa, (double)verts[3 * (int64_t)f[0] + c]), __dmul_rn(wb, (double)verts[3 * (int64_t)f[1] + c])),
                         __dmul_rn(wc, (double)verts[3 * (int64_t)f[2] + c]));
    pts[3 * i + c] = __double2float_rn(p);
  }
  face_id[i] = (int32_t)lo;
}

// ----------------------------------------------------------------------------- nearest neighbour
// float <-> unsigned key with the same order (finite values and infinities), for min / max by integer atomics
__device__ __forceinline__ uint32_t float_key(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

int grid_side(int64_t n_ref) {
  int g = (int)ceil(sqrt((double)n_ref / kPtsPerCell));
  return max(1, min(g, kMaxSide));
}

struct Grid {
  float lo[3], hi[3], h;
  int dims[3];
};

// The grid of the reference points from their bbox (keys[0..2] min, keys[3..5] max): cubic cells of side h = the
// largest extent / side (1 for a single point), at most `side` cells per axis, at least one.
__device__ __forceinline__ Grid make_grid(const uint32_t* __restrict__ keys, int side) {
  Grid g;
#pragma unroll
  for (int a = 0; a < 3; ++a) g.lo[a] = key_float(keys[a]), g.hi[a] = key_float(keys[3 + a]);
  float ext = fmaxf(fmaxf(__fsub_rn(g.hi[0], g.lo[0]), __fsub_rn(g.hi[1], g.lo[1])), __fsub_rn(g.hi[2], g.lo[2]));
  g.h = __fdiv_rn(ext, (float)side);
  if (!(g.h > 0.f) || !isfinite(g.h)) g.h = 1.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float t = __fdiv_rn(__fsub_rn(g.hi[a], g.lo[a]), g.h);
    g.dims[a] = t < (float)side ? (int)t + 1 : side;
  }
  return g;
}

// cell coordinate of x along axis a (position t in cells, clamped to the grid)
__device__ __forceinline__ int cell_of(const Grid& g, int a, float x, float& t) {
  t = __fdiv_rn(__fsub_rn(x, g.lo[a]), g.h);
  float c = floorf(t);
  return c < 0.f ? 0 : (c >= (float)(g.dims[a] - 1) ? g.dims[a] - 1 : (int)c);   // NaN -> cell 0
}

__global__ void bbox_kernel(const float* __restrict__ ref, int64_t n, uint32_t* __restrict__ keys) {
  uint32_t mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      uint32_t k = float_key(__ldg(ref + 3 * i + a));
      mn[a] = min(mn[a], k), mx[a] = max(mx[a], k);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) atomicMin(keys + a, mn[a]), atomicMax(keys + 3 + a, mx[a]);
  }
}

// counts[cell] += 1 for every reference point; its cell and its rank among the cell's points (arrival order)
__global__ void bin_kernel(const float* __restrict__ ref, int64_t n, const uint32_t* __restrict__ keys, int side,
                           int32_t* __restrict__ counts, int32_t* __restrict__ cell, int32_t* __restrict__ rank) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Grid g = make_grid(keys, side);
  float t;
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = cell_of(g, a, __ldg(ref + 3 * i + a), t);
  int id = (c[2] * g.dims[1] + c[1]) * g.dims[0] + c[0];
  cell[i] = id;
  rank[i] = atomicAdd(counts + id, 1);
}

// sorted[start[cell] + rank] = (x, y, z, index bits): the points of a cell, and of a row of cells along x, are contiguous
__global__ void scatter_kernel(const float* __restrict__ ref, int64_t n, const int32_t* __restrict__ start,
                               const int32_t* __restrict__ cell, const int32_t* __restrict__ rank, float4* __restrict__ sorted) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  sorted[start[cell[i]] + rank[i]] = make_float4(ref[3 * i], ref[3 * i + 1], ref[3 * i + 2], __int_as_float((int)i));
}

__device__ __forceinline__ void visit(const float4* __restrict__ sorted, int a, int b, float qx, float qy, float qz, float& best,
                                      int& bi) {
  for (int j = a; j < b; ++j) {
    float4 p = __ldg(sorted + j);
    float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    int id = __float_as_int(p.w);
    if (d2 < best || (d2 == best && id < bi)) best = d2, bi = id;
  }
}

// Squared lower bound, along one axis, of the distance from the query to any point of the cells at offset j from the
// query's cell: the gap to the nearest face of those cells (lo / hi: the query's distance to its cell's lower / upper face,
// in cells) or the query's distance `out` to the bbox, whichever is larger.  kCellSlack covers the rounding of the cell
// positions of the query and of the points.
__device__ __forceinline__ float axis_bound(int j, float lo, float hi, float out, float h) {
  float gap = 0.f;
  if (j != 0) gap = __fmul_rn(fmaxf(__fsub_rn(__fadd_rn((float)(abs(j) - 1), j < 0 ? lo : hi), 2.f * kCellSlack), 0.f), h);
  float b = fmaxf(gap, out);
  return __fmul_rn(b, b);
}

// One thread per query.  Rows of cells along x (contiguous in `sorted`) are visited ring by ring of Chebyshev radius r in
// the (y, z) plane, with row / ring lower bounds and the x extent of a row cut by the best distance found so far.  A cell
// is skipped only when its bound times kBoundSlack exceeds that distance (strictly: equal distances go to the tie rule).
__global__ void nearest_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ start, const uint32_t* __restrict__ keys,
                               int side, const float* __restrict__ query, int64_t nq, float* __restrict__ dist2,
                               int32_t* __restrict__ index) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  Grid g = make_grid(keys, side);
  float q[3] = {query[3 * i], query[3 * i + 1], query[3 * i + 2]}, lo[3], hi[3], out[3];
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float t;
    c[a] = cell_of(g, a, q[a], t);
    float tc = fminf(fmaxf(t, (float)c[a]), (float)(c[a] + 1));      // clamped into the query's cell
    lo[a] = __fsub_rn(tc, (float)c[a]), hi[a] = __fsub_rn((float)(c[a] + 1), tc);
    out[a] = fmaxf(fmaxf(__fsub_rn(g.lo[a], q[a]), __fsub_rn(q[a], g.hi[a])), 0.f);
  }
  auto bound = [&](int a, int j) { return axis_bound(j, lo[a], hi[a], out[a], g.h); };
  float best = __int_as_float(0x7f800000);   // +inf
  int bi = INT32_MAX;
  const int rowlen = g.dims[0], plane = g.dims[0] * g.dims[1];
  int own = (c[2] * g.dims[1] + c[1]) * rowlen + c[0];
  visit(sorted, __ldg(start + own), __ldg(start + own + 1), q[0], q[1], q[2], best, bi);   // a first finite distance
  int rmax = max(max(c[1], g.dims[1] - 1 - c[1]), max(c[2], g.dims[2] - 1 - c[2]));
  float bx0 = bound(0, 0);
  for (int r = 0; r <= rmax; ++r) {
    if (r > 0) {   // every row of ring r has |jy| = r or |jz| = r; the bounds grow with r
      float by = fminf(bound(1, -r), bound(1, r)), bz = fminf(bound(2, -r), bound(2, r));
      float ring = __fadd_rn(bx0, fminf(__fadd_rn(by, bound(2, 0)), __fadd_rn(bound(1, 0), bz)));
      if (__fmul_rn(ring, kBoundSlack) > best) break;
    }
    int z0 = max(-r, -c[2]), z1 = min(r, g.dims[2] - 1 - c[2]);
    int y0 = max(-r, -c[1]), y1 = min(r, g.dims[1] - 1 - c[1]);
    for (int jz = z0; jz <= z1; ++jz) {
      bool face = jz == -r || jz == r;
      for (int jy = face ? y0 : -r; jy <= (face ? y1 : r); jy += face ? 1 : 2 * r) {
        if (jy < y0 || jy > y1) continue;
        float yz = __fadd_rn(bound(1, jy), bound(2, jz));
        if (__fmul_rn(__fadd_rn(yz, bx0), kBoundSlack) > best) continue;
        int x0 = 0, x1 = 0;
        while (c[0] + x0 > 0 && !(__fmul_rn(__fadd_rn(yz, bound(0, x0 - 1)), kBoundSlack) > best)) --x0;
        while (c[0] + x1 < rowlen - 1 && !(__fmul_rn(__fadd_rn(yz, bound(0, x1 + 1)), kBoundSlack) > best)) ++x1;
        int row = (c[2] + jz) * plane + (c[1] + jy) * rowlen + c[0];
        visit(sorted, __ldg(start + row + x0), __ldg(start + row + x1 + 1), q[0], q[1], q[2], best, bi);
      }
    }
  }
  dist2[i] = best;
  index[i] = bi == INT32_MAX ? -1 : bi;
}

// The scratch of o2345_surface_sample: the CDF, then the chunk offsets and the total.
struct SampleScratch {
  int64_t nf;
  Carver c;
  double* cdf = c.take<double>(nf);
  double* tot = c.take<double>(sum_chunks(nf) + 1);
};

// The scratch of o2345_nearest, carved in this order (a Carver without a base only measures it).
struct NNScratch {
  int64_t n_ref;
  Carver c;
  int side = grid_side(n_ref);
  int64_t cells = (int64_t)side * side * side;
  float4* sorted = c.take<float4>(n_ref);
  int32_t* start = c.take<int32_t>(cells + 1);
  int32_t* sums = c.take<int32_t>(scan_blocks(cells + 1));
  int32_t* cell = c.take<int32_t>(n_ref);
  int32_t* rank = c.take<int32_t>(n_ref);
  uint32_t* keys = c.take<uint32_t>(6);
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_surface_sample_scratch_bytes(int64_t nf) {
  if (nf < 1) return -1;
  return SampleScratch{nf, {}}.c.bytes;
}

extern "C" int o2345_surface_sample(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t n, uint64_t seed,
                                    void* scratch, int64_t scratch_bytes, float* pts, int32_t* face_id, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && pts && face_id, "verts, faces, pts and face_id are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX && nf >= 1 && nf <= INT32_MAX, "need 1 <= nv, nf <= 2^31-1");
  O2345_CHECK_ARG(n >= 1 && n <= INT32_MAX, "need 1 <= n <= 2^31-1");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_surface_sample_scratch_bytes(nf),
                  "scratch smaller than o2345_surface_sample_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  SampleScratch S{nf, {(char*)scratch}};
  face_weights_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, nv, faces, nf, S.cdf);
  O2345_LAUNCH_CHECK();
  O2345_TRY(cumsum_f64_chunked(S.cdf, nf, S.tot, s));
  double total = 0.0;   // the one host synchronisation: a surface without area has nothing to sample
  O2345_CUDA(cudaMemcpyAsync(&total, S.tot + sum_chunks(nf), sizeof(double), cudaMemcpyDeviceToHost, s));
  O2345_CUDA(cudaStreamSynchronize(s));
  if (!(total > 0.0)) {
    set_error("%s: the faces have no area (every face is degenerate or has an index outside [0, nv))", __func__);
    return O2345_EINVAL;
  }
  sample_kernel<<<cdiv(n, 256), 256, 0, s>>>(verts, faces, S.cdf, nf, total, n, seed, pts, face_id);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int64_t o2345_nn_scratch_bytes(int64_t n_ref, int64_t n_query) {
  if (n_ref < 1 || n_ref > INT32_MAX - 1 || n_query < 1 || n_query > INT32_MAX) return -1;
  return NNScratch{n_ref, {}}.c.bytes;
}

extern "C" int o2345_nearest(const float* ref, int64_t n_ref, const float* query, int64_t n_query, void* scratch,
                             int64_t scratch_bytes, float* dist2, int32_t* index, o2345_stream_t stream) {
  O2345_CHECK_ARG(ref && query && dist2 && index, "ref, query, dist2 and index are required");
  O2345_CHECK_ARG(n_ref >= 1 && n_ref <= INT32_MAX - 1 && n_query >= 1 && n_query <= INT32_MAX,
                  "need 1 <= n_ref < 2^31-1 and 1 <= n_query <= 2^31-1");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_nn_scratch_bytes(n_ref, n_query), "scratch smaller than o2345_nn_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  NNScratch S{n_ref, {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.keys, 0xff, 12, s));
  O2345_CUDA(cudaMemsetAsync(S.keys + 3, 0, 12, s));
  O2345_CUDA(cudaMemsetAsync(S.start, 0, 4 * (S.cells + 1), s));
  bbox_kernel<<<min(cdiv(n_ref, 256), sm_count() * 8), 256, 0, s>>>(ref, n_ref, S.keys);
  O2345_LAUNCH_CHECK();
  bin_kernel<<<cdiv(n_ref, 256), 256, 0, s>>>(ref, n_ref, S.keys, S.side, S.start, S.cell, S.rank);
  O2345_LAUNCH_CHECK();
  O2345_TRY(scan_i32(S.start, S.cells + 1, S.sums, nullptr, s));
  scatter_kernel<<<cdiv(n_ref, 256), 256, 0, s>>>(ref, n_ref, S.start, S.cell, S.rank, S.sorted);
  O2345_LAUNCH_CHECK();
  nearest_kernel<<<cdiv(n_query, 128), 128, 0, s>>>(S.sorted, S.start, S.keys, S.side, query, n_query, dist2, index);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
