// Mesh cleaning (ops.clean_mesh, o2345/mesh_clean.py, run.py / simplify_mesh.py --min_component): drops the components
// of a mesh that are small next to the largest one or enclosed by it.  The rules are in include/o2345.h (o2345_clean_mesh).
//
//   components  union-find over the vertices, joined along face edges (union_find, mesh_common.cuh); per vertex root the
//               least face by atomicMin; the component heads (faces that are their component's least face) compacted in
//               ascending order (o2345_compact), so component c is the c-th head;
//   buckets     per component its face count (scan_i32: offsets), and the faces sorted by component, ascending inside each
//               one, by a stable least-significant-bit-first split per bit of the label (radix_sort_i32);
//   area        one thread per face: its area in fp64; one block per component: the ordered sum of its faces' areas;
//   largest     one block: the greatest area, the least component on ties;
//   winding     one block per other component: the ordered sum of the largest component's solid angles at the centroid
//               of the component's least face (Van Oosterom-Strackee, with an atan2 of round-to-nearest operations only);
//   keep        one thread per component, then the kept faces and the vertices they reference compacted in input order.
//
// Every floating-point operation is an explicit round-to-nearest intrinsic in the order oracle/clean_oracle.py repeats
// with numpy float64 (no FMA contraction), and every sum runs in a fixed order, so all outputs are bit-identical to the
// oracle and independent of thread scheduling.  The only atomics are on integers.
#include "mesh_common.cuh"

namespace o2345 {
namespace {

enum { kErr = 0, kChanged = 1, kHeads = 2, kOnes = 3, kLargest = 4, kKeptComps = 5, kEnclosed = 6, kKeptVerts = 7,
       kKeptFaces = 8, kCtr = 9 };
constexpr int kSumThreads = 256;   // threads of a block running one ordered sum

// The ordered sum of val(0 .. n-1) by a block of kSumThreads: sequential inside chunks of kSumChunk consecutive terms,
// then sequential over the chunk totals in ascending order, each sum starting from +0.0.  The result is thread 0's.
template <class Val>
__device__ double ordered_sum(int64_t n, Val val) {
  __shared__ double part[kSumThreads];
  double run = 0.0;
  for (int64_t base = 0; base < n; base += (int64_t)kSumThreads * kSumChunk) {
    const int64_t a = base + (int64_t)threadIdx.x * kSumChunk, b = min(a + kSumChunk, n);
    double s = 0.0;
#pragma unroll 4
    for (int64_t i = a; i < b; ++i) s = __dadd_rn(s, val(i));
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int k = 0; k < kSumThreads && base + (int64_t)k * kSumChunk < n; ++k) run = __dadd_rn(run, part[k]);
    __syncthreads();
  }
  return run;
}

// u x v
__device__ __forceinline__ D3 cross(D3 u, D3 v) {
  return {__dsub_rn(__dmul_rn(u.y, v.z), __dmul_rn(u.z, v.y)), __dsub_rn(__dmul_rn(u.z, v.x), __dmul_rn(u.x, v.z)),
          __dsub_rn(__dmul_rn(u.x, v.y), __dmul_rn(u.y, v.x))};
}

// 1 / (2k + 1), the Taylor coefficients of atan
__constant__ double kAtanC[12] = {1.0 / 1,  1.0 / 3,  1.0 / 5,  1.0 / 7,  1.0 / 9,  1.0 / 11,
                                  1.0 / 13, 1.0 / 15, 1.0 / 17, 1.0 / 19, 1.0 / 21, 1.0 / 23};
constexpr double kPi = 3.141592653589793, kHalfPi = 1.5707963267948966;

// atan2(y, x) from round-to-nearest +, -, *, / and sqrt only, so numpy repeats it bit for bit (0 for y = x = 0): t =
// min(|x|, |y|) / max(|x|, |y|), halved twice by atan t = 2 atan(t / (1 + sqrt(1 + t^2))) to |u| <= tan(pi / 16), the
// Taylor series to u^23 (Horner), then the octant.  Accurate to a few ulp.
__device__ __forceinline__ double atan2_rn(double y, double x) {
  const double ax = fabs(x), ay = fabs(y);
  if (ax == 0.0 && ay == 0.0) return 0.0;
  const bool swap = ay > ax;
  double u = swap ? __ddiv_rn(ax, ay) : __ddiv_rn(ay, ax);
#pragma unroll
  for (int h = 0; h < 2; ++h) u = __ddiv_rn(u, __dadd_rn(1.0, __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(u, u)))));
  const double u2 = __dmul_rn(u, u);
  double p = kAtanC[11];
#pragma unroll
  for (int k = 10; k >= 0; --k) p = __dsub_rn(kAtanC[k], __dmul_rn(u2, p));
  double r = __dmul_rn(4.0, __dmul_rn(u, p));
  if (swap) r = __dsub_rn(kHalfPi, r);
  if (x < 0.0) r = __dsub_rn(kPi, r);
  return y < 0.0 ? -r : r;
}

// The solid angle of triangle ABC seen from p: 2 atan2(a . (b x c), |a||b||c| + (a . b)|c| + (a . c)|b| + (b . c)|a|),
// a = A - p etc., the denominator summed left to right.
__device__ __forceinline__ double solid_angle(D3 A, D3 B, D3 C, D3 p) {
  const D3 a = sub3(A, p), b = sub3(B, p), c = sub3(C, p);
  const double la = __dsqrt_rn(dot3(a, a)), lb = __dsqrt_rn(dot3(b, b)), lc = __dsqrt_rn(dot3(c, c));
  const double det = dot3(a, cross(b, c));
  double den = __dmul_rn(__dmul_rn(la, lb), lc);
  den = __dadd_rn(den, __dmul_rn(dot3(a, b), lc));
  den = __dadd_rn(den, __dmul_rn(dot3(a, c), lb));
  den = __dadd_rn(den, __dmul_rn(dot3(b, c), la));
  return __dmul_rn(2.0, atan2_rn(det, den));
}

// One thread per face: its two edges from corner 0 join the corners' sets.
__global__ void hook_kernel(const int32_t* __restrict__ F, int64_t nf, int32_t* parent, int32_t* __restrict__ changed) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  unite(parent, F[3 * f], F[3 * f + 1], changed);
  unite(parent, F[3 * f], F[3 * f + 2], changed);
}

// least[r] := the least face whose corners have root r (least is filled with 0x7f7f7f7f first)
__global__ void least_face_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ parent,
                                  int32_t* __restrict__ least) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nf) atomicMin(least + parent[F[3 * f]], (int32_t)f);
}

__global__ void head_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ parent,
                            const int32_t* __restrict__ least, uint8_t* __restrict__ head) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nf) head[f] = least[parent[F[3 * f]]] == f;
}

// One thread per face: its component (the rank of its least face among the heads), its count, and its area
// 0.5 sqrt(n . n), n = (B - A) x (C - A), in fp64.
__global__ void label_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                             const int32_t* __restrict__ parent, const int32_t* __restrict__ least,
                             const int32_t* __restrict__ head_rank, int32_t* __restrict__ label, int32_t* __restrict__ cnt,
                             double* __restrict__ face_area) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int c[3] = {F[3 * f], F[3 * f + 1], F[3 * f + 2]};
  const int lab = head_rank[least[parent[c[0]]]];
  label[f] = lab;
  atomicAdd(cnt + lab, 1);
  D3 n = cross3(vert(V, c[0]), vert(V, c[1]), vert(V, c[2]));
  face_area[f] = __dmul_rn(0.5, __dsqrt_rn(dot3(n, n)));
}

// One block per component: its area, the ordered sum of its faces' areas in ascending face order.
__global__ void __launch_bounds__(kSumThreads) area_kernel(const int32_t* __restrict__ off, const int32_t* __restrict__ order,
                                                            const double* __restrict__ face_area, double* __restrict__ area) {
  const int32_t* list = order + off[blockIdx.x];
  double s = ordered_sum(off[blockIdx.x + 1] - off[blockIdx.x], [&](int64_t i) { return face_area[list[i]]; });
  if (threadIdx.x == 0) area[blockIdx.x] = s;
}

// One block: *largest := the component of greatest area, the least one on ties.
__global__ void __launch_bounds__(1024) largest_kernel(const double* __restrict__ area, int nc, int32_t* __restrict__ largest) {
  __shared__ double ba[1024];
  __shared__ int bi[1024];
  double a = -1.0;
  int best = -1;
  for (int c = threadIdx.x; c < nc; c += blockDim.x)
    if (area[c] > a) a = area[c], best = c;   // ascending c: the first of equal areas stays
  ba[threadIdx.x] = a, bi[threadIdx.x] = best;
  __syncthreads();
  for (int h = blockDim.x / 2; h > 0; h /= 2) {
    if (threadIdx.x < h) {
      double a2 = ba[threadIdx.x + h];
      int i2 = bi[threadIdx.x + h];
      if (i2 >= 0 && (a2 > ba[threadIdx.x] || (a2 == ba[threadIdx.x] && i2 < bi[threadIdx.x])))
        ba[threadIdx.x] = a2, bi[threadIdx.x] = i2;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *largest = bi[0];
}

// One block per component c other than the largest L: winding[c] := (ordered sum over L's faces, ascending, of their
// solid angles at the centroid ((A + B) + C) / 3 of c's least face) / (4 pi); winding[L] := 0.
__global__ void __launch_bounds__(kSumThreads, 1) winding_kernel(const float* __restrict__ V, const int32_t* __restrict__ F,
                                                               const int32_t* __restrict__ heads,
                                                               const int32_t* __restrict__ off,
                                                               const int32_t* __restrict__ order,
                                                               const int32_t* __restrict__ largest,
                                                               double* __restrict__ winding) {
  const int c = blockIdx.x, L = *largest;
  if (c == L) {
    if (threadIdx.x == 0) winding[c] = 0.0;
    return;
  }
  const int64_t h = heads[c];
  const D3 A = vert(V, F[3 * h]), B = vert(V, F[3 * h + 1]), C = vert(V, F[3 * h + 2]);
  const D3 p = {__ddiv_rn(__dadd_rn(__dadd_rn(A.x, B.x), C.x), 3.0), __ddiv_rn(__dadd_rn(__dadd_rn(A.y, B.y), C.y), 3.0),
                __ddiv_rn(__dadd_rn(__dadd_rn(A.z, B.z), C.z), 3.0)};
  const int32_t* list = order + off[L];
  double s = ordered_sum(off[L + 1] - off[L], [&](int64_t i) {
    const int64_t g = list[i];
    return solid_angle(vert(V, F[3 * g]), vert(V, F[3 * g + 1]), vert(V, F[3 * g + 2]), p);
  });
  if (threadIdx.x == 0) winding[c] = __ddiv_rn(s, 4.0 * kPi);
}

// One thread per component: keep[c] := c is the largest, or area[c] >= F area[L] and |winding[c]| < 0.5 (not enclosed).
__global__ void keep_kernel(const double* __restrict__ area, const double* __restrict__ winding, int nc, double F,
                            int32_t* __restrict__ ctr, uint8_t* __restrict__ keep) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  const int L = ctr[kLargest];
  const bool enclosed = c != L && fabs(winding[c]) >= 0.5;
  const bool k = c == L || (!enclosed && area[c] >= __dmul_rn(F, area[L]));
  keep[c] = k;
  if (k) atomicAdd(ctr + kKeptComps, 1);
  if (enclosed) atomicAdd(ctr + kEnclosed, 1);
}

// One thread per face: its keep flag, and the flags of the vertices a kept face references (vflag zeroed first).
__global__ void face_keep_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ label,
                                 const uint8_t* __restrict__ keep, uint8_t* __restrict__ fflag, uint8_t* __restrict__ vflag) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const uint8_t k = keep[label[f]];
  fflag[f] = k;
  if (k) vflag[F[3 * f]] = 1, vflag[F[3 * f + 1]] = 1, vflag[F[3 * f + 2]] = 1;
}

// out[k] := kept face rows[k] renumbered through vmap, for k < *count
__global__ void remap_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ rows, const int32_t* __restrict__ count,
                             const int32_t* __restrict__ vmap, int32_t* __restrict__ out) {
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= *count) return;
  const int64_t f = rows[k];
#pragma unroll
  for (int j = 0; j < 3; ++j) out[3 * k + j] = vmap[F[3 * f + j]];
}

// The scratch of o2345_clean_mesh, carved in this order (a Carver without a base only measures it).
struct CleanScratch {
  int64_t nv, nf;
  Carver c;
  int32_t* ctr = c.take<int32_t>(kCtr);
  int32_t* parent = c.take<int32_t>(nv);
  int32_t* least = c.take<int32_t>(nv);
  uint8_t* head = c.take<uint8_t>(nf);
  int32_t* heads = c.take<int32_t>(nf);
  int32_t* head_rank = c.take<int32_t>(nf);
  int32_t* off = c.take<int32_t>(nf + 1);
  int32_t* order = c.take<int32_t>(nf);
  int32_t* next = c.take<int32_t>(nf);
  int32_t* ones = c.take<int32_t>(nf);
  int32_t* sums = c.take<int32_t>(scan_blocks(nf + 1));
  double* face_area = c.take<double>(nf);
  uint8_t* fflag = c.take<uint8_t>(nf);
  uint8_t* vflag = c.take<uint8_t>(nv);
  int32_t* vmap = c.take<int32_t>(nv);
  int32_t* rows = c.take<int32_t>(nf);
  int32_t* cscratch = c.take<int32_t>(o2345_compact_scratch_ints(nv > nf ? nv : nf));
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_clean_mesh_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 1 || nv > INT32_MAX - 1 || nf < 1 || nf > INT32_MAX / 3) return -1;
  return CleanScratch{nv, nf, {}}.c.bytes;
}

extern "C" int o2345_clean_mesh(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, double min_component,
                                void* scratch, int64_t scratch_bytes, int32_t* label, double* area, double* winding,
                                uint8_t* keep, int32_t* vertex_index, int32_t* faces_out, int32_t* counts_host,
                                o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && label && area && winding && keep && vertex_index && faces_out && counts_host,
                  "verts, faces, label, area, winding, keep, vertex_index, faces_out and counts_host are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX - 1 && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv < 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(min_component > 0.0 && min_component <= 1.0, "min_component must lie in (0, 1]");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_clean_mesh_scratch_bytes(nv, nf),
                  "scratch smaller than o2345_clean_mesh_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  CleanScratch S{nv, nf, {(char*)scratch}};
  int32_t host[kCtr];
  auto read = [&]() {
    O2345_CUDA(cudaMemcpyAsync(host, S.ctr, sizeof(host), cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };
  O2345_CUDA(cudaMemsetAsync(S.ctr, 0, 4 * kCtr, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.ctr + kErr, s));
  O2345_TRY(read());   // the union-find follows the face indices: they are checked on the host first
  O2345_TRY(mesh_check_status(host[kErr], __func__));

  // components, numbered by their least face
  O2345_TRY(union_find(S.parent, nv, S.ctr + kChanged, [&] {
    hook_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, nf, S.parent, S.ctr + kChanged);
    O2345_LAUNCH_CHECK();
    return O2345_OK;
  }, s));
  O2345_CUDA(cudaMemsetAsync(S.least, 0x7f, 4 * nv, s));   // 0x7f7f7f7f: above every face index
  least_face_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, nf, S.parent, S.least);
  head_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, nf, S.parent, S.least, S.head);
  O2345_LAUNCH_CHECK();
  O2345_TRY(o2345_compact(S.head, nf, S.heads, S.head_rank, S.ctr + kHeads, S.cscratch, stream));
  O2345_CUDA(cudaMemsetAsync(S.off, 0, 4 * (nf + 1), s));
  label_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, faces, nf, S.parent, S.least, S.head_rank, label, S.off, S.face_area);
  O2345_LAUNCH_CHECK();
  O2345_TRY(read());
  const int nc = host[kHeads];

  // buckets: offsets, and the faces sorted by component (stable, so ascending inside each)
  O2345_TRY(scan_i32(S.off, nc + 1, S.sums, nullptr, s));
  int bits = 0;
  while ((1ll << bits) < nc) ++bits;
  O2345_TRY(radix_sort_i32(S.order, S.next, label, nf, bits, S.ones, S.sums, S.ctr + kOnes, s));

  area_kernel<<<nc, kSumThreads, 0, s>>>(S.off, S.order, S.face_area, area);
  largest_kernel<<<1, 1024, 0, s>>>(area, nc, S.ctr + kLargest);
  winding_kernel<<<nc, kSumThreads, 0, s>>>(verts, faces, S.heads, S.off, S.order, S.ctr + kLargest, winding);
  keep_kernel<<<cdiv(nc, 256), 256, 0, s>>>(area, winding, nc, min_component, S.ctr, keep);
  O2345_CUDA(cudaMemsetAsync(S.vflag, 0, nv, s));
  face_keep_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, nf, label, keep, S.fflag, S.vflag);
  O2345_LAUNCH_CHECK();
  O2345_TRY(o2345_compact(S.vflag, nv, vertex_index, S.vmap, S.ctr + kKeptVerts, S.cscratch, stream));
  O2345_TRY(o2345_compact(S.fflag, nf, S.rows, nullptr, S.ctr + kKeptFaces, S.cscratch, stream));
  remap_kernel<<<cdiv(nf, 256), 256, 0, s>>>(faces, S.rows, S.ctr + kKeptFaces, S.vmap, faces_out);
  O2345_LAUNCH_CHECK();
  O2345_TRY(read());
  counts_host[0] = nc;
  counts_host[1] = host[kLargest];
  counts_host[2] = host[kKeptComps];
  counts_host[3] = host[kEnclosed];
  counts_host[4] = host[kKeptVerts];
  counts_host[5] = host[kKeptFaces];
  return O2345_OK;
}
