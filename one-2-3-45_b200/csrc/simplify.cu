// Mesh simplification (ops.simplify_mesh, o2345/mesh_simplify.py): parallel half-edge collapse driven by quadric error.
//
//   input      one thread per face / vertex: index and finiteness checks, faces with a repeated index dropped (ordered
//              compaction, o2345_compact);
//   per round  vertex -> face adjacency (vertex_faces, mesh_common.cu: sorted by face index), then one thread per
//              vertex: locks and valence; the vertex quadrics (first round only, summed in ascending face order); the
//              proposal of every unlocked vertex (its legal neighbour with the least (cost, index)) and its claim, an
//              atomicMin of the 64-bit key over the closed 1-rings of both ends; acceptance where the key holds every
//              claim; at most k = ceil((F - target) / 2) accepted by a one-block search for the k-th least key; apply
//              (u -> v in u's faces, the two faces of uv dropped, Q_v += Q_u) and an ordered compaction of the faces;
//   output     the referenced vertices in ascending order, the faces renumbered into them.
//
// Accepted collapses touch disjoint closed 1-rings, so they apply in parallel and the result does not depend on thread
// order.  The count of accepted proposals is read on the host once per round (the loop's only synchronisation).  Every
// floating-point operation is an explicit round-to-nearest intrinsic in the order oracle/simplify_oracle.py repeats with
// numpy (no FMA contraction), so the output is bit-identical to the oracle.
#include "mesh_common.cuh"

namespace o2345 {
namespace {

constexpr int kSelect = 1024;                 // threads of the k-th key search
constexpr uint64_t kNone = ~0ull;             // no proposal / no claim
enum { kErr = 0, kFaces = 1, kAccepted = 2, kAlive = 3, kUsed = 4, kCtr = 8 };

// ----------------------------------------------------------------------------- input
// dst[i] = src[rows[i]] (faces)
__global__ void gather_faces_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ rows, int64_t n,
                                    int32_t* __restrict__ dst) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t r = rows[i];
  dst[3 * i] = src[3 * r], dst[3 * i + 1] = src[3 * r + 1], dst[3 * i + 2] = src[3 * r + 2];
}

// ----------------------------------------------------------------------------- adjacency (vertex_faces, mesh_common.cu)
// One thread per vertex: counts its distinct neighbours and locks it unless every edge at it has exactly two faces and
// its faces form one closed fan (vertex_lock, mesh_common.cuh).
__global__ void vertex_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ off, const int32_t* __restrict__ adj,
                              int nv, uint8_t* __restrict__ locked, int32_t* __restrict__ val) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  locked[u] = vertex_lock(F, adj + off[u], off[u + 1] - off[u], u, val + u);
}

// Q[u] = sum over u's faces, in ascending face order, of w (p p^T) (10 entries, i <= j)
__global__ void quadric_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                               const int32_t* __restrict__ adj, int nv, double* __restrict__ Q) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) q[i] = 0.0;
  for (int j = off[u]; j < off[u + 1]; ++j) {
    int f = adj[j];
    D3 A = vert(V, F[3 * f]);
    D3 n = cross3(A, vert(V, F[3 * f + 1]), vert(V, F[3 * f + 2]));
    double ln = __dsqrt_rn(dot3(n, n));
    double p[4] = {0.0, 0.0, 0.0, 0.0}, w = 0.0;
    if (ln > 0.0) {
      p[0] = __ddiv_rn(n.x, ln), p[1] = __ddiv_rn(n.y, ln), p[2] = __ddiv_rn(n.z, ln);
      p[3] = -__dadd_rn(__dadd_rn(__dmul_rn(p[0], A.x), __dmul_rn(p[1], A.y)), __dmul_rn(p[2], A.z));
      w = __dmul_rn(ln, 0.5);
    }
    int k = 0;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = a; b < 4; ++b, ++k) q[k] = __dadd_rn(q[k], ln > 0.0 ? __dmul_rn(w, __dmul_rn(p[a], p[b])) : 0.0);
  }
#pragma unroll
  for (int i = 0; i < 10; ++i) Q[10 * (int64_t)u + i] = q[i];
}

// ----------------------------------------------------------------------------- one round
// v^T (Q_u + Q_v) v at v = (x, y, z, 1), rounded to fp32; anything not > 0 becomes +0
__device__ __forceinline__ float collapse_cost(const double* __restrict__ Q, const float* __restrict__ V, int u, int v) {
  constexpr int S[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) q[i] = __dadd_rn(Q[10 * (int64_t)u + i], Q[10 * (int64_t)v + i]);
  D3 p = vert(V, v);
  double r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[S[i][0]], p.x), __dmul_rn(q[S[i][1]], p.y)), __dmul_rn(q[S[i][2]], p.z)),
                     q[S[i][3]]);
  float c = __double2float_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], p.x), __dmul_rn(r[1], p.y)), __dmul_rn(r[2], p.z)), r[3]));
  return c > 0.f ? c : 0.f;
}

__device__ __forceinline__ void claim_ring(const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                                           const int32_t* __restrict__ adj, int x, uint64_t key, uint64_t* __restrict__ claim) {
  for (int j = off[x]; j < off[x + 1]; ++j) {
    int f = adj[j];
#pragma unroll
    for (int k = 0; k < 3; ++k) atomicMin((unsigned long long*)claim + F[3 * f + k], (unsigned long long)key);
  }
}

__device__ __forceinline__ bool holds_ring(const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                                           const int32_t* __restrict__ adj, int x, uint64_t key, const uint64_t* __restrict__ claim) {
  for (int j = off[x]; j < off[x + 1]; ++j) {
    int f = adj[j];
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (claim[F[3 * f + k]] != key) return false;
  }
  return true;
}

// Every unlocked u proposes its legal neighbour with the least (cost, index) and claims both closed 1-rings with the
// key (bits(cost) << 32) | u.
__global__ void propose_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                               const int32_t* __restrict__ adj, const uint8_t* __restrict__ locked,
                               const int32_t* __restrict__ val, const double* __restrict__ Q, int nv, int32_t* __restrict__ target,
                               uint64_t* __restrict__ key, uint64_t* __restrict__ claim) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  key[u] = kNone;
  if (locked[u]) return;
  const int32_t* L = adj + off[u];
  int d = off[u + 1] - off[u];
  uint64_t best = kNone;
  for (int j = 0; j < d; ++j) {
    int x[2];
    others(F, L[j], u, x[0], x[1]);
    for (int t = 0; t < 2; ++t) {
      bool before = false;
      for (int i = 0; i < j && !before; ++i) before = has(F, L[i], x[t]);
      if (before || !legal_collapse(V, F, off, adj, val, u, x[t])) continue;
      uint64_t c = ((uint64_t)__float_as_uint(collapse_cost(Q, V, u, x[t])) << 32) | (uint32_t)x[t];
      best = c < best ? c : best;
    }
  }
  if (best == kNone) return;
  int v = (int)(uint32_t)best;
  uint64_t k = (best & 0xffffffff00000000ull) | (uint32_t)u;
  target[u] = v, key[u] = k;
  claim_ring(F, off, adj, u, k, claim);
  claim_ring(F, off, adj, v, k, claim);
}

__global__ void accept_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ off, const int32_t* __restrict__ adj,
                              const int32_t* __restrict__ target, const uint64_t* __restrict__ key,
                              const uint64_t* __restrict__ claim, int nv, uint8_t* __restrict__ acc) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  uint64_t k = key[u];
  acc[u] = k != kNone && holds_ring(F, off, adj, u, k, claim) && holds_ring(F, off, adj, target[u], k, claim);
}

// one block: *thresh = the k-th least key of the m accepted proposals (keys are distinct)
__global__ void __launch_bounds__(kSelect) select_kernel(const int32_t* __restrict__ list, int m, const uint64_t* __restrict__ key,
                                                     int k, uint64_t* __restrict__ thresh) {
  __shared__ int tot;
  uint64_t lo = 0, hi = kNone;
  while (lo < hi) {
    uint64_t mid = lo + ((hi - lo) >> 1);
    int c = 0;
    for (int i = threadIdx.x; i < m; i += kSelect) c += key[list[i]] <= mid;
    if (threadIdx.x == 0) tot = 0;
    __syncthreads();
    atomicAdd(&tot, c);
    __syncthreads();
    if (tot >= k) hi = mid;
    else lo = mid + 1;
    __syncthreads();
  }
  if (threadIdx.x == 0) *thresh = lo;
}

// u -> v: u's faces take v, the two faces of uv die, Q_v += Q_u
__global__ void apply_kernel(const int32_t* __restrict__ list, int m, const uint64_t* __restrict__ key,
                             const uint64_t* __restrict__ thresh, const int32_t* __restrict__ target,
                             const int32_t* __restrict__ off, const int32_t* __restrict__ adj, int32_t* __restrict__ F,
                             uint8_t* __restrict__ alive, double* __restrict__ Q) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  int u = list[i];
  if (key[u] > *thresh) return;
  int v = target[u];
  for (int j = off[u]; j < off[u + 1]; ++j) {
    int f = adj[j];
    if (has(F, f, v)) {
      alive[f] = 0;
      continue;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (F[3 * f + k] == u) F[3 * f + k] = v;
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) Q[10 * (int64_t)v + k] = __dadd_rn(Q[10 * (int64_t)v + k], Q[10 * (int64_t)u + k]);
}

// ----------------------------------------------------------------------------- output
__global__ void mark_kernel(const int32_t* __restrict__ F, int64_t n3, uint8_t* __restrict__ used) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) used[F[i]] = 1;
}

__global__ void renumber_kernel(const int32_t* __restrict__ F, int64_t n3, const int32_t* __restrict__ remap,
                                int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) out[i] = remap[F[i]];
}

__global__ void counts_kernel(const int32_t* __restrict__ ctr, int64_t nf, int rounds, int32_t* __restrict__ out) {
  out[0] = ctr[kUsed], out[1] = (int32_t)nf, out[2] = rounds;
}

// The scratch of o2345_simplify, carved in this order (a Carver without a base only measures it).
struct Scratch {
  int64_t nv, nf;
  Carver c;
  int64_t nmax = nv > nf ? nv : nf;
  double* Q = c.take<double>(10 * nv);
  uint64_t* key = c.take<uint64_t>(nv);
  uint64_t* claim = c.take<uint64_t>(nv);
  int32_t* ctr = c.take<int32_t>(kCtr + 2);   // counters, then the 64-bit selection threshold
  int32_t* faces_a = c.take<int32_t>(3 * nf);
  int32_t* faces_b = c.take<int32_t>(3 * nf);
  int32_t* adj = c.take<int32_t>(3 * nf);
  int32_t* rows = c.take<int32_t>(nmax);
  int32_t* cscratch = c.take<int32_t>(o2345_compact_scratch_ints(nmax));
  int32_t* off = c.take<int32_t>(nv + 1);
  int32_t* sums = c.take<int32_t>(scan_blocks(nv + 1));
  int32_t* cursor = c.take<int32_t>(nv);
  int32_t* val = c.take<int32_t>(nv);
  int32_t* target = c.take<int32_t>(nv);
  int32_t* remap = c.take<int32_t>(nv);
  uint8_t* flags = c.take<uint8_t>(nmax);
  uint8_t* acc = c.take<uint8_t>(nv);
  uint8_t* locked = c.take<uint8_t>(nv);
};

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_simplify_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 1 || nv > INT32_MAX - 1 || nf < 1 || nf > INT32_MAX / 3) return -1;
  return Scratch{nv, nf, {}}.c.bytes;
}

extern "C" int o2345_simplify(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t target_faces,
                              void* scratch, int64_t scratch_bytes, int32_t* vertex_index, int32_t* out_faces,
                              int32_t* out_counts, o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && vertex_index && out_faces && out_counts, "verts, faces, vertex_index, out_faces and out_counts are required");
  O2345_CHECK_ARG(nv >= 1 && nv <= INT32_MAX - 1 && nf >= 1 && nf <= INT32_MAX / 3, "need 1 <= nv < 2^31-1 and 1 <= nf <= (2^31-1)/3");
  O2345_CHECK_ARG(target_faces >= 0, "target_faces must be >= 0");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_simplify_scratch_bytes(nv, nf), "scratch smaller than o2345_simplify_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  Scratch S{nv, nf, {(char*)scratch}};
  uint64_t* thresh = (uint64_t*)(S.ctr + kCtr);
  int32_t host[kCtr];
  auto read_counters = [&]() {
    O2345_CUDA(cudaMemcpyAsync(host, S.ctr, sizeof(host), cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };

  O2345_CUDA(cudaMemsetAsync(S.ctr, 0, 4 * kCtr, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, S.flags, S.ctr + kErr, s));
  O2345_TRY(o2345_compact(S.flags, nf, S.rows, nullptr, S.ctr + kFaces, S.cscratch, stream));
  O2345_TRY(read_counters());
  O2345_TRY(mesh_check_status(host[kErr], __func__));
  int64_t F = host[kFaces];
  if (F > 0) {
    gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(faces, S.rows, F, S.faces_a);
    O2345_LAUNCH_CHECK();
  }
  int32_t *cur = S.faces_a, *nxt = S.faces_b;
  int rounds = 0;
  const int vb = cdiv(nv, 128);
  while (F > target_faces) {
    O2345_TRY(vertex_faces(cur, F, nv, S.off, S.sums, S.cursor, S.adj, s));
    vertex_kernel<<<vb, 128, 0, s>>>(cur, S.off, S.adj, (int)nv, S.locked, S.val);
    if (rounds == 0) quadric_kernel<<<vb, 128, 0, s>>>(verts, cur, S.off, S.adj, (int)nv, S.Q);
    O2345_CUDA(cudaMemsetAsync(S.claim, 0xff, 8 * nv, s));
    propose_kernel<<<vb, 128, 0, s>>>(verts, cur, S.off, S.adj, S.locked, S.val, S.Q, (int)nv, S.target, S.key, S.claim);
    accept_kernel<<<vb, 128, 0, s>>>(cur, S.off, S.adj, S.target, S.key, S.claim, (int)nv, S.acc);
    O2345_LAUNCH_CHECK();
    O2345_TRY(o2345_compact(S.acc, nv, S.rows, nullptr, S.ctr + kAccepted, S.cscratch, stream));
    O2345_TRY(read_counters());   // the round's one host synchronisation
    const int64_t m = host[kAccepted], k = (F - target_faces + 1) / 2;
    if (m == 0) break;            // no legal collapse is left
    O2345_CUDA(cudaMemsetAsync(thresh, 0xff, 8, s));
    if (m > k) select_kernel<<<1, kSelect, 0, s>>>(S.rows, (int)m, S.key, (int)k, thresh);
    O2345_CUDA(cudaMemsetAsync(S.flags, 1, F, s));
    apply_kernel<<<cdiv(m, 128), 128, 0, s>>>(S.rows, (int)m, S.key, thresh, S.target, S.off, S.adj, cur, S.flags, S.Q);
    O2345_LAUNCH_CHECK();
    O2345_TRY(o2345_compact(S.flags, F, S.rows, nullptr, S.ctr + kAlive, S.cscratch, stream));
    F -= 2 * (m < k ? m : k);
    if (F > 0) gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(cur, S.rows, F, nxt);
    O2345_LAUNCH_CHECK();
    int32_t* t = cur;
    cur = nxt, nxt = t;
    ++rounds;
  }
  O2345_CUDA(cudaMemsetAsync(S.flags, 0, nv, s));
  if (F > 0) mark_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, S.flags);
  O2345_TRY(o2345_compact(S.flags, nv, vertex_index, S.remap, S.ctr + kUsed, S.cscratch, stream));
  if (F > 0) renumber_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, S.remap, out_faces);
  counts_kernel<<<1, 1, 0, s>>>(S.ctr, F, rounds, out_counts);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
