// Mesh simplification (ops.simplify_mesh, o2345/mesh_simplify.py): parallel half-edge collapse driven by quadric error.
//
//   input      one thread per face / vertex: index and finiteness checks, faces with a repeated index dropped (ordered
//              compaction, o2345_compact);
//   per round  vertex -> face adjacency (degree count, scan, scatter, per-vertex sort by face index), then one thread per
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
#include "common.cuh"

namespace o2345 {
namespace {

constexpr int kSB = 1024;                     // elements per block of the degree scan
constexpr uint64_t kNone = ~0ull;             // no proposal / no claim
enum { kErr = 0, kFaces = 1, kAccepted = 2, kAlive = 3, kUsed = 4, kCtr = 8 };

// ----------------------------------------------------------------------------- exclusive scan of int32
__device__ __forceinline__ int block_exclusive_scan(int v, int& total) {
  __shared__ int warp_tot[32];
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += t;
  }
  if (lane == 31) warp_tot[w] = s;
  __syncthreads();
  if (w == 0) {
    int t = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int q = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += q;
    }
    warp_tot[lane] = t;
  }
  __syncthreads();
  int excl = s - v + (w > 0 ? warp_tot[w - 1] : 0);
  total = warp_tot[31];
  __syncthreads();
  return excl;
}

__global__ void __launch_bounds__(kSB) scan_block_kernel(int32_t* __restrict__ vals, int64_t n, int32_t* __restrict__ sums) {
  int64_t i = (int64_t)blockIdx.x * kSB + threadIdx.x;
  int v = i < n ? vals[i] : 0, total;
  int excl = block_exclusive_scan(v, total);
  if (i < n) vals[i] = excl;
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kSB) scan_tops_kernel(int32_t* __restrict__ sums, int nb) {
  int carry = 0;
  for (int base = 0; base < nb; base += kSB) {
    int i = base + threadIdx.x, v = i < nb ? sums[i] : 0, total;
    int excl = block_exclusive_scan(v, total);
    if (i < nb) sums[i] = carry + excl;
    carry += total;
  }
}

__global__ void scan_add_kernel(int32_t* __restrict__ vals, int64_t n, const int32_t* __restrict__ sums) {
  int64_t i = (int64_t)blockIdx.x * kSB + threadIdx.x;
  if (i < n) vals[i] += sums[blockIdx.x];
}

// ----------------------------------------------------------------------------- geometry, fp64 from the fp32 vertices
struct D3 {
  double x, y, z;
};

__device__ __forceinline__ D3 vert(const float* __restrict__ V, int i) {
  return {(double)__ldg(V + 3 * (int64_t)i), (double)__ldg(V + 3 * (int64_t)i + 1), (double)__ldg(V + 3 * (int64_t)i + 2)};
}

// (b - a) x (c - a), as metrics.cu's face weights
__device__ __forceinline__ D3 cross3(D3 a, D3 b, D3 c) {
  double e1x = __dsub_rn(b.x, a.x), e1y = __dsub_rn(b.y, a.y), e1z = __dsub_rn(b.z, a.z);
  double e2x = __dsub_rn(c.x, a.x), e2y = __dsub_rn(c.y, a.y), e2z = __dsub_rn(c.z, a.z);
  return {__dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y)), __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z)),
          __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x))};
}

__device__ __forceinline__ double dot3(D3 a, D3 b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}

// the two other corners of face f (in corner order after u)
__device__ __forceinline__ void others(const int32_t* __restrict__ F, int f, int u, int& a, int& b) {
  int c0 = F[3 * f], c1 = F[3 * f + 1], c2 = F[3 * f + 2];
  if (c0 == u) a = c1, b = c2;
  else if (c1 == u) a = c2, b = c0;
  else a = c0, b = c1;
}

__device__ __forceinline__ bool has(const int32_t* __restrict__ F, int f, int x) {
  return F[3 * f] == x || F[3 * f + 1] == x || F[3 * f + 2] == x;
}

// ----------------------------------------------------------------------------- input
// flags[f] = face f has three distinct indices; err bit 1: an index outside [0, nv), bit 2: a non-finite coordinate
__global__ void check_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                             uint8_t* __restrict__ flags, int32_t* __restrict__ ctr) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nf) {
    int a = F[3 * i], b = F[3 * i + 1], c = F[3 * i + 2];
    bool in = a >= 0 && a < nv && b >= 0 && b < nv && c >= 0 && c < nv;
    if (!in) atomicOr(ctr + kErr, 1);
    flags[i] = in && a != b && b != c && a != c;
  }
  if (i < nv) {
    for (int k = 0; k < 3; ++k)
      if (!isfinite(V[3 * i + k])) atomicOr(ctr + kErr, 2);
  }
}

// dst[i] = src[rows[i]] (faces)
__global__ void gather_faces_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ rows, int64_t n,
                                    int32_t* __restrict__ dst) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t r = rows[i];
  dst[3 * i] = src[3 * r], dst[3 * i + 1] = src[3 * r + 1], dst[3 * i + 2] = src[3 * r + 2];
}

// ----------------------------------------------------------------------------- adjacency
__global__ void degree_kernel(const int32_t* __restrict__ F, int64_t n3, int32_t* __restrict__ deg) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) atomicAdd(deg + F[i], 1);
}

__global__ void fill_kernel(const int32_t* __restrict__ F, int64_t n3, const int32_t* __restrict__ off,
                            int32_t* __restrict__ cursor, int32_t* __restrict__ adj) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  int v = F[i];
  adj[off[v] + atomicAdd(cursor + v, 1)] = (int32_t)(i / 3);
}

// One thread per vertex: sorts its faces by index (the scatter's order depends on scheduling), counts its distinct
// neighbours and locks it unless every edge at it has exactly two faces and its faces form one closed fan.
__global__ void vertex_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ off, int32_t* __restrict__ adj,
                              int nv, uint8_t* __restrict__ locked, int32_t* __restrict__ val) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  int32_t* L = adj + off[u];
  int d = off[u + 1] - off[u];
  for (int i = 1; i < d; ++i) {
    int f = L[i], j = i - 1;
    while (j >= 0 && L[j] > f) L[j + 1] = L[j], --j;
    L[j + 1] = f;
  }
  int nval = 0;
  bool ok = d > 0;
  for (int j = 0; j < d; ++j) {
    int ab[2];
    others(F, L[j], u, ab[0], ab[1]);
    for (int t = 0; t < 2; ++t) {
      int cnt = 0;
      bool before = false;
      for (int i = 0; i < d; ++i)
        if (has(F, L[i], ab[t])) ++cnt, before |= i < j;
      nval += !before;
      ok &= cnt == 2;
    }
  }
  if (ok) {   // walk across the edges from face 0 until the walk returns to it
    int a, b, x, prev = 0, seen = 1;
    others(F, L[0], u, a, b);
    x = b;
    for (int step = 0; step < d; ++step) {
      int j = -1, nx = -1;
      for (int i = 0; i < d && j < 0; ++i) {
        if (i == prev) continue;
        int p, q;
        others(F, L[i], u, p, q);
        if (p == x) j = i, nx = q;
        else if (q == x) j = i, nx = p;
      }
      if (j <= 0) break;
      ++seen, x = nx, prev = j;
    }
    ok = seen == d;
  }
  locked[u] = !ok;
  val[u] = nval;
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

// u -> v for an unlocked u (every edge at u has two faces): link condition, valences, no flipped or collapsed face
__device__ bool legal(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                      const int32_t* __restrict__ adj, const int32_t* __restrict__ val, int u, int v) {
  const int32_t* Lu = adj + off[u];
  const int32_t* Lv = adj + off[v];
  int du = off[u + 1] - off[u], dv = off[v + 1] - off[v];
  int o[2] = {-1, -1}, no = 0;
  for (int i = 0; i < du; ++i) {
    int p, q;
    others(F, Lu[i], u, p, q);
    if (p == v || q == v) o[no++ & 1] = p == v ? q : p;
  }
  if (o[0] == o[1] || val[o[0]] < 4 || val[o[1]] < 4 || val[u] + val[v] - 4 < 3) return false;
  for (int i = 0; i < du; ++i) {
    int x[2];
    others(F, Lu[i], u, x[0], x[1]);
    for (int t = 0; t < 2; ++t) {
      if (x[t] == v || x[t] == o[0] || x[t] == o[1]) continue;
      for (int j = 0; j < dv; ++j)
        if (has(F, Lv[j], x[t])) return false;
    }
  }
  D3 pv = vert(V, v);
  for (int i = 0; i < du; ++i) {
    int f = Lu[i];
    if (has(F, f, v)) continue;
    int c[3] = {F[3 * f], F[3 * f + 1], F[3 * f + 2]};
    D3 P[3] = {vert(V, c[0]), vert(V, c[1]), vert(V, c[2])};
    D3 n0 = cross3(P[0], P[1], P[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (c[k] == u) P[k] = pv;
    if (!(dot3(cross3(P[0], P[1], P[2]), n0) > 0.0)) return false;
  }
  return true;
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
      if (before || !legal(V, F, off, adj, val, u, x[t])) continue;
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
__global__ void __launch_bounds__(kSB) select_kernel(const int32_t* __restrict__ list, int m, const uint64_t* __restrict__ key,
                                                     int k, uint64_t* __restrict__ thresh) {
  __shared__ int tot;
  uint64_t lo = 0, hi = kNone;
  while (lo < hi) {
    uint64_t mid = lo + ((hi - lo) >> 1);
    int c = 0;
    for (int i = threadIdx.x; i < m; i += kSB) c += key[list[i]] <= mid;
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

struct Layout {
  int64_t nb, bytes;
  int64_t faces_a, faces_b, flags, acc, locked, rows, cscratch, off, sums, cursor, adj, val, target, remap, Q, key, claim, ctr;
};

int64_t align16(int64_t x) { return (x + 15) & ~(int64_t)15; }

Layout layout(int64_t nv, int64_t nf) {
  Layout L;
  int64_t nmax = nv > nf ? nv : nf;
  L.nb = (nv + 1 + kSB - 1) / kSB;
  int64_t o = 0;
  auto take = [&](int64_t& at, int64_t bytes) { at = o, o = align16(o + bytes); };
  take(L.Q, 80 * nv);
  take(L.key, 8 * nv);
  take(L.claim, 8 * nv);
  take(L.ctr, 4 * kCtr + 8);            // counters, then the 64-bit selection threshold
  take(L.faces_a, 12 * nf);
  take(L.faces_b, 12 * nf);
  take(L.adj, 12 * nf);
  take(L.rows, 4 * nmax);
  take(L.cscratch, 4 * o2345_compact_scratch_ints(nmax));
  take(L.off, 4 * (nv + 1));
  take(L.sums, 4 * L.nb);
  take(L.cursor, 4 * nv);
  take(L.val, 4 * nv);
  take(L.target, 4 * nv);
  take(L.remap, 4 * nv);
  take(L.flags, nmax);
  take(L.acc, nv);
  take(L.locked, nv);
  L.bytes = o;
  return L;
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_simplify_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 1 || nv > INT32_MAX - 1 || nf < 1 || nf > INT32_MAX / 3) return -1;
  return layout(nv, nf).bytes;
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
  Layout Lo = layout(nv, nf);
  char* p = (char*)scratch;
  auto* fa = (int32_t*)(p + Lo.faces_a);
  auto* fb = (int32_t*)(p + Lo.faces_b);
  auto* flags = (uint8_t*)(p + Lo.flags);
  auto* acc = (uint8_t*)(p + Lo.acc);
  auto* locked = (uint8_t*)(p + Lo.locked);
  auto* rows = (int32_t*)(p + Lo.rows);
  auto* cs = (int32_t*)(p + Lo.cscratch);
  auto* off = (int32_t*)(p + Lo.off);
  auto* sums = (int32_t*)(p + Lo.sums);
  auto* cursor = (int32_t*)(p + Lo.cursor);
  auto* adj = (int32_t*)(p + Lo.adj);
  auto* val = (int32_t*)(p + Lo.val);
  auto* target = (int32_t*)(p + Lo.target);
  auto* remap = (int32_t*)(p + Lo.remap);
  auto* Q = (double*)(p + Lo.Q);
  auto* key = (uint64_t*)(p + Lo.key);
  auto* claim = (uint64_t*)(p + Lo.claim);
  auto* ctr = (int32_t*)(p + Lo.ctr);
  auto* thresh = (uint64_t*)(ctr + kCtr);
  int32_t host[kCtr];
  auto read_counters = [&]() {
    O2345_CUDA(cudaMemcpyAsync(host, ctr, sizeof(host), cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };
  int rc;
#define O2345_TRY(x) \
  if ((rc = (x)) != O2345_OK) return rc

  O2345_CUDA(cudaMemsetAsync(ctr, 0, 4 * kCtr, s));
  int64_t nmax = nv > nf ? nv : nf;
  check_kernel<<<cdiv(nmax, 256), 256, 0, s>>>(verts, nv, faces, nf, flags, ctr);
  O2345_LAUNCH_CHECK();
  O2345_TRY(o2345_compact(flags, nf, rows, nullptr, ctr + kFaces, cs, stream));
  O2345_TRY(read_counters());
  if (host[kErr] & 1) {
    set_error("%s: a face index is outside [0, nv)", __func__);
    return O2345_EINVAL;
  }
  if (host[kErr] & 2) {
    set_error("%s: a vertex coordinate is not finite", __func__);
    return O2345_EINVAL;
  }
  int64_t F = host[kFaces];
  if (F > 0) {
    gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(faces, rows, F, fa);
    O2345_LAUNCH_CHECK();
  }
  int32_t *cur = fa, *nxt = fb;
  int rounds = 0;
  const int vb = cdiv(nv, 128);
  while (F > target_faces) {
    const int64_t n3 = 3 * F;
    O2345_CUDA(cudaMemsetAsync(off, 0, 4 * (nv + 1), s));
    O2345_CUDA(cudaMemsetAsync(cursor, 0, 4 * nv, s));
    degree_kernel<<<cdiv(n3, 256), 256, 0, s>>>(cur, n3, off);
    scan_block_kernel<<<(int)Lo.nb, kSB, 0, s>>>(off, nv + 1, sums);
    scan_tops_kernel<<<1, kSB, 0, s>>>(sums, (int)Lo.nb);
    scan_add_kernel<<<(int)Lo.nb, kSB, 0, s>>>(off, nv + 1, sums);
    fill_kernel<<<cdiv(n3, 256), 256, 0, s>>>(cur, n3, off, cursor, adj);
    vertex_kernel<<<vb, 128, 0, s>>>(cur, off, adj, (int)nv, locked, val);
    if (rounds == 0) quadric_kernel<<<vb, 128, 0, s>>>(verts, cur, off, adj, (int)nv, Q);
    O2345_CUDA(cudaMemsetAsync(claim, 0xff, 8 * nv, s));
    propose_kernel<<<vb, 128, 0, s>>>(verts, cur, off, adj, locked, val, Q, (int)nv, target, key, claim);
    accept_kernel<<<vb, 128, 0, s>>>(cur, off, adj, target, key, claim, (int)nv, acc);
    O2345_LAUNCH_CHECK();
    O2345_TRY(o2345_compact(acc, nv, rows, nullptr, ctr + kAccepted, cs, stream));
    O2345_TRY(read_counters());   // the round's one host synchronisation
    const int64_t m = host[kAccepted], k = (F - target_faces + 1) / 2;
    if (m == 0) break;            // no legal collapse is left
    O2345_CUDA(cudaMemsetAsync(thresh, 0xff, 8, s));
    if (m > k) select_kernel<<<1, kSB, 0, s>>>(rows, (int)m, key, (int)k, thresh);
    O2345_CUDA(cudaMemsetAsync(flags, 1, F, s));
    apply_kernel<<<cdiv(m, 128), 128, 0, s>>>(rows, (int)m, key, thresh, target, off, adj, cur, flags, Q);
    O2345_LAUNCH_CHECK();
    O2345_TRY(o2345_compact(flags, F, rows, nullptr, ctr + kAlive, cs, stream));
    F -= 2 * (m < k ? m : k);
    if (F > 0) gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(cur, rows, F, nxt);
    O2345_LAUNCH_CHECK();
    int32_t* t = cur;
    cur = nxt, nxt = t;
    ++rounds;
  }
  O2345_CUDA(cudaMemsetAsync(flags, 0, nv, s));
  if (F > 0) mark_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, flags);
  O2345_TRY(o2345_compact(flags, nv, vertex_index, remap, ctr + kUsed, cs, stream));
  if (F > 0) renumber_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, remap, out_faces);
  counts_kernel<<<1, 1, 0, s>>>(ctr, F, rounds, out_counts);
  O2345_LAUNCH_CHECK();
#undef O2345_TRY
  return O2345_OK;
}
