// Isotropic remeshing (ops.remesh_mesh, o2345/mesh_remesh.py, simplify_mesh.py --remesh) and closest points on a
// mesh (ops.closest_points).  The rules are in include/o2345.h (o2345_remesh, o2345_closest_points).
//
//   closest   an LBVH over the reference faces (lbvh.cuh); one thread per point, a stack traversal nearer child first that
//             skips a node whose box distance, rounded downward and less a slack, exceeds the best squared distance so far;
//             each leaf's closest point is the 7-region test of mesh_common.cuh in fp64;
//   split     per round: vertex -> face adjacency (vertex_faces), one thread per face: the key of each of its long edges
//             (bits(fp32 squared length) << 32 | edge id) and the greatest (face max); one thread per face: the canonical
//             half-edges that hold the face max of each of their one or two faces split; ordered compaction numbers the
//             new vertices (edge order) and the new faces (face order); the counts are read on the host (the round's one
//             synchronisation) and checked against the capacities; one thread per split edge writes the midpoint, one per
//             split face rewrites it and appends its second half;
//   collapse  per round: adjacency, locks and valences (vertex_lock, mesh_common.cuh), one thread per unlocked vertex: its
//             shortest short legal neighbour and claims on both closed 1-rings (the simplifier's scheme), acceptance, then
//             u -> v and an ordered compaction of the surviving faces;
//   flip      per round: adjacency, locks, valences; one thread per face: each canonical interior half-edge's gain and
//             legality, claims on its four vertices keyed on (gain, edge id), acceptance and the two faces rewritten;
//   relax     adjacency and locks, one thread per vertex (Jacobi into a second buffer);
//   project   one thread per unlocked vertex: the closest point of the reference mesh.
//
// Every floating-point operation is an explicit round-to-nearest intrinsic (round-down for the pruning bound) in the order
// oracle/remesh_oracle.py repeats with numpy; selections are claims on 64-bit keys, so every output is independent of
// thread scheduling and bit-identical to the oracle.
#include <cfloat>
#include <cmath>

#include "lbvh.cuh"

namespace o2345 {
namespace {

enum { kErr = 0, kCount = 1, kCount2 = 2, kUsed = 3, kCtr = 4 };
constexpr uint64_t kNone = ~0ull;
constexpr int kMaxSplitRounds = 64;     // per iteration; a round that splits nothing ends the phase sooner
constexpr int kMaxGain = 1 << 30;
constexpr float kPadScale = 0x1p-13f;      // the LBVH's face-box pad (any pad >= 0 keeps the search exact)

// ----------------------------------------------------------------------------- closest point
struct Hit {
  double d2;
  int face;
  D3 q;
};

// the least (squared distance, face) over the faces of the LBVH (faces of leaf i: order[i], corners tri[9 i ..])
__device__ Hit closest_on_mesh(D3 p, int64_t nf, const int2* __restrict__ child, const float4* __restrict__ box,
                               const float* __restrict__ tri, const int32_t* __restrict__ order, double slack) {
  Hit best{INFINITY, INT32_MAX, {0.0, 0.0, 0.0}};
  auto bound = [&](int node) {   // the node box's squared distance to p, every step rounded downward, less the slack
    const float4 lo = __ldg(box + 2 * node), hi = __ldg(box + 2 * node + 1);
    const double L[3] = {lo.x, lo.y, lo.z}, H[3] = {hi.x, hi.y, hi.z}, P[3] = {p.x, p.y, p.z};
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double g = P[c] < L[c] ? __dsub_rd(L[c], P[c]) : (P[c] > H[c] ? __dsub_rd(P[c], H[c]) : 0.0);
      g = fmax(__dsub_rd(g, slack), 0.0);
      s = c == 0 ? __dmul_rd(g, g) : __dadd_rd(s, __dmul_rd(g, g));
    }
    return s;
  };
  const int first_leaf = (int)(nf - 1);
  int stack[kLbvhStack];
  int sp = 0, node = 0;
  while (true) {
    if (node >= first_leaf) {
      const int i = node - first_leaf;
      const float* t = tri + 9 * (int64_t)i;
      const D3 A = {__ldg(t), __ldg(t + 1), __ldg(t + 2)}, B = {__ldg(t + 3), __ldg(t + 4), __ldg(t + 5)},
               C = {__ldg(t + 6), __ldg(t + 7), __ldg(t + 8)};
      const Bary l = closest_point(p, A, B, C);
      const D3 q = {__dadd_rn(__dadd_rn(__dmul_rn(l.a, A.x), __dmul_rn(l.b, B.x)), __dmul_rn(l.c, C.x)),
                    __dadd_rn(__dadd_rn(__dmul_rn(l.a, A.y), __dmul_rn(l.b, B.y)), __dmul_rn(l.c, C.y)),
                    __dadd_rn(__dadd_rn(__dmul_rn(l.a, A.z), __dmul_rn(l.b, B.z)), __dmul_rn(l.c, C.z))};
      const D3 d = sub3(q, p);
      const double d2 = dot3(d, d);
      const int f = __ldg(order + i);
      if (d2 < best.d2 || (d2 == best.d2 && f < best.face)) best = {d2, f, q};
    } else {
      const int2 c = __ldg(child + node);
      const double b0 = bound(c.x), b1 = bound(c.y);
      const bool h0 = !(b0 > best.d2), h1 = !(b1 > best.d2);
      if (h0 && h1) {
        const bool first0 = b0 <= b1;
        stack[sp++] = first0 ? c.y : c.x;
        node = first0 ? c.x : c.y;
        continue;
      }
      if (h0 || h1) {
        node = h0 ? c.x : c.y;
        continue;
      }
    }
    // pop, dropping nodes that the best found since they were pushed excludes
    bool found = false;
    while (sp > 0 && !found) {
      node = stack[--sp];
      found = !(bound(node) > best.d2);
    }
    if (!found) return best;
  }
}

// the slack of the pruning bound: max |box coordinate| 2^-44 (geom: box lo xyz, hi xyz)
__device__ __forceinline__ double box_slack(const float* __restrict__ geom) {
  double m = 0.0;
  for (int c = 0; c < 6; ++c) m = fmax(m, fabs((double)geom[c]));
  return __dmul_rn(m, 0x1p-44);
}

__global__ void closest_kernel(const float* __restrict__ pts, int64_t n, int64_t nf, const int2* __restrict__ child,
                               const float4* __restrict__ box, const float* __restrict__ tri, const int32_t* __restrict__ order,
                               const float* __restrict__ geom, float* __restrict__ out, int32_t* __restrict__ face) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) {
    out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = __int_as_float(0x7fc00000);
    face[i] = -1;
    return;
  }
  const Hit h = closest_on_mesh({x, y, z}, nf, child, box, tri, order, box_slack(geom));
  out[3 * i] = __double2float_rn(h.q.x), out[3 * i + 1] = __double2float_rn(h.q.y), out[3 * i + 2] = __double2float_rn(h.q.z);
  face[i] = h.face;
}

__global__ void nan_kernel(float* __restrict__ out, int32_t* __restrict__ face, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = __int_as_float(0x7fc00000);
  face[i] = -1;
}

// ----------------------------------------------------------------------------- edges
__device__ __forceinline__ double len2(const float* __restrict__ V, int a, int b) {
  const D3 d = sub3(vert(V, b), vert(V, a));
  return dot3(d, d);
}

// The faces of edge ab among a's faces L[0, d): their count, the least (g) and another one (h, -1 when there is none).
__device__ __forceinline__ int edge_faces(const int32_t* __restrict__ F, const int32_t* __restrict__ L, int d, int b, int& g,
                                          int& h) {
  int cnt = 0;
  g = -1, h = -1;
  for (int i = 0; i < d; ++i)
    if (has(F, L[i], b)) {
      if (cnt == 0) g = L[i];
      else if (cnt == 1) h = L[i];
      ++cnt;
    }
  return cnt;
}

// ----------------------------------------------------------------------------- split
// One thread per face: fmax[f] := the greatest key (bits(fp32 len^2) << 32) | edge id of its long edges with one or two
// faces (0 when none; a long edge's key is > 0), fk[f] := the corner that starts that edge (-1 when none).  The edge id is
// the canonical half-edge 3 g + k of the edge's least face g.
__global__ void split_key_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                                 const int32_t* __restrict__ off, const int32_t* __restrict__ adj, double hi2,
                                 uint64_t* __restrict__ fmax_, int32_t* __restrict__ fk) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  uint64_t best = 0;
  int bk = -1;
  for (int k = 0; k < 3; ++k) {
    const int a = F[3 * f + k], b = F[3 * f + (k + 1) % 3];
    const double l2 = len2(V, a, b);
    if (!(l2 > hi2)) continue;
    int g, h;
    if (edge_faces(F, adj + off[a], off[a + 1] - off[a], b, g, h) > 2) continue;
    int kg = 0;
    while (!(F[3 * g + kg] == a && F[3 * g + (kg + 1) % 3] == b) && !(F[3 * g + kg] == b && F[3 * g + (kg + 1) % 3] == a)) ++kg;
    const uint64_t key = ((uint64_t)__float_as_uint(__double2float_rn(l2)) << 32) | (uint32_t)(3 * g + kg);
    if (key > best) best = key, bk = k;
  }
  fmax_[f] = best, fk[f] = bk;
}

// One thread per face: the half-edge 3 f + fk[f] (the face's greatest) splits when it is canonical (f is the edge's least
// face) and is the greatest of its other face too.  hflag [3 nf] is cleared by the caller.
__global__ void split_pick_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ off,
                                  const int32_t* __restrict__ adj, const uint64_t* __restrict__ fmax_,
                                  const int32_t* __restrict__ fk, uint8_t* __restrict__ hflag) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int k = fk[f];
  if (k < 0) return;
  const uint64_t key = fmax_[f];
  if ((int64_t)(uint32_t)key != 3 * f + k) return;   // not canonical: the least face decides
  const int a = F[3 * f + k], b = F[3 * f + (k + 1) % 3];
  int g, h;
  edge_faces(F, adj + off[a], off[a + 1] - off[a], b, g, h);
  if (h < 0 || fmax_[h] == key) hflag[3 * f + k] = 1;
}

// face flags: the face's greatest edge split
__global__ void split_faces_kernel(int64_t nf, const uint64_t* __restrict__ fmax_, const int32_t* __restrict__ fk,
                                   const uint8_t* __restrict__ hflag, uint8_t* __restrict__ fflag) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  fflag[f] = fk[f] >= 0 && hflag[(uint32_t)fmax_[f]];
}

// new vertex nv + i := the fp32 midpoint (a + b) * 0.5 of split half-edge rows[i]
__global__ void midpoint_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ rows, int m, int nv,
                                float* __restrict__ V) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int h = rows[i], f = h / 3, k = h % 3;
  const int64_t a = F[3 * f + k], b = F[3 * f + (k + 1) % 3];
#pragma unroll
  for (int c = 0; c < 3; ++c) V[3 * ((int64_t)nv + i) + c] = __fmul_rn(__fadd_rn(V[3 * a + c], V[3 * b + c]), 0.5f);
}

// split face rows[j] = (p, q, r) on edge pq (corners k, k + 1) with new vertex m: it becomes (p, m, r) and face nf + j
// is (m, q, r)
__global__ void split_apply_kernel(int32_t* __restrict__ F, const int32_t* __restrict__ rows, int m, int64_t nf, int nv,
                                   const uint64_t* __restrict__ fmax_, const int32_t* __restrict__ fk,
                                   const int32_t* __restrict__ hidx) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int64_t f = rows[j], g = nf + j;
  const int k = fk[f], mv = nv + hidx[(uint32_t)fmax_[f]];
  const int c[3] = {F[3 * f], F[3 * f + 1], F[3 * f + 2]};
#pragma unroll
  for (int t = 0; t < 3; ++t) F[3 * g + t] = c[t];
  F[3 * f + (k + 1) % 3] = mv;
  F[3 * g + k] = mv;
}

// ----------------------------------------------------------------------------- collapse
__global__ void vertex_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ off, const int32_t* __restrict__ adj,
                              int nv, uint8_t* __restrict__ locked, int32_t* __restrict__ val) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  locked[u] = vertex_lock(F, adj + off[u], off[u + 1] - off[u], u, val + u);
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

// Every unlocked u proposes its short legal neighbour v with the least (bits(fp32 len^2), v) whose collapse leaves no
// edge at v longer than hi (every other neighbour x of u: len^2(v, x) <= hi2) and claims both closed 1-rings with
// (bits << 32) | u.
__global__ void collapse_propose_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                                        const int32_t* __restrict__ adj, const uint8_t* __restrict__ locked,
                                        const int32_t* __restrict__ val, int nv, double lo2, double hi2,
                                        int32_t* __restrict__ target, uint64_t* __restrict__ key, uint64_t* __restrict__ claim) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  key[u] = kNone;
  if (locked[u]) return;
  const int32_t* L = adj + off[u];
  const int d = off[u + 1] - off[u];
  uint64_t best = kNone;
  for (int j = 0; j < d; ++j) {
    int x[2];
    others(F, L[j], u, x[0], x[1]);
    for (int t = 0; t < 2; ++t) {
      bool before = false;
      for (int i = 0; i < j && !before; ++i) before = has(F, L[i], x[t]);
      if (before) continue;
      const double l2 = len2(V, u, x[t]);
      if (!(l2 < lo2)) continue;
      const uint64_t c = ((uint64_t)__float_as_uint(__double2float_rn(l2)) << 32) | (uint32_t)x[t];
      if (c >= best || !legal_collapse(V, F, off, adj, val, u, x[t])) continue;
      bool ok = true;
      for (int i = 0; i < d && ok; ++i) {
        int y[2];
        others(F, L[i], u, y[0], y[1]);
        for (int s = 0; s < 2; ++s) ok &= y[s] == x[t] || !(len2(V, x[t], y[s]) > hi2);
      }
      if (ok) best = c;
    }
  }
  if (best == kNone) return;
  const int v = (int)(uint32_t)best;
  const uint64_t k = (best & 0xffffffff00000000ull) | (uint32_t)u;
  target[u] = v, key[u] = k;
  claim_ring(F, off, adj, u, k, claim);
  claim_ring(F, off, adj, v, k, claim);
}

__global__ void collapse_accept_kernel(const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                                       const int32_t* __restrict__ adj, const int32_t* __restrict__ target,
                                       const uint64_t* __restrict__ key, const uint64_t* __restrict__ claim, int nv,
                                       uint8_t* __restrict__ acc) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  uint64_t k = key[u];
  acc[u] = k != kNone && holds_ring(F, off, adj, u, k, claim) && holds_ring(F, off, adj, target[u], k, claim);
}

// u -> v: u's faces take v, the two faces of uv die (alive [nf] set to 1 by the caller)
__global__ void collapse_apply_kernel(const int32_t* __restrict__ list, int m, const int32_t* __restrict__ target,
                                      const int32_t* __restrict__ off, const int32_t* __restrict__ adj, int32_t* __restrict__ F,
                                      uint8_t* __restrict__ alive) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int u = list[i], v = target[u];
  for (int j = off[u]; j < off[u + 1]; ++j) {
    const int f = adj[j];
    if (has(F, f, v)) {
      alive[f] = 0;
      continue;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (F[3 * f + k] == u) F[3 * f + k] = v;
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

// ----------------------------------------------------------------------------- flip
__device__ __forceinline__ int dev2(int val, bool locked) {
  const int e = val - (locked ? 4 : 6);
  return e * e;
}

// One thread per face f, per corner k: the canonical half-edge ab (a = corner k) with exactly two faces, f = (a, b, c)
// and the other face holding b -> a with third vertex d.  The flip to cd is legal when c != d, cd is not an edge,
// val(a), val(b) > 3, and the new faces (a, d, c), (d, b, c) have normals whose fp64 dot with both old faces' normals is
// > 0; it proposes when it lowers the sum of (val - target)^2 over a, b, c, d and claims the four vertices with
// ((kMaxGain - gain) << 32) | (3 f + k).
__global__ void flip_propose_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                                    const int32_t* __restrict__ off, const int32_t* __restrict__ adj,
                                    const uint8_t* __restrict__ locked, const int32_t* __restrict__ val,
                                    uint64_t* __restrict__ hkey, uint64_t* __restrict__ claim) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  for (int k = 0; k < 3; ++k) {
    hkey[3 * f + k] = kNone;
    const int a = F[3 * f + k], b = F[3 * f + (k + 1) % 3], c = F[3 * f + (k + 2) % 3];
    int g, h;
    if (edge_faces(F, adj + off[a], off[a + 1] - off[a], b, g, h) != 2 || g != f) continue;
    int d = -1;
    for (int t = 0; t < 3; ++t)
      if (F[3 * h + t] == b && F[3 * h + (t + 1) % 3] == a) d = F[3 * h + (t + 2) % 3];
    if (d < 0 || d == c || val[a] <= 3 || val[b] <= 3) continue;
    bool cd = false;
    for (int j = off[c]; j < off[c + 1] && !cd; ++j) cd = has(F, adj[j], d);
    if (cd) continue;
    const int before = dev2(val[a], locked[a]) + dev2(val[b], locked[b]) + dev2(val[c], locked[c]) + dev2(val[d], locked[d]);
    const int after = dev2(val[a] - 1, locked[a]) + dev2(val[b] - 1, locked[b]) + dev2(val[c] + 1, locked[c]) +
                      dev2(val[d] + 1, locked[d]);
    const int gain = before - after;
    if (gain <= 0) continue;
    const D3 A = vert(V, a), B = vert(V, b), C = vert(V, c), Dd = vert(V, d);
    const D3 n0 = cross3(A, B, C), n1 = cross3(B, A, Dd), m0 = cross3(A, Dd, C), m1 = cross3(Dd, B, C);
    if (!(dot3(m0, n0) > 0.0 && dot3(m0, n1) > 0.0 && dot3(m1, n0) > 0.0 && dot3(m1, n1) > 0.0)) continue;
    const uint64_t key = ((uint64_t)(kMaxGain - gain) << 32) | (uint32_t)(3 * f + k);
    hkey[3 * f + k] = key;
    atomicMin((unsigned long long*)claim + a, (unsigned long long)key);
    atomicMin((unsigned long long*)claim + b, (unsigned long long)key);
    atomicMin((unsigned long long*)claim + c, (unsigned long long)key);
    atomicMin((unsigned long long*)claim + d, (unsigned long long)key);
  }
}

__global__ void flip_accept_kernel(const int32_t* __restrict__ F, int64_t nf, const int32_t* __restrict__ off,
                                   const int32_t* __restrict__ adj, const uint64_t* __restrict__ hkey,
                                   const uint64_t* __restrict__ claim, uint8_t* __restrict__ hflag) {
  int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= 3 * nf) return;
  const uint64_t key = hkey[h];
  bool ok = key != kNone;
  if (ok) {
    const int64_t f = h / 3;
    const int k = (int)(h % 3);
    const int a = F[3 * f + k], b = F[3 * f + (k + 1) % 3], c = F[3 * f + (k + 2) % 3];
    int g, o;
    edge_faces(F, adj + off[a], off[a + 1] - off[a], b, g, o);
    int d = -1;
    for (int t = 0; t < 3; ++t)
      if (F[3 * o + t] == b && F[3 * o + (t + 1) % 3] == a) d = F[3 * o + (t + 2) % 3];
    ok = claim[a] == key && claim[b] == key && claim[c] == key && claim[d] == key;
  }
  hflag[h] = ok;
}

// accepted flip rows[i] = 3 f + k: f := (a, d, c), its other face := (d, b, c).  (Reads only the two faces it rewrites;
// accepted flips share no vertex, so no face.)
__global__ void flip_apply_kernel(const int32_t* __restrict__ rows, int m, const int32_t* __restrict__ off,
                                  const int32_t* __restrict__ adj, int32_t* __restrict__ F) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int h = rows[i], f = h / 3, k = h % 3;
  const int a = F[3 * f + k], b = F[3 * f + (k + 1) % 3], c = F[3 * f + (k + 2) % 3];
  int g, o;
  edge_faces(F, adj + off[a], off[a + 1] - off[a], b, g, o);
  int d = -1;
  for (int t = 0; t < 3; ++t)
    if (F[3 * o + t] == b && F[3 * o + (t + 1) % 3] == a) d = F[3 * o + (t + 2) % 3];
  F[3 * f] = a, F[3 * f + 1] = d, F[3 * f + 2] = c;
  F[3 * o] = d, F[3 * o + 1] = b, F[3 * o + 2] = c;
}

// ----------------------------------------------------------------------------- relax, project
// One thread per vertex: an unlocked vertex moves to p + (d - n (d . n)), d = c - p, c the mean of its neighbours (summed
// in ascending index order in fp64), n its vertex normal rounded to fp32; everything else is copied.
__global__ void relax_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
                             const int32_t* __restrict__ adj, const uint8_t* __restrict__ locked, int nv,
                             float* __restrict__ out) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  if (locked[u]) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[3 * (int64_t)u + c] = V[3 * (int64_t)u + c];
    return;
  }
  const int32_t* L = adj + off[u];
  const int d = off[u + 1] - off[u];
  D3 s = {0.0, 0.0, 0.0};
  int cnt = 0, last = -1;
  while (true) {   // neighbours in ascending order: the least one above the last
    int next = INT32_MAX;
    for (int j = 0; j < d; ++j)
      for (int t = 0; t < 3; ++t) {
        const int x = F[3 * L[j] + t];
        if (x != u && x > last && x < next) next = x;
      }
    if (next == INT32_MAX) break;
    const D3 q = vert(V, next);
    s = {__dadd_rn(s.x, q.x), __dadd_rn(s.y, q.y), __dadd_rn(s.z, q.z)};
    ++cnt, last = next;
  }
  const double n_ = (double)cnt;
  const D3 c = {__ddiv_rn(s.x, n_), __ddiv_rn(s.y, n_), __ddiv_rn(s.z, n_)};
  const D3 r = vertex_normal(V, F, L, d);
  const D3 n = {(double)__double2float_rn(r.x), (double)__double2float_rn(r.y), (double)__double2float_rn(r.z)};
  const D3 p = vert(V, u), e = sub3(c, p);
  const double t = dot3(e, n);
  out[3 * (int64_t)u] = __double2float_rn(__dadd_rn(p.x, __dsub_rn(e.x, __dmul_rn(n.x, t))));
  out[3 * (int64_t)u + 1] = __double2float_rn(__dadd_rn(p.y, __dsub_rn(e.y, __dmul_rn(n.y, t))));
  out[3 * (int64_t)u + 2] = __double2float_rn(__dadd_rn(p.z, __dsub_rn(e.z, __dmul_rn(n.z, t))));
}

__global__ void project_kernel(float* __restrict__ V, const uint8_t* __restrict__ locked, int nv, int64_t nf,
                               const int2* __restrict__ child, const float4* __restrict__ box, const float* __restrict__ tri,
                               const int32_t* __restrict__ order, const float* __restrict__ geom) {
  int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv || locked[u]) return;
  const Hit h = closest_on_mesh(vert(V, u), nf, child, box, tri, order, box_slack(geom));
  V[3 * (int64_t)u] = __double2float_rn(h.q.x), V[3 * (int64_t)u + 1] = __double2float_rn(h.q.y);
  V[3 * (int64_t)u + 2] = __double2float_rn(h.q.z);
}

// ----------------------------------------------------------------------------- output
__global__ void mark_kernel(const int32_t* __restrict__ F, int64_t n3, uint8_t* __restrict__ used) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) used[F[i]] = 1;
}

__global__ void out_verts_kernel(const float* __restrict__ V, const int32_t* __restrict__ rows, int64_t n, float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = rows[i];
  out[3 * i] = V[3 * r], out[3 * i + 1] = V[3 * r + 1], out[3 * i + 2] = V[3 * r + 2];
}

__global__ void renumber_kernel(const int32_t* __restrict__ F, int64_t n3, const int32_t* __restrict__ remap,
                                int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) out[i] = remap[F[i]];
}

// The scratch of o2345_closest_points.
struct ClosestScratch {
  int64_t nv, nf;
  Carver c;
  Lbvh bvh{c, nf};
};

// The scratch of o2345_remesh, carved in this order (a Carver without a base only measures it).
struct RemeshScratch {
  int64_t nv, nf, vcap, fcap;
  Carver c;
  Lbvh bvh{c, nf};
  int64_t hmax = 3 * fcap > vcap ? 3 * fcap : vcap;
  int32_t* ctr = c.take<int32_t>(kCtr);
  float* va = c.take<float>(3 * vcap);
  float* vb = c.take<float>(3 * vcap);
  int32_t* fa = c.take<int32_t>(3 * fcap);
  int32_t* fb = c.take<int32_t>(3 * fcap);
  int32_t* off = c.take<int32_t>(vcap + 1);
  int32_t* sums = c.take<int32_t>(scan_blocks(vcap + 1));
  int32_t* cursor = c.take<int32_t>(vcap);
  int32_t* adj = c.take<int32_t>(3 * fcap);
  int32_t* val = c.take<int32_t>(vcap);
  uint8_t* locked = c.take<uint8_t>(vcap);
  uint64_t* hkey = c.take<uint64_t>(3 * fcap);
  uint64_t* fmax = c.take<uint64_t>(fcap);
  int32_t* fk = c.take<int32_t>(fcap);
  uint8_t* hflag = c.take<uint8_t>(hmax);
  int32_t* hidx = c.take<int32_t>(3 * fcap);
  int32_t* rows = c.take<int32_t>(hmax);
  int32_t* cscratch = c.take<int32_t>(o2345_compact_scratch_ints(hmax));
  uint8_t* fflag = c.take<uint8_t>(fcap);
  int32_t* frows = c.take<int32_t>(fcap);
  uint64_t* claim = c.take<uint64_t>(vcap);
  uint64_t* vkey = c.take<uint64_t>(vcap);
  int32_t* target = c.take<int32_t>(vcap);
  int32_t* remap = c.take<int32_t>(vcap);
};

bool sizes_ok(int64_t nv, int64_t nf) { return nv >= 1 && nv <= INT32_MAX - 1 && nf >= 1 && nf <= (1 << 29); }

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_closest_points_scratch_bytes(int64_t nv, int64_t nf) {
  if (nv < 0 || nv > INT32_MAX - 1 || nf < 0 || nf > (1 << 29)) return -1;
  return ClosestScratch{nv, nf, {}}.c.bytes;
}

extern "C" int o2345_closest_points(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* points,
                                    int64_t n, void* scratch, int64_t scratch_bytes, float* out_points, int32_t* out_face,
                                    o2345_stream_t stream) {
  O2345_CHECK_ARG(nv >= 0 && nv <= INT32_MAX - 1 && nf >= 0 && nf <= (1 << 29) && n >= 0 && n <= INT32_MAX,
                  "need 0 <= nv < 2^31-1, 0 <= nf <= 2^29 and 0 <= n < 2^31");
  O2345_CHECK_ARG((verts || nv == 0) && (faces || nf == 0) && (points && out_points && out_face || n == 0),
                  "verts, faces, points, out_points and out_face are required");
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_closest_points_scratch_bytes(nv, nf),
                  "scratch smaller than o2345_closest_points_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  ClosestScratch S{nv, nf, {(char*)scratch}};
  O2345_CUDA(cudaMemsetAsync(S.bvh.ctr, 0, 4 * 8, s));
  if (nv > 0 || nf > 0) {
    int32_t err = 0;
    O2345_TRY(mesh_check(verts, nv, faces, nf, nullptr, S.bvh.ctr, s));
    O2345_CUDA(cudaMemcpyAsync(&err, S.bvh.ctr, 4, cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    O2345_TRY(mesh_check_status(err, __func__));
  }
  if (n == 0) return O2345_OK;
  if (nf == 0) {
    nan_kernel<<<cdiv(n, 256), 256, 0, s>>>(out_points, out_face, n);
    O2345_LAUNCH_CHECK();
    return O2345_OK;
  }
  O2345_TRY(S.bvh.build(verts, nv, faces, nf, kPadScale, s));
  closest_kernel<<<cdiv(n, 128), 128, 0, s>>>(points, n, nf, S.bvh.child, S.bvh.box, S.bvh.tri, S.bvh.order, S.bvh.geom,
                                              out_points, out_face);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int64_t o2345_remesh_scratch_bytes(int64_t nv, int64_t nf, int64_t vertex_capacity, int64_t face_capacity) {
  if (!sizes_ok(nv, nf) || vertex_capacity < nv || vertex_capacity > INT32_MAX - 1 || face_capacity < nf ||
      face_capacity > (1 << 29))
    return -1;
  return RemeshScratch{nv, nf, vertex_capacity, face_capacity, {}}.c.bytes;
}

extern "C" int o2345_remesh(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float target_length,
                            int iterations, int64_t vertex_capacity, int64_t face_capacity, void* scratch,
                            int64_t scratch_bytes, float* out_verts, int32_t* out_faces, int64_t* counts_host,
                            o2345_stream_t stream) {
  O2345_CHECK_ARG(verts && faces && out_verts && out_faces && counts_host, "verts, faces, out_verts, out_faces and counts_host are required");
  O2345_CHECK_ARG(sizes_ok(nv, nf), "need 1 <= nv < 2^31-1 and 1 <= nf <= 2^29");
  O2345_CHECK_ARG(target_length >= 0x1p-60f, "target_length must be >= 2^-60 (+inf collapses as far as the rules allow)");
  O2345_CHECK_ARG(iterations >= 0 && iterations <= 1000, "need 0 <= iterations <= 1000");
  O2345_CHECK_ARG(vertex_capacity <= INT32_MAX - 1 && face_capacity <= (1 << 29), "capacities out of range");
  if (vertex_capacity < nv || face_capacity < nf) {
    counts_host[0] = nv, counts_host[1] = nf;
    set_error("%s: the capacities are smaller than the input", __func__);
    return O2345_ENOSPC;
  }
  O2345_CHECK_ARG(scratch && scratch_bytes >= o2345_remesh_scratch_bytes(nv, nf, vertex_capacity, face_capacity),
                  "scratch smaller than o2345_remesh_scratch_bytes");
  O2345_CHECK_ARG(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  RemeshScratch S{nv, nf, vertex_capacity, face_capacity, {(char*)scratch}};
  const double Ld = (double)target_length, hi = Ld * (4.0 / 3.0), lo = Ld * 0.8, hi2 = hi * hi, lo2 = lo * lo;
  int32_t host[kCtr];
  auto read_counters = [&]() {
    O2345_CUDA(cudaMemcpyAsync(host, S.ctr, sizeof(host), cudaMemcpyDeviceToHost, s));
    O2345_CUDA(cudaStreamSynchronize(s));
    return O2345_OK;
  };

  O2345_CUDA(cudaMemsetAsync(S.ctr, 0, 4 * kCtr, s));
  O2345_TRY(mesh_check(verts, nv, faces, nf, S.fflag, S.ctr + kErr, s));
  O2345_TRY(o2345_compact(S.fflag, nf, S.frows, nullptr, S.ctr + kCount, S.cscratch, stream));
  O2345_TRY(read_counters());
  O2345_TRY(mesh_check_status(host[kErr], __func__));
  int64_t F = host[kCount], NV = nv;
  O2345_CUDA(cudaMemcpyAsync(S.va, verts, 12 * nv, cudaMemcpyDeviceToDevice, s));
  if (F > 0) gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(faces, S.frows, F, S.fa);
  O2345_LAUNCH_CHECK();
  O2345_TRY(S.bvh.build(verts, nv, faces, nf, kPadScale, s));   // the reference surface: the input as given
  float *V = S.va, *V2 = S.vb;
  int32_t *cur = S.fa, *nxt = S.fb;
  int64_t split_rounds = 0, collapse_rounds = 0, flip_rounds = 0;
  auto adjacency = [&]() {
    O2345_TRY(vertex_faces(cur, F, NV, S.off, S.sums, S.cursor, S.adj, s));
    vertex_kernel<<<cdiv(NV, 128), 128, 0, s>>>(cur, S.off, S.adj, (int)NV, S.locked, S.val);
    O2345_LAUNCH_CHECK();
    return O2345_OK;
  };

  for (int it = 0; it < iterations && F > 0; ++it) {
    // 1. split
    for (int r = 0; r < kMaxSplitRounds; ++r) {
      O2345_TRY(vertex_faces(cur, F, NV, S.off, S.sums, S.cursor, S.adj, s));
      split_key_kernel<<<cdiv(F, 128), 128, 0, s>>>(V, cur, F, S.off, S.adj, hi2, S.fmax, S.fk);
      O2345_CUDA(cudaMemsetAsync(S.hflag, 0, 3 * F, s));
      split_pick_kernel<<<cdiv(F, 128), 128, 0, s>>>(cur, F, S.off, S.adj, S.fmax, S.fk, S.hflag);
      split_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(F, S.fmax, S.fk, S.hflag, S.fflag);
      O2345_LAUNCH_CHECK();
      O2345_TRY(o2345_compact(S.hflag, 3 * F, S.rows, S.hidx, S.ctr + kCount, S.cscratch, stream));
      O2345_TRY(o2345_compact(S.fflag, F, S.frows, nullptr, S.ctr + kCount2, S.cscratch, stream));
      O2345_TRY(read_counters());   // the round's one host synchronisation
      const int64_t m = host[kCount], mf = host[kCount2];
      if (m == 0) break;
      if (NV + m > vertex_capacity || F + mf > face_capacity) {
        counts_host[0] = NV + m, counts_host[1] = F + mf;
        set_error("%s: a split round needs %lld vertices and %lld faces", __func__, (long long)(NV + m), (long long)(F + mf));
        return O2345_ENOSPC;
      }
      midpoint_kernel<<<cdiv(m, 128), 128, 0, s>>>(cur, S.rows, (int)m, (int)NV, V);
      split_apply_kernel<<<cdiv(mf, 128), 128, 0, s>>>(cur, S.frows, (int)mf, F, (int)NV, S.fmax, S.fk, S.hidx);
      O2345_LAUNCH_CHECK();
      NV += m, F += mf;
      ++split_rounds;
    }
    // 2. collapse: every round removes 2 faces per accepted collapse, so there are at most F / 2 rounds
    while (F > 0) {
      O2345_TRY(adjacency());
      O2345_CUDA(cudaMemsetAsync(S.claim, 0xff, 8 * NV, s));
      collapse_propose_kernel<<<cdiv(NV, 128), 128, 0, s>>>(V, cur, S.off, S.adj, S.locked, S.val, (int)NV, lo2, hi2,
                                                            S.target, S.vkey, S.claim);
      collapse_accept_kernel<<<cdiv(NV, 128), 128, 0, s>>>(cur, S.off, S.adj, S.target, S.vkey, S.claim, (int)NV, S.hflag);
      O2345_LAUNCH_CHECK();
      O2345_TRY(o2345_compact(S.hflag, NV, S.rows, nullptr, S.ctr + kCount, S.cscratch, stream));
      O2345_TRY(read_counters());
      const int64_t m = host[kCount];
      if (m == 0) break;
      O2345_CUDA(cudaMemsetAsync(S.fflag, 1, F, s));
      collapse_apply_kernel<<<cdiv(m, 128), 128, 0, s>>>(S.rows, (int)m, S.target, S.off, S.adj, cur, S.fflag);
      O2345_LAUNCH_CHECK();
      O2345_TRY(o2345_compact(S.fflag, F, S.frows, nullptr, S.ctr + kCount, S.cscratch, stream));
      F -= 2 * m;
      if (F > 0) gather_faces_kernel<<<cdiv(F, 256), 256, 0, s>>>(cur, S.frows, F, nxt);
      O2345_LAUNCH_CHECK();
      int32_t* t = cur;
      cur = nxt, nxt = t;
      ++collapse_rounds;
    }
    // 3. flip: every accepted flip lowers the integer sum of (val - target)^2 over the mesh, so the rounds end
    while (F > 0) {
      O2345_TRY(adjacency());
      O2345_CUDA(cudaMemsetAsync(S.claim, 0xff, 8 * NV, s));
      flip_propose_kernel<<<cdiv(F, 128), 128, 0, s>>>(V, cur, F, S.off, S.adj, S.locked, S.val, S.hkey, S.claim);
      flip_accept_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, F, S.off, S.adj, S.hkey, S.claim, S.hflag);
      O2345_LAUNCH_CHECK();
      O2345_TRY(o2345_compact(S.hflag, 3 * F, S.rows, nullptr, S.ctr + kCount, S.cscratch, stream));
      O2345_TRY(read_counters());
      const int64_t m = host[kCount];
      if (m == 0) break;
      flip_apply_kernel<<<cdiv(m, 128), 128, 0, s>>>(S.rows, (int)m, S.off, S.adj, cur);
      O2345_LAUNCH_CHECK();
      ++flip_rounds;
    }
    if (F == 0) break;
    // 4. relax (Jacobi) and 5. project
    O2345_TRY(adjacency());
    relax_kernel<<<cdiv(NV, 128), 128, 0, s>>>(V, cur, S.off, S.adj, S.locked, (int)NV, V2);
    project_kernel<<<cdiv(NV, 128), 128, 0, s>>>(V2, S.locked, (int)NV, nf, S.bvh.child, S.bvh.box, S.bvh.tri, S.bvh.order,
                                                 S.bvh.geom);
    O2345_LAUNCH_CHECK();
    float* t = V;
    V = V2, V2 = t;
  }

  O2345_CUDA(cudaMemsetAsync(S.hflag, 0, NV, s));
  if (F > 0) mark_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, S.hflag);
  O2345_TRY(o2345_compact(S.hflag, NV, S.rows, S.remap, S.ctr + kUsed, S.cscratch, stream));
  O2345_TRY(read_counters());
  const int64_t nout = host[kUsed];
  if (nout > 0) out_verts_kernel<<<cdiv(nout, 256), 256, 0, s>>>(V, S.rows, nout, out_verts);
  if (F > 0) renumber_kernel<<<cdiv(3 * F, 256), 256, 0, s>>>(cur, 3 * F, S.remap, out_faces);
  O2345_LAUNCH_CHECK();
  counts_host[0] = nout, counts_host[1] = F, counts_host[2] = split_rounds, counts_host[3] = collapse_rounds;
  counts_host[4] = flip_rounds;
  return O2345_OK;
}
