// Shared pieces of the mesh kernels (metrics.cu, simplify.cu, texture.cu, project.cu, clean.cu, ao.cu, remesh.cu): fp64
// vectors from the fp32 vertices with explicit round-to-nearest operations in the order the numpy oracles repeat (no FMA
// contraction), the 7-region closest point, the vertex normal, the simplifier's locks and legal collapses, the input check
// and the vertex -> face adjacency.
#pragma once
#include "common.cuh"

namespace o2345 {

struct D3 {
  double x, y, z;
};

__device__ __forceinline__ D3 vert(const float* __restrict__ V, int i) {
  return {(double)__ldg(V + 3 * (int64_t)i), (double)__ldg(V + 3 * (int64_t)i + 1), (double)__ldg(V + 3 * (int64_t)i + 2)};
}

__device__ __forceinline__ D3 sub3(D3 a, D3 b) { return {__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)}; }

__device__ __forceinline__ double dot3(D3 a, D3 b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}

// (b - a) x (c - a): twice the area vector of triangle abc
__device__ __forceinline__ D3 cross3(D3 a, D3 b, D3 c) {
  D3 e1 = sub3(b, a), e2 = sub3(c, a);
  return {__dsub_rn(__dmul_rn(e1.y, e2.z), __dmul_rn(e1.z, e2.y)), __dsub_rn(__dmul_rn(e1.z, e2.x), __dmul_rn(e1.x, e2.z)),
          __dsub_rn(__dmul_rn(e1.x, e2.y), __dmul_rn(e1.y, e2.x))};
}

// a / |a| in fp64; false when |a| is not a positive finite number
__device__ __forceinline__ bool unit3(D3 a, D3& out) {
  double l = __dsqrt_rn(dot3(a, a));
  if (!(l > 0.0 && l < INFINITY)) return false;
  out = {__ddiv_rn(a.x, l), __ddiv_rn(a.y, l), __ddiv_rn(a.z, l)};
  return true;
}

// Barycentrics (of a, b, c) of the point of triangle abc closest to p: the 7-region test (three corners, three edges,
// the interior), in fp64.  A zero-length edge or a zero-area interior cannot divide by zero: the corner a is taken.
struct Bary {
  double a, b, c;
};

__device__ __forceinline__ Bary closest_point(D3 p, D3 a, D3 b, D3 c) {
  D3 ab = sub3(b, a), ac = sub3(c, a), ap = sub3(p, a);
  double d1 = dot3(ab, ap), d2 = dot3(ac, ap);
  if (d1 <= 0.0 && d2 <= 0.0) return {1.0, 0.0, 0.0};
  D3 bp = sub3(p, b);
  double d3 = dot3(ab, bp), d4 = dot3(ac, bp);
  if (d3 >= 0.0 && d4 <= d3) return {0.0, 1.0, 0.0};
  double vc = __dsub_rn(__dmul_rn(d1, d4), __dmul_rn(d3, d2));
  if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
    double t = __dsub_rn(d1, d3), v = t > 0.0 ? __ddiv_rn(d1, t) : 0.0;
    return {__dsub_rn(1.0, v), v, 0.0};
  }
  D3 cp = sub3(p, c);
  double d5 = dot3(ab, cp), d6 = dot3(ac, cp);
  if (d6 >= 0.0 && d5 <= d6) return {0.0, 0.0, 1.0};
  double vb = __dsub_rn(__dmul_rn(d5, d2), __dmul_rn(d1, d6));
  if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
    double t = __dsub_rn(d2, d6), w = t > 0.0 ? __ddiv_rn(d2, t) : 0.0;
    return {__dsub_rn(1.0, w), 0.0, w};
  }
  double va = __dsub_rn(__dmul_rn(d3, d6), __dmul_rn(d5, d4));
  double e43 = __dsub_rn(d4, d3), e56 = __dsub_rn(d5, d6);
  if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) {
    double t = __dadd_rn(e43, e56), w = t > 0.0 ? __ddiv_rn(e43, t) : 0.0;
    return {0.0, __dsub_rn(1.0, w), w};
  }
  double den = __dadd_rn(__dadd_rn(va, vb), vc);
  if (!(den > 0.0)) return {1.0, 0.0, 0.0};
  double v = __ddiv_rn(vb, den), w = __ddiv_rn(vc, den);
  return {__dsub_rn(__dsub_rn(1.0, v), w), v, w};
}

// The unit normal of a vertex with faces L[0, d): the sum of the faces' (B - A) x (C - A) in that (ascending face) order
// in fp64, divided by its length; (0, 0, 0) for no faces or a zero sum.  o2345_vertex_normals rounds it once to fp32.
__device__ __forceinline__ D3 vertex_normal(const float* __restrict__ V, const int32_t* __restrict__ F,
                                            const int32_t* __restrict__ L, int d) {
  D3 s = {0.0, 0.0, 0.0};
  for (int j = 0; j < d; ++j) {
    int64_t f = L[j];
    D3 n = cross3(vert(V, F[3 * f]), vert(V, F[3 * f + 1]), vert(V, F[3 * f + 2]));
    s = {__dadd_rn(s.x, n.x), __dadd_rn(s.y, n.y), __dadd_rn(s.z, n.z)};
  }
  D3 r = {0.0, 0.0, 0.0};
  unit3(s, r);
  return r;
}

// ----------------------------------------------------------------------------- half-edge collapse rules
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

// Counts u's distinct neighbours (*val) and returns whether u is locked: unless every edge at u has exactly two faces
// and its faces form one closed fan (a vertex without faces is locked).  L = adj + off[u], d = its face count.
__device__ __forceinline__ bool vertex_lock(const int32_t* __restrict__ F, const int32_t* __restrict__ L, int d, int u,
                                            int32_t* val) {
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
  *val = nval;
  return !ok;
}

// The collapse u -> v for an unlocked u (every edge at u has two faces) is legal: the link condition (the vertices
// adjacent to both are exactly the two opposite uv), valences (both opposite >= 4, val(u) + val(v) - 4 >= 3) and no face
// of u without v flips or collapses (n' . n > 0 in fp64).  simplify.cu and remesh.cu.
__device__ __forceinline__ bool legal_collapse(const float* __restrict__ V, const int32_t* __restrict__ F, const int32_t* __restrict__ off,
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

// the three corner indices of a face lie in [0, nv)
__device__ __forceinline__ bool face_ok(const int c[3], int64_t nv) {
  return c[0] >= 0 && c[0] < nv && c[1] >= 0 && c[1] < nv && c[2] >= 0 && c[2] < nv;
}

// mesh_common.cu.  Launches the input check of a mesh: *err |= 1 for a face index outside [0, nv), |= 2 for a non-finite
// vertex coordinate (*err is cleared by the caller); flags[f] (when not null) := face f has three distinct indices in
// [0, nv).  mesh_check_status turns the bits, once read on the host, into O2345_OK or O2345_EINVAL with its message.
int mesh_check(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, uint8_t* flags, int32_t* err,
               cudaStream_t stream);
int mesh_check_status(int32_t err, const char* func);

// mesh_common.cu.  Vertex -> face adjacency of faces [nf,3] whose indices all lie in [0, nv): off [nv + 1] the exclusive
// offsets (off[nv] = 3 nf), adj [3 nf] the faces of vertex u at adj[off[u] .. off[u + 1]), ascending (a face that holds u
// twice is listed twice).  Scratch: sums [scan_blocks(nv + 1)], cursor [nv].  Degree count, scan_i32, scatter, then one
// thread per vertex sorts its list (the scatter's order depends on scheduling).
int vertex_faces(const int32_t* faces, int64_t nf, int64_t nv, int32_t* off, int32_t* sums, int32_t* cursor, int32_t* adj,
                 cudaStream_t stream);

// mesh_common.cu.  order[0, n) := 0 .. n-1 sorted stably by key[i] (>= 0) over the key's low `bits` bits: one stable
// split per bit, least significant first, each on a scan_i32 of the one bits (clean.cu's faces by component, ao.cu's faces
// by Morton code).  next, ones: n int32 each; sums: scan_blocks(n); n_ones: one int32.  order and next swap with every
// pass, so the sorted list is wherever order points on return.
int radix_sort_i32(int32_t*& order, int32_t*& next, const int32_t* key, int64_t n, int bits, int32_t* ones, int32_t* sums,
                   int32_t* n_ones, cudaStream_t stream);

// Union-find over n elements (texture.cu's chart components, clean.cu's vertex components).  Parents only ever point at
// lower indices, so every set ends rooted at its least element.
__device__ __forceinline__ int find_root(const int32_t* parent, int x) {
  for (int p = parent[x]; p != x; p = parent[x]) x = p;
  return x;
}

// Hooks the larger of the roots of a and b under the smaller (atomicMin); *changed := 1 when the roots differed.
__device__ __forceinline__ void unite(int32_t* parent, int a, int b, int32_t* changed) {
  int ra = find_root(parent, a), rb = find_root(parent, b);
  if (ra != rb) {
    atomicMin(parent + max(ra, rb), min(ra, rb));
    *changed = 1;
  }
}

// mesh_common.cu.  p[i] := i for i in [0, n).
int iota_i32(int32_t* p, int64_t n, cudaStream_t stream);
// mesh_common.cu.  One pass's tail: every parent[i] := its root, then *again := *changed (read on the host), *changed := 0.
int union_find_settle(int32_t* parent, int64_t n, int32_t* changed, bool& again, cudaStream_t stream);

// parent[0, n) := the sets joined by hook(), each element pointing at its set's least element: parent := identity, then
// passes of hook() (which launches the caller's kernel of unite() calls on `changed`) each followed by one compression,
// until a pass joins nothing.  Synchronises once per pass.
template <class Hook>
int union_find(int32_t* parent, int64_t n, int32_t* changed, Hook hook, cudaStream_t stream) {
  O2345_TRY(iota_i32(parent, n, stream));
  O2345_CUDA(cudaMemsetAsync(changed, 0, 4, stream));
  for (bool again = true; again;) {
    O2345_TRY(hook());
    O2345_TRY(union_find_settle(parent, n, changed, again, stream));
  }
  return O2345_OK;
}

}  // namespace o2345
