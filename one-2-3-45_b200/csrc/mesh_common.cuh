// Shared pieces of the mesh kernels (metrics.cu, simplify.cu, texture.cu, project.cu, clean.cu, ao.cu): fp64 vectors from the fp32 vertices with
// explicit round-to-nearest operations in the order the numpy oracles repeat (no FMA contraction), the input check and
// the vertex -> face adjacency.
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
