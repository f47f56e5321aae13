// Shared pieces of the mesh kernels (metrics.cu, simplify.cu, texture.cu, project.cu): fp64 vectors from the fp32 vertices with
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

}  // namespace o2345
