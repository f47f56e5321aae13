// Block-parallel marching cubes on the dense -sdf grid (row B10 of SURVEY.md section 8).
// Replaces mcubes.marching_cubes (PyMCubes, single CPU thread; reference
// sparse_neus_renderer.py:932) and the 64 device->host chunk copies of extract_fields (:901-904).
//
//   classify   one thread per lattice point: the 8-corner case index of the cell it anchors,
//              and one flag per owned lattice edge (+x,+y,+z) whose end points straddle iso;
//   compact    (o2345_compact) -> shared vertex ids, one per crossing edge, ascending edge order;
//   emit       vertices by linear interpolation in float64 index units (PyMCubes semantics),
//              triangles through the generated case table (o2345/mc_tables.py).
#include "common.cuh"

namespace o2345 {
namespace {

__global__ void mc_classify_kernel(const float* __restrict__ u, int R, float iso, uint8_t* __restrict__ cases,
                                   uint8_t* __restrict__ cell_flags, uint8_t* __restrict__ edge_flags) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t n = (int64_t)R * R * R;
  if (i >= n) return;
  int z = (int)(i % R), y = (int)((i / R) % R), x = (int)(i / ((int64_t)R * R));
  bool in0 = u[i] > iso;
  bool hx = x + 1 < R, hy = y + 1 < R, hz = z + 1 < R;
  edge_flags[3 * i + 0] = hx && ((u[i + (int64_t)R * R] > iso) != in0);
  edge_flags[3 * i + 1] = hy && ((u[i + R] > iso) != in0);
  edge_flags[3 * i + 2] = hz && ((u[i + 1] > iso) != in0);
  if (hx && hy && hz) {
    int c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int64_t j = i + (int64_t)(k & 1) * R * R + (int64_t)((k >> 1) & 1) * R + ((k >> 2) & 1);
      c |= (u[j] > iso ? 1 : 0) << k;
    }
    int64_t cell = ((int64_t)x * (R - 1) + y) * (R - 1) + z;
    cases[cell] = (uint8_t)c;
    cell_flags[cell] = (c != 0 && c != 255) ? 1 : 0;
  }
}

__global__ void mc_vertices_kernel(const float* __restrict__ u, int R, double iso, const int32_t* __restrict__ edges,
                                   const int32_t* __restrict__ count, double* __restrict__ verts) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  int e = edges[i];
  int axis = e % 3;
  int64_t p = e / 3;
  int z = (int)(p % R), y = (int)((p / R) % R), x = (int)(p / ((int64_t)R * R));
  int64_t q = p + (axis == 0 ? (int64_t)R * R : axis == 1 ? R : 1);
  double f0 = (double)u[p], f1 = (double)u[q];
  double t = (iso - f0) / (f1 - f0);
  double v[3] = {(double)x, (double)y, (double)z};
  v[axis] += t;
  verts[3 * (int64_t)i] = v[0], verts[3 * (int64_t)i + 1] = v[1], verts[3 * (int64_t)i + 2] = v[2];
}

__global__ void mc_tri_counts_kernel(const uint8_t* __restrict__ cases, const int32_t* __restrict__ cells,
                                     const int32_t* __restrict__ count, const uint8_t* __restrict__ n_tri,
                                     int32_t* __restrict__ counts, int64_t max_cells) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_cells) return;
  counts[i] = i < *count ? n_tri[cases[cells[i]]] : 0;
}

__global__ void mc_triangles_kernel(const uint8_t* __restrict__ cases, int R, const int32_t* __restrict__ cells,
                                    const int32_t* __restrict__ count, const int32_t* __restrict__ tri_offs,
                                    const int8_t* __restrict__ tri_table, const uint8_t* __restrict__ n_tri,
                                    const int8_t* __restrict__ edge_owner, const int32_t* __restrict__ vert_index,
                                    int32_t* __restrict__ tris) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  int cell = cells[i];
  int C = R - 1;
  int z = cell % C, y = (cell / C) % C, x = cell / (C * C);
  int c = cases[cell];
  int nt = n_tri[c];
  int64_t o = tri_offs[i];
  for (int t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) {
      int e = tri_table[c * 16 + 3 * t + j];
      const int8_t* ow = edge_owner + 4 * e;
      int64_t p = ((int64_t)(x + ow[0]) * R + (y + ow[1])) * R + (z + ow[2]);
      tris[3 * (o + t) + j] = vert_index[3 * p + ow[3]];
    }
}

}  // namespace
}  // namespace o2345

using namespace o2345;

extern "C" int o2345_mc_classify(const float* u, int R, float iso, uint8_t* cases, uint8_t* cell_flags,
                                 uint8_t* edge_flags, o2345_stream_t stream) {
  O2345_CHECK_ARG(u && cases && cell_flags && edge_flags, "null pointer");
  O2345_CHECK_ARG(R >= 2 && R <= 812, "grid side out of range (3*R^3 must fit int32)");
  int64_t n = (int64_t)R * R * R;
  mc_classify_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(u, R, iso, cases, cell_flags, edge_flags);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_mc_vertices(const float* u, int R, float iso, const int32_t* edges, const int32_t* count,
                                 int64_t max_verts, double* verts, o2345_stream_t stream) {
  O2345_CHECK_ARG(u && edges && count && verts, "null pointer");
  if (max_verts == 0) return O2345_OK;
  mc_vertices_kernel<<<cdiv(max_verts, 256), 256, 0, (cudaStream_t)stream>>>(u, R, (double)iso, edges, count, verts);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

extern "C" int o2345_mc_tri_offsets(const uint8_t* cases, const int32_t* cells, const int32_t* count,
                                    int64_t max_cells, const uint8_t* n_tri_table, int32_t* offsets,
                                    int32_t* total, int32_t* scratch, o2345_stream_t stream) {
  O2345_CHECK_ARG(cases && cells && count && n_tri_table && offsets && total && scratch, "null pointer");
  if (max_cells == 0) return O2345_OK;
  cudaStream_t st = (cudaStream_t)stream;
  mc_tri_counts_kernel<<<cdiv(max_cells, 256), 256, 0, st>>>(cases, cells, count, n_tri_table, offsets, max_cells);
  O2345_LAUNCH_CHECK();
  return scan_i32(offsets, max_cells, scratch, total, st);
}

extern "C" int o2345_mc_triangles(const uint8_t* cases, int R, const int32_t* cells, const int32_t* count,
                                  int64_t max_cells, const int32_t* tri_offsets, const int8_t* tri_table,
                                  const uint8_t* n_tri_table, const int8_t* edge_owner, const int32_t* vert_index,
                                  int32_t* tris, o2345_stream_t stream) {
  O2345_CHECK_ARG(cases && cells && count && tri_offsets && tri_table && n_tri_table && edge_owner && vert_index && tris, "null pointer");
  if (max_cells == 0) return O2345_OK;
  mc_triangles_kernel<<<cdiv(max_cells, 128), 128, 0, (cudaStream_t)stream>>>(cases, R, cells, count, tri_offsets, tri_table,
                                                                              n_tri_table, edge_owner, vert_index, tris);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
