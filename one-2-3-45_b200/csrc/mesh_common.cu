// The input check, the vertex -> face adjacency, the union-find passes and the stable radix sort of the mesh calls
// (simplify.cu, texture.cu, clean.cu, ao.cu); see mesh_common.cuh.
#include "mesh_common.cuh"

namespace o2345 {
namespace {

__global__ void check_kernel(const float* __restrict__ V, int64_t nv, const int32_t* __restrict__ F, int64_t nf,
                             uint8_t* __restrict__ flags, int32_t* __restrict__ err) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nf) {
    int c[3] = {F[3 * i], F[3 * i + 1], F[3 * i + 2]};
    bool in = face_ok(c, nv);
    if (!in) atomicOr(err, 1);
    if (flags) flags[i] = in && c[0] != c[1] && c[1] != c[2] && c[0] != c[2];
  }
  if (i < nv) {
    for (int k = 0; k < 3; ++k)
      if (!isfinite(V[3 * i + k])) atomicOr(err, 2);
  }
}

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

// one thread per vertex: insertion sort of its faces by index
__global__ void sort_kernel(const int32_t* __restrict__ off, int64_t nv, int32_t* __restrict__ adj) {
  int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nv) return;
  int32_t* L = adj + off[u];
  int d = off[u + 1] - off[u];
  for (int i = 1; i < d; ++i) {
    int f = L[i], j = i - 1;
    while (j >= 0 && L[j] > f) L[j + 1] = L[j], --j;
    L[j + 1] = f;
  }
}

__global__ void iota_kernel(int32_t* __restrict__ p, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = (int32_t)i;
}

__global__ void compress_kernel(int32_t* parent, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) parent[i] = find_root(parent, (int)i);
}

// One pass of the stable split: ones[i] := bit b of the key of order[i]
__global__ void bit_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ key, int64_t n, int b,
                           int32_t* __restrict__ ones) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ones[i] = (key[order[i]] >> b) & 1;
}

// ... and after the scan of ones (total *n_ones), the zeros keep their order at the front, the ones at the back
__global__ void split_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ key, int64_t n, int b,
                             const int32_t* __restrict__ ones_before, const int32_t* __restrict__ n_ones,
                             int32_t* __restrict__ next) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t f = order[i], o = ones_before[i];
  next[(key[f] >> b) & 1 ? n - *n_ones + o : i - o] = f;
}

}  // namespace

int iota_i32(int32_t* p, int64_t n, cudaStream_t stream) {
  iota_kernel<<<cdiv(n, 256), 256, 0, stream>>>(p, n);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

int union_find_settle(int32_t* parent, int64_t n, int32_t* changed, bool& again, cudaStream_t stream) {
  compress_kernel<<<cdiv(n, 256), 256, 0, stream>>>(parent, n);
  O2345_LAUNCH_CHECK();
  int32_t h = 0;
  O2345_CUDA(cudaMemcpyAsync(&h, changed, 4, cudaMemcpyDeviceToHost, stream));
  O2345_CUDA(cudaStreamSynchronize(stream));
  O2345_CUDA(cudaMemsetAsync(changed, 0, 4, stream));
  again = h != 0;
  return O2345_OK;
}

int radix_sort_i32(int32_t*& order, int32_t*& next, const int32_t* key, int64_t n, int bits, int32_t* ones, int32_t* sums,
                   int32_t* n_ones, cudaStream_t stream) {
  O2345_TRY(iota_i32(order, n, stream));
  for (int b = 0; b < bits; ++b) {
    bit_kernel<<<cdiv(n, 256), 256, 0, stream>>>(order, key, n, b, ones);
    O2345_LAUNCH_CHECK();
    O2345_TRY(scan_i32(ones, n, sums, n_ones, stream));
    split_kernel<<<cdiv(n, 256), 256, 0, stream>>>(order, key, n, b, ones, n_ones, next);
    O2345_LAUNCH_CHECK();
    int32_t* t = order;
    order = next, next = t;
  }
  return O2345_OK;
}

int vertex_faces(const int32_t* faces, int64_t nf, int64_t nv, int32_t* off, int32_t* sums, int32_t* cursor, int32_t* adj,
                 cudaStream_t stream) {
  const int64_t n3 = 3 * nf;
  O2345_CUDA(cudaMemsetAsync(off, 0, 4 * (nv + 1), stream));
  O2345_CUDA(cudaMemsetAsync(cursor, 0, 4 * nv, stream));
  if (n3 > 0) degree_kernel<<<cdiv(n3, 256), 256, 0, stream>>>(faces, n3, off);
  O2345_LAUNCH_CHECK();
  O2345_TRY(scan_i32(off, nv + 1, sums, nullptr, stream));
  if (n3 > 0) fill_kernel<<<cdiv(n3, 256), 256, 0, stream>>>(faces, n3, off, cursor, adj);
  sort_kernel<<<cdiv(nv, 128), 128, 0, stream>>>(off, nv, adj);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

int mesh_check(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, uint8_t* flags, int32_t* err,
               cudaStream_t stream) {
  check_kernel<<<cdiv(nv > nf ? nv : nf, 256), 256, 0, stream>>>(verts, nv, faces, nf, flags, err);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

int mesh_check_status(int32_t err, const char* func) {
  if (err & 1) {
    set_error("%s: a face index is outside [0, nv)", func);
    return O2345_EINVAL;
  }
  if (err & 2) {
    set_error("%s: a vertex coordinate is not finite", func);
    return O2345_EINVAL;
  }
  return O2345_OK;
}

}  // namespace o2345
