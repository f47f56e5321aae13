// The input check of the mesh calls (simplify.cu, texture.cu); see mesh_common.cuh.
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

}  // namespace

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
