// Shared helpers for libo2345_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/o2345.h"

namespace o2345 {

void set_error(const char* fmt, ...);

#define O2345_CHECK_ARG(cond, msg)                          \
  do {                                                      \
    if (!(cond)) {                                          \
      ::o2345::set_error("%s: %s", __func__, msg);          \
      return O2345_EINVAL;                                  \
    }                                                       \
  } while (0)

#define O2345_CUDA(call)                                                            \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) {                                                       \
      ::o2345::set_error("%s: %s -> %s", __func__, #call, cudaGetErrorString(e__)); \
      return O2345_ECUDA;                                                           \
    }                                                                               \
  } while (0)

#define O2345_LAUNCH_CHECK() O2345_CUDA(cudaGetLastError())

// returns the status of an o2345 call that failed (its error text is already set)
#define O2345_TRY(call)                \
  do {                                 \
    int rc__ = (call);                 \
    if (rc__ != O2345_OK) return rc__; \
  } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// Hands out 16-byte-aligned blocks of one scratch buffer in the order of the take() calls.  A Carver without a base
// only measures: after the same calls, `bytes` is the size the buffer needs.  Every offset is a multiple of 16, so each
// block is as aligned as the base (up to 16 bytes).
struct Carver {
  char* base = nullptr;
  int64_t bytes = 0;
  template <typename T>
  T* take(int64_t count) {
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (count * (int64_t)sizeof(T) + 15) & ~(int64_t)15;
    return p;
  }
};

// ---- scan.cu
constexpr int kScanBlock = 1024;   // elements per block of an int32 prefix sum
inline int64_t scan_blocks(int64_t n) { return (n + kScanBlock - 1) / kScanBlock; }
// vals[0, n) := its exclusive prefix sum in place (three launches); block_sums: scan_blocks(n) int32; *total := the sum
// (when total is not null).
int scan_i32(int32_t* vals, int64_t n, int32_t* block_sums, int32_t* total, cudaStream_t stream);

constexpr int kSumChunk = 1024;    // elements per sequential chunk of cumsum_f64_chunked
inline int64_t sum_chunks(int64_t n) { return (n + kSumChunk - 1) / kSumChunk; }
// x[0, n) := its inclusive prefix sum in fp64, in a fixed order that does not depend on the launch: sequential inside
// chunks of kSumChunk elements, then over the chunk totals (three launches).  chunk_tot: sum_chunks(n) + 1 doubles; on
// return chunk_tot[k] is the sum of the chunks before k and chunk_tot[sum_chunks(n)] the total.
int cumsum_f64_chunked(double* x, int64_t n, double* chunk_tot, cudaStream_t stream);

// "Once per device" guard for per-function attributes (cudaFuncSetAttribute applies to the CURRENT device only, and a
// process may drive several devices, e.g. run.py --gpu_idx): need() is true the first time it is called on a device.
struct PerDeviceOnce {
  unsigned long long seen = 0;
  bool need() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d > 63) return true;
    if ((seen >> d) & 1ull) return false;
    seen |= 1ull << d;
    return true;
  }
};

// Number of SMs of the current device (cached).  Grids of persistent kernels are sized
// as a multiple of this (132 on H100 SXM).
int sm_count();

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Point gi of a point source (explicit list, lattice or ray samples).
__device__ __forceinline__ void load_point(const o2345_points& src, int64_t gi, float& x, float& y, float& z) {
  if (src.mode == O2345_PTS_EXPLICIT) {
    x = __ldg(src.pts + 3 * gi), y = __ldg(src.pts + 3 * gi + 1), z = __ldg(src.pts + 3 * gi + 2);
  } else if (src.mode == O2345_PTS_LATTICE) {
    int R = src.R;
    int64_t ix = gi / ((int64_t)R * R);
    int iy = (int)((gi / R) % R), iz = (int)(gi % R);
    x = __ldg(src.lin + ix), y = __ldg(src.lin + iy), z = __ldg(src.lin + iz);
  } else {
    int64_t r = gi / src.S;
    int s = (int)(gi - r * src.S);
    float t = __ldg(src.z + r * src.z_stride + s);
    // o + d * t with separately rounded multiply and add (torch evaluates it that way)
    x = __fadd_rn(__ldg(src.rays_o + 3 * r), __fmul_rn(__ldg(src.rays_d + 3 * r), t));
    y = __fadd_rn(__ldg(src.rays_o + 3 * r + 1), __fmul_rn(__ldg(src.rays_d + 3 * r + 1), t));
    z = __fadd_rn(__ldg(src.rays_o + 3 * r + 2), __fmul_rn(__ldg(src.rays_d + 3 * r + 2), t));
  }
}

// Programmatic dependent launch (PDL).  The ~660 kernels of a UNet pass are launched with programmatic stream
// serialization: kernel N+1 may be scheduled while kernel N drains, runs its prologue (barrier init, descriptor prefetch,
// index math) and then blocks in pdl_wait() until kernel N has completed and flushed its writes.
// Every kernel launched this way calls pdl_wait() before its first access to memory another kernel may have written (or
// may still read), so the chain stays transitively ordered; kernels launched normally are unaffected (wait is a no-op).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();  // api.cu: environment O2345_PDL (default on; "0" switches the launch attribute off)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Same, for kernels that run as thread-block clusters of (cluster_x, 1, cluster_z) CTAs ((1, 1, 1): no cluster attribute).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x,
                                      int cluster_z, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  int n = 1;
  if (cluster_x > 1 || cluster_z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x, attr[n].val.clusterDim.y = 1, attr[n].val.clusterDim.z = cluster_z;
    ++n;
  }
  cfg.attrs = attr, cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace o2345
