// Prefix sums of the library: the int32 exclusive scan (marching-cubes triangle offsets, mesh adjacency, the
// nearest-neighbour cell offsets), the ordered stream compaction built on it (o2345_compact), and the fixed-order fp64
// cumulative sum (surface-sample CDF, texture-atlas area sum).
//
//   int32 scan   kScanBlock elements per block: a block scan (warp shuffles, then one warp over the warp totals) writes
//                each block's sum, one block scans the block sums tile by tile, and the block offsets are added back;
//   compaction   the same three phases with the flag count per block, the shared block-sum scan, and a scatter of the
//                kept indices to their ranks (ascending order: rows[k] = the k-th kept index);
//   fp64 sum     one thread per chunk sums its chunk sequentially, one thread the chunk totals, then the offsets are
//                added, so the rounding does not depend on the launch configuration.
#include "common.cuh"

namespace o2345 {
namespace {

// Block-wide exclusive scan of one int per thread (blockDim.x == kScanBlock); total := the block's sum.
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
  __syncthreads();   // warp_tot may be reused by the next call
  return excl;
}

__global__ void __launch_bounds__(kScanBlock) scan_block_kernel(int32_t* __restrict__ vals, int64_t n,
                                                                int32_t* __restrict__ block_sums) {
  int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  int v = i < n ? vals[i] : 0, total;
  int excl = block_exclusive_scan(v, total);
  if (i < n) vals[i] = excl;
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// one block: exclusive scan of the nb block sums in place, tile by tile; *total (if not null) := their sum
__global__ void __launch_bounds__(kScanBlock) scan_tops_kernel(int32_t* __restrict__ block_sums, int nb,
                                                               int32_t* __restrict__ total) {
  int carry = 0;
  for (int base = 0; base < nb; base += kScanBlock) {
    int i = base + threadIdx.x, v = i < nb ? block_sums[i] : 0, tile;
    int excl = block_exclusive_scan(v, tile);
    if (i < nb) block_sums[i] = carry + excl;
    carry += tile;
  }
  if (total && threadIdx.x == 0) *total = carry;
}

__global__ void scan_add_kernel(int32_t* __restrict__ vals, int64_t n, const int32_t* __restrict__ block_sums) {
  int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  if (i < n) vals[i] += block_sums[blockIdx.x];
}

__global__ void compact_count_kernel(const uint8_t* __restrict__ flags, int64_t n, int32_t* __restrict__ block_sums) {
  int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  int f = (i < n && flags[i]) ? 1 : 0;
  int c = __syncthreads_count(f);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = c;
}

__global__ void __launch_bounds__(kScanBlock) compact_scatter_kernel(const uint8_t* __restrict__ flags, int64_t n,
                                                                     const int32_t* __restrict__ block_offs,
                                                                     int32_t* __restrict__ rows, int32_t* __restrict__ index) {
  int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  int f = (i < n && flags[i]) ? 1 : 0, total;
  int pos = block_offs[blockIdx.x] + block_exclusive_scan(f, total);
  if (i < n) {
    if (f) rows[pos] = (int32_t)i;
    if (index) index[i] = f ? pos : -1;
  }
}

// one thread per chunk: in-place sequential cumulative sum of the chunk, its total -> tot[chunk]
__global__ void chunk_scan_kernel(double* __restrict__ x, int64_t n, double* __restrict__ tot, int64_t nchunks) {
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nchunks) return;
  int64_t a = k * kSumChunk, b = min(a + kSumChunk, n);
  double run = 0.0;
#pragma unroll 8
  for (int64_t t = a; t < b; ++t) run = __dadd_rn(run, x[t]), x[t] = run;
  tot[k] = run;
}

// one thread: tot[k] := sum of the totals of chunks 0 .. k-1 (sequential), tot[nchunks] := the total
__global__ void chunk_offsets_kernel(double* __restrict__ tot, int64_t nchunks) {
  double run = 0.0;
  for (int64_t k = 0; k < nchunks; ++k) {
    double v = tot[k];
    tot[k] = run;
    run = __dadd_rn(run, v);
  }
  tot[nchunks] = run;
}

__global__ void chunk_add_kernel(double* __restrict__ x, int64_t n, const double* __restrict__ off) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) x[t] = __dadd_rn(x[t], off[t / kSumChunk]);
}

}  // namespace

int scan_i32(int32_t* vals, int64_t n, int32_t* block_sums, int32_t* total, cudaStream_t stream) {
  int nb = (int)scan_blocks(n);
  scan_block_kernel<<<nb, kScanBlock, 0, stream>>>(vals, n, block_sums);
  scan_tops_kernel<<<1, kScanBlock, 0, stream>>>(block_sums, nb, total);
  scan_add_kernel<<<nb, kScanBlock, 0, stream>>>(vals, n, block_sums);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

int cumsum_f64_chunked(double* x, int64_t n, double* chunk_tot, cudaStream_t stream) {
  int64_t nchunks = sum_chunks(n);
  chunk_scan_kernel<<<cdiv(nchunks, 64), 64, 0, stream>>>(x, n, chunk_tot, nchunks);
  chunk_offsets_kernel<<<1, 1, 0, stream>>>(chunk_tot, nchunks);
  chunk_add_kernel<<<cdiv(n, 256), 256, 0, stream>>>(x, n, chunk_tot);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}

}  // namespace o2345

using namespace o2345;

extern "C" int64_t o2345_scan_scratch_ints(int64_t n) { return scan_blocks(n) + 1; }

extern "C" int64_t o2345_compact_scratch_ints(int64_t n) { return scan_blocks(n) + 1; }

extern "C" int o2345_compact(const uint8_t* flags, int64_t n, int32_t* rows, int32_t* index, int32_t* count,
                             int32_t* scratch, o2345_stream_t stream) {
  O2345_CHECK_ARG(flags && rows && count && scratch, "null pointer");
  O2345_CHECK_ARG(n > 0 && n < ((int64_t)1 << 31), "element count out of range");
  int nb = (int)scan_blocks(n);
  cudaStream_t st = (cudaStream_t)stream;
  compact_count_kernel<<<nb, kScanBlock, 0, st>>>(flags, n, scratch);
  scan_tops_kernel<<<1, kScanBlock, 0, st>>>(scratch, nb, count);
  compact_scatter_kernel<<<nb, kScanBlock, 0, st>>>(flags, n, scratch, rows, index);
  O2345_LAUNCH_CHECK();
  return O2345_OK;
}
