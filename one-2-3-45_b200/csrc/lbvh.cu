// The LBVH build of ao.cu and remesh.cu; see lbvh.cuh.
#include "lbvh.cuh"

namespace o2345 {
namespace {

enum { kOnes = 1, kLo = 2, kHi = 5 };

// IEEE bits -> int32 that orders like the floats (atomicMin / atomicMax on them are exact min / max)
__device__ __forceinline__ int f2o(float f) {
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float o2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__device__ __forceinline__ float comp(float3 v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : v.z); }

__global__ void init_box_kernel(int32_t* __restrict__ ctr) {
  if (threadIdx.x < 3) ctr[kLo + threadIdx.x] = INT32_MAX, ctr[kHi + threadIdx.x] = INT32_MIN;
}

// the box of the nv vertices: per-thread min / max, warp reductions, one atomic per warp and bound
__global__ void box_kernel(const float* __restrict__ V, int64_t nv, int32_t* __restrict__ ctr) {
  int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int o = f2o(V[3 * i + c]);
      lo[c] = min(lo[c], o), hi[c] = max(hi[c], o);
    }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    lo[c] = __reduce_min_sync(0xffffffffu, lo[c]);
    hi[c] = __reduce_max_sync(0xffffffffu, hi[c]);
  }
  if ((threadIdx.x & 31) == 0)
    for (int c = 0; c < 3; ++c) atomicMin(ctr + kLo + c, lo[c]), atomicMax(ctr + kHi + c, hi[c]);
}

// geom := (box lo xyz, box hi xyz, pad): pad = fp32(D) pad_scale, D = sqrt((dx dx + dy dy) + dz dz) in fp64
__global__ void geom_kernel(const int32_t* __restrict__ ctr, float pad_scale, float* __restrict__ geom) {
  double d2 = 0.0;
  for (int c = 0; c < 3; ++c) {
    const float lo = o2f(ctr[kLo + c]), hi = o2f(ctr[kHi + c]);
    geom[c] = lo, geom[3 + c] = hi;
    const double e = __dsub_rn((double)hi, (double)lo);
    d2 = c == 0 ? __dmul_rn(e, e) : __dadd_rn(d2, __dmul_rn(e, e));
  }
  geom[6] = __fmul_rn(__double2float_rn(__dsqrt_rn(d2)), pad_scale);
}

__device__ __forceinline__ uint32_t spread10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

__device__ __forceinline__ void face_box(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t f, float3 c[3],
                                         float3& lo, float3& hi) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int64_t v = F[3 * f + j];
    c[j] = make_float3(V[3 * v], V[3 * v + 1], V[3 * v + 2]);
  }
  lo = make_float3(fminf(fminf(c[0].x, c[1].x), c[2].x), fminf(fminf(c[0].y, c[1].y), c[2].y), fminf(fminf(c[0].z, c[1].z), c[2].z));
  hi = make_float3(fmaxf(fmaxf(c[0].x, c[1].x), c[2].x), fmaxf(fmaxf(c[0].y, c[1].y), c[2].y), fmaxf(fmaxf(c[0].z, c[1].z), c[2].z));
}

// key[f] := the 30-bit Morton code of face f's box centre in the vertex box (10 bits per axis)
__global__ void morton_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                              const float* __restrict__ geom, int32_t* __restrict__ key) {
  int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  float3 c[3], lo, hi;
  face_box(V, F, f, c, lo, hi);
  uint32_t q[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float ext = geom[3 + a] - geom[a];
    const float x = (0.5f * (comp(lo, a) + comp(hi, a)) - geom[a]) * (ext > 0.f ? 1024.f / ext : 0.f);
    q[a] = (uint32_t)fminf(fmaxf(x, 0.f), 1023.f);
  }
  key[f] = (int32_t)((spread10(q[0]) << 2) | (spread10(q[1]) << 1) | spread10(q[2]));
}

// Leaf i (node nf - 1 + i) is face order[i]: its Morton code, its padded box and its corners in face order.
__global__ void leaf_kernel(const float* __restrict__ V, const int32_t* __restrict__ F, int64_t nf,
                            const int32_t* __restrict__ order, const int32_t* __restrict__ key, const float* __restrict__ geom,
                            int32_t* __restrict__ mkey, float4* __restrict__ box, float* __restrict__ tri) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf) return;
  const int64_t f = order[i];
  mkey[i] = key[f];
  float3 c[3], lo, hi;
  face_box(V, F, f, c, lo, hi);
  const float pad = geom[6];
  const int64_t node = nf - 1 + i;
  box[2 * node] = make_float4(__fsub_rn(lo.x, pad), __fsub_rn(lo.y, pad), __fsub_rn(lo.z, pad), 0.f);
  box[2 * node + 1] = make_float4(__fadd_rn(hi.x, pad), __fadd_rn(hi.y, pad), __fadd_rn(hi.z, pad), 0.f);
#pragma unroll
  for (int j = 0; j < 3; ++j) tri[9 * i + 3 * j] = c[j].x, tri[9 * i + 3 * j + 1] = c[j].y, tri[9 * i + 3 * j + 2] = c[j].z;
}

// the common prefix length of the keys (code, position) of leaves i and j; -1 outside [0, n)
__device__ __forceinline__ int delta(const int32_t* __restrict__ mkey, int64_t n, int64_t i, int64_t j) {
  if (j < 0 || j >= n) return -1;
  const uint64_t a = ((uint64_t)(uint32_t)mkey[i] << 32) | (uint64_t)i, b = ((uint64_t)(uint32_t)mkey[j] << 32) | (uint64_t)j;
  return __clzll((long long)(a ^ b));
}

// Inner node i of the radix tree (Karras 2012): its range, split and children (node ids: inner 0 .. nf - 2, leaf i at
// nf - 1 + i).
__global__ void tree_kernel(const int32_t* __restrict__ mkey, int64_t nf, int2* __restrict__ child, int32_t* __restrict__ parent) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf - 1) return;
  const int d = delta(mkey, nf, i, i + 1) > delta(mkey, nf, i, i - 1) ? 1 : -1;
  const int dmin = delta(mkey, nf, i, i - d);
  int64_t lmax = 2;
  while (delta(mkey, nf, i, i + lmax * d) > dmin) lmax *= 2;
  int64_t l = 0;
  for (int64_t t = lmax / 2; t >= 1; t /= 2)
    if (delta(mkey, nf, i, i + (l + t) * d) > dmin) l += t;
  const int64_t j = i + l * d;
  const int dnode = delta(mkey, nf, i, j);
  int64_t s = 0, t = l;
  do {
    t = (t + 1) >> 1;
    if (delta(mkey, nf, i, i + (s + t) * d) > dnode) s += t;
  } while (t > 1);
  const int64_t g = i + s * d + min(d, 0);
  const int left = (int)(min(i, j) == g ? nf - 1 + g : g), right = (int)(max(i, j) == g + 1 ? nf - 1 + g + 1 : g + 1);
  child[i] = make_int2(left, right);
  parent[left] = (int)i, parent[right] = (int)i;
}

// Bottom-up boxes: from every leaf, the second thread to arrive at a node writes the min / max of its children's boxes.
__global__ void refit_kernel(int64_t nf, const int2* __restrict__ child, const int32_t* __restrict__ parent,
                             int32_t* __restrict__ visit, float4* box) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf) return;
  int node = parent[nf - 1 + i];
  while (true) {
    __threadfence();
    if (atomicAdd(visit + node, 1) == 0) return;
    const int2 c = child[node];
    const float4 al = __ldcg(box + 2 * c.x), ah = __ldcg(box + 2 * c.x + 1);
    const float4 bl = __ldcg(box + 2 * c.y), bh = __ldcg(box + 2 * c.y + 1);
    box[2 * node] = make_float4(fminf(al.x, bl.x), fminf(al.y, bl.y), fminf(al.z, bl.z), 0.f);
    box[2 * node + 1] = make_float4(fmaxf(ah.x, bh.x), fmaxf(ah.y, bh.y), fmaxf(ah.z, bh.z), 0.f);
    if (node == 0) return;
    node = parent[node];
  }
}

}  // namespace

int Lbvh::build(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float pad_scale, cudaStream_t s) {
  init_box_kernel<<<1, 32, 0, s>>>(ctr);
  box_kernel<<<min(cdiv(nv, 256), 4 * sm_count()), 256, 0, s>>>(verts, nv, ctr);
  geom_kernel<<<1, 1, 0, s>>>(ctr, pad_scale, geom);
  morton_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, faces, nf, geom, key);
  O2345_LAUNCH_CHECK();
  O2345_TRY(radix_sort_i32(order, next, key, nf, 30, ones, sums, ctr + kOnes, s));
  leaf_kernel<<<cdiv(nf, 256), 256, 0, s>>>(verts, faces, nf, order, key, geom, mkey, box, tri);
  O2345_LAUNCH_CHECK();
  if (nf > 1) {
    O2345_CUDA(cudaMemsetAsync(visit, 0, 4 * (nf - 1), s));
    tree_kernel<<<cdiv(nf - 1, 256), 256, 0, s>>>(mkey, nf, child, parent);
    refit_kernel<<<cdiv(nf, 256), 256, 0, s>>>(nf, child, parent, visit, box);
    O2345_LAUNCH_CHECK();
  }
  return O2345_OK;
}

}  // namespace o2345
