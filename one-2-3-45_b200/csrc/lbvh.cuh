// The LBVH over the faces of a mesh (ao.cu's ray casts, remesh.cu's closest points), built on the device in lbvh.cu:
//
//   box    the box of the vertices by integer atomics on order-preserving bit patterns (exact, any order), then its fp64
//          diagonal D and the face-box pad fp32(D) pad_scale in one thread;
//   keys   30-bit Morton codes of the face-box centres in that box, sorted stably from face order (radix_sort_i32,
//          mesh_common.cuh), so equal codes stay in face order and (code, position) is a unique key;
//   tree   the radix tree of Karras (2012) over those keys: inner nodes 0 .. nf - 2, leaf i at node nf - 1 + i is face
//          order[i]; leaf boxes are the face boxes grown by the pad, and each inner node's box is the exact min / max of its
//          children's, filled bottom-up by the second thread to reach it (one atomic counter per node), so the boxes do not
//          depend on which thread comes second.
//
// A node's box therefore contains the padded box of every face below it.
#pragma once
#include "mesh_common.cuh"

namespace o2345 {

constexpr int kLbvhStack = 64;   // keys have 62 bits below the 2 leading zeros: the tree is at most 62 inner levels deep

// The device buffers of an LBVH over nf >= 1 faces, carved from a scratch buffer in this order.
struct Lbvh {
  int32_t* ctr;    // 8: [0] free for the caller, [1] the sort's count of ones, [2..4] / [5..7] the box as ordered ints
  float* geom;     // 8: box lo xyz, hi xyz, pad
  int32_t *key, *order, *next, *ones, *sums, *mkey;
  int2* child;     // [nf - 1] children of the inner nodes
  int32_t* parent; // [2 nf - 1] parent of every node
  int32_t* visit;  // [nf - 1] refit counters
  float4* box;     // [2 nf - 1][2] lo, hi per node
  float* tri;      // [nf][9] the corners of leaf i's face, in face order

  Lbvh(Carver& c, int64_t nf)
      : ctr(c.take<int32_t>(8)), geom(c.take<float>(8)), key(c.take<int32_t>(nf)), order(c.take<int32_t>(nf)),
        next(c.take<int32_t>(nf)), ones(c.take<int32_t>(nf)), sums(c.take<int32_t>(scan_blocks(nf))),
        mkey(c.take<int32_t>(nf)), child(c.take<int2>(nf)), parent(c.take<int32_t>(2 * nf)), visit(c.take<int32_t>(nf)),
        box(c.take<float4>(4 * nf)), tri(c.take<float>(9 * nf)) {}

  // Builds the tree of faces [nf,3] (indices checked by the caller) of verts [nv,3], face boxes grown by fp32(D) pad_scale;
  // ctr[0] is left untouched.  On return `order` points at the leaf order (leaf i is face order[i]).
  int build(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float pad_scale, cudaStream_t stream);
};

}  // namespace o2345
