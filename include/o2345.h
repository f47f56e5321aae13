/*
 * libo2345_sm90.so -- C-ABI of the H100-native (sm_90a) kernels behind One-2-3-45's
 * SparseNeuS-style reconstruction hot path (SURVEY.md section 8, rows B1-B15).
 *
 * The reference has no FFI of its own for this path: its boundary is plain Python classes
 * (SparseSdfNetwork, SparseNeuSRenderer, FeatureNet, GeneralRenderingNetwork, Projector) that
 * call PyTorch/ATen, torchsparse v1.4.0, inplace_abn and PyMCubes.  Each entry point below
 * names the reference call site(s) it replaces; INTEGRATION.md shows the ctypes stub a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - all floating point data is fp32, dense and contiguous in the stated layout;
 *   - the caller allocates every buffer (outputs and scratch); nothing is allocated or
 *     freed behind the ABI and no call synchronises the device (except the five that say so:
 *     o2345_lod_children and o2345_surface_sample read a device-side check, o2345_simplify reads
 *     a count once per round, o2345_texture_atlas reads its checks once and a fit flag per trial,
 *     o2345_vertex_normals reads its checks once, o2345_chart_atlas reads its checks, a flag per component pass,
 *     two values per chart round and a fit flag per trial, o2345_clean_mesh reads its checks, a flag per
 *     component pass, the component count and its counts, o2345_ambient_occlusion and o2345_closest_points read their
 *     checks once, o2345_remesh reads its checks, its counts once per round and the output count);
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it;
 *   - return value 0 on success, negative O2345_E* otherwise; o2345_last_error() returns a
 *     thread-local description of the most recent failure.
 */
#ifndef O2345_H_
#define O2345_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define O2345_OK 0
#define O2345_EINVAL (-1)
#define O2345_ECUDA (-2)
#define O2345_EUNSUPPORTED (-3)
#define O2345_ENOSPC (-4) /* o2345_remesh: the caller's capacities are too small (the counts it needs are returned) */

#define O2345_ABI_VERSION 14 /* 2: o2345_epilogue, precision arguments of sdf_query / render_blend, GroupNorm as affine
                                 3: split-K inside the GEMM kernel (cluster per tile, private planes in the workspace), o2345_last_trap, o2345_debug_gemm_force
                                 4: the lod-1 refinement group (o2345_sdf_voxels, o2345_prune_*, o2345_lod_children, ...)
                                 5: render_blend precision 2 (the wgmma kernel, O2345_BLEND_TC5) is gone
                                 6: rays of many cameras in one launch: render_blend dir_mode 2, o2345_ray_midpoints_per_ray
                                 7: the GEMM epilogue's GroupNorm column statistics are gone: o2345_epilogue lost its last two fields,
                                    and the norm + patch gather entry point that read the tables went with them
                                 8: the mesh rasterizer: o2345_raster, o2345_raster_scratch_bytes, o2345_debug_raster_split
                                 9: mesh scoring: o2345_surface_sample(_scratch_bytes), o2345_nearest, o2345_nn_scratch_bytes
                                10: mesh simplification: o2345_simplify, o2345_simplify_scratch_bytes
                                11: texture baking: o2345_texture_atlas, o2345_texel_points, o2345_texture_fill,
                                    o2345_transfer_colors and their scratch-size functions
                                12: normal maps: o2345_tangent_normals, o2345_normal_quantise, o2345_vertex_normals(_scratch_bytes);
                                    o2345_raster_mesh gained normals, tangents and face_ntex (after tex_info)
                                13: multi-face charts: o2345_chart_atlas(_scratch_bytes), o2345_tangent_normals_decoded
                                14: input-view projection: o2345_project_view, o2345_face_normals; mesh cleaning:
                                    o2345_clean_mesh(_scratch_bytes); ambient occlusion: o2345_ambient_occlusion(_scratch_bytes);
                                    remeshing: o2345_closest_points(_scratch_bytes), o2345_remesh(_scratch_bytes), O2345_ENOSPC
                                    (added entry points only: the binding resolves every entry point by name, so a library
                                    without them fails to load) */

typedef void* o2345_stream_t;

int o2345_abi_version(void);
/* Copies the last error message of the calling thread into buf (NUL terminated). */
int o2345_last_error(char* buf, size_t n);
/* Fills (major, minor, sm_count) of the current device; fails if it is not sm_90. */
int o2345_device_info(int* major, int* minor, int* sms);

/* ------------------------------------------------------------------------------------------
 * B8 / B9 / B10: SDF query = quirky trilinear latent fetch + positional embedding +
 * weight-normed 39->128->128->128 MLP (+ analytic d sdf / d x).
 * Replaces SparseSdfNetwork.sdf            reconstruction/models/sparse_sdf_network.py:402-420
 *          ops.grid_sampler.grid_sample_3d reconstruction/ops/grid_sampler.py:64-216
 *          LatentSDFLayer.forward          reconstruction/models/sparse_sdf_network.py:111-136
 *          Embedding.forward               reconstruction/models/embedder.py:81-101
 *          SparseSdfNetwork.gradient       reconstruction/models/sparse_sdf_network.py:476-499
 *          extract_fields (lattice mode)   reconstruction/models/sparse_neus_renderer.py:882-905
 * ------------------------------------------------------------------------------------------ */

/* Number of floats of the packed MLP weights (see o2345_sdf_pack_weights). */
#define O2345_SDF_PE 39
#define O2345_SDF_HID 128
#define O2345_SDF_LAT 16
#define O2345_SDF_IN1 144
/* layout (floats): W0t[39][128] b0[128] W1t[144][128] b1[128] W2t[144][128] b2[128]
 *                  W1[128][144] W0[128][48]   (un-transposed copies for the backward pass)  */
#define O2345_SDF_PACK_FLOATS (39 * 128 + 128 + 2 * (144 * 128 + 128) + 128 * 144 + 128 * 48)

/* w0 [128,39], w1 [128,144], w2 [128,144] are the EFFECTIVE (weight-normed) matrices,
 * row-major as nn.Linear stores them; b* the biases.  Writes the packed blob. */
int o2345_sdf_pack_weights(const float* w0, const float* b0, const float* w1, const float* b1,
                           const float* w2, const float* b2, float* pack, o2345_stream_t stream);

/* Where the query points come from. */
#define O2345_PTS_EXPLICIT 0 /* pts [n,3]                                                   */
#define O2345_PTS_LATTICE 1  /* point i = (lin[i/(R*R)], lin[(i/R)%R], lin[i%R]), n = R^3     */
#define O2345_PTS_RAYS 2     /* point i = o[r] + d[r] * z[r*z_stride + s], r = i / S, s = i % S */

typedef struct o2345_points {
  int mode;
  const float* pts;    /* EXPLICIT: [n,3]                                  */
  const float* lin;    /* LATTICE: [R] coordinates                          */
  int R;               /* LATTICE                                           */
  const float* rays_o; /* RAYS: [n_rays,3]                                  */
  const float* rays_d; /* RAYS: [n_rays,3]                                  */
  const float* z;      /* RAYS: depth of sample s on ray r                  */
  int S;               /* RAYS: samples per ray                             */
  int z_stride;        /* RAYS: row stride of z in floats                   */
} o2345_points;

/* vol_cl: conditional volume, channel-last [D,D,D,16] (voxel (x,y,z) -> ((x*D+y)*D+z)*16).
 * active: optional uint8 [n]; points with active[i]==0 are not evaluated and receive
 *         sdf = inactive_sdf, feat = 0, latent = 0, grad = 0 (reference
 *         sparse_neus_renderer.py:135-139, 229-241).
 * Outputs (any may be NULL): sdf [n], feat [n,127], latent [n,16], grad [n,3].
 * If negate != 0 the sdf output is written as -sdf (extract_fields' u = -sdf). */
#define O2345_SDF_FP32 0      /* fp32 FMA GEMMs                                                                        */
#define O2345_SDF_TC_SPLIT 1  /* forward GEMMs on tensor cores, every operand split into fp16 hi + lo (three MMAs per
                                 product, fp32 accumulate): agrees with the fp32 kernel to ~1e-6                         */
int o2345_sdf_query(const o2345_points* src, int64_t n, const float* vol_cl, int D, const float* wpack,
                    const uint8_t* active, float inactive_sdf, int negate, int precision, float* sdf, float* feat,
                    float* latent, float* grad, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * B3 / B4 / B5 / B7: cost-volume build.
 * Replaces generate_grid + back_project_sparse_type (called twice) + aggregate_multiview_features
 *          + sparse_to_dense_volume:  reconstruction/ops/generate_grids.py:4-19,
 *          reconstruction/ops/back_project.py:5-86,
 *          reconstruction/models/sparse_sdf_network.py:221-284,321-346.
 * ------------------------------------------------------------------------------------------ */

/* proj [V,4,4] = K @ w2c per view (row-major), origin [3] world position of voxel (0,0,0).
 * mask_bits[D^3]: bit v set iff voxel is inside view v's frustum (|gx|<=1, |gy|<=1, z>0);
 * keep[D^3] = popcount(mask) > min_views.  V <= 32. */
int o2345_frustum_mask(const float* proj, int V, const float* origin, float voxel_size, int D, int sizeH,
                       int sizeW, int min_views, uint32_t* mask_bits, uint8_t* keep, o2345_stream_t stream);

/* Ordered stream compaction: rows[k] = i of the k-th non-zero flag (ascending i), index[i] = k or -1
 * (index may be NULL), *count = number kept.  scratch: o2345_compact_scratch_ints(n) int32. */
int64_t o2345_compact_scratch_ints(int64_t n);
int o2345_compact(const uint8_t* flags, int64_t n, int32_t* rows, int32_t* index, int32_t* count,
                  int32_t* scratch, o2345_stream_t stream);

/* feats_nhwc [V,h,w,16] compressed feature maps (channel-last).  For every kept voxel (rows,
 * *count, at most max_rows) writes cost[row] = [var(16), mean(16)] over the V views; features are
 * NOT masked, counts come from mask_bits (reference sparse_sdf_network.py:234-245). */
int o2345_costvol_gather(const float* feats_nhwc, int V, int h, int w, int sizeH, int sizeW, const float* proj,
                         const float* origin, float voxel_size, int D, const int32_t* rows, const int32_t* count,
                         int64_t max_rows, const uint32_t* mask_bits, float* cost, o2345_stream_t stream);

/* Scatter rows [n,16] into vol_cl [D^3,16] (channel-last), optionally vol_cf [16,D^3] (the
 * reference layout [1,16,X,Y,Z]) and occ [D^3] (1.0 where a row exists).  Outputs are zero-filled first. */
int o2345_dense_scatter(const float* feat, const int32_t* rows, const int32_t* count, int64_t max_rows, int D,
                        float* vol_cl, float* vol_cf, float* occ, o2345_stream_t stream);

/* Nearest occupancy lookup, ATen grid_sample(mode='nearest', align_corners=False) semantics
 * (reference sparse_neus_renderer.py:153-169).  out[i] = 1 iff occ at the nearest voxel > 0. */
int o2345_occ_nearest(const o2345_points* src, int64_t n, const float* occ, int D, uint8_t* out,
                      o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Lod-1 refinement (num_lods = 2): lod-0 SDF volume, pruning, children, cost rows with parent features.
 * Replaces SparseSdfNetwork.get_sdf_volume            reconstruction/models/sparse_sdf_network.py:441-474
 *          get_valid_sparse_coords_by_sdf             reconstruction/models/sparse_neus_renderer.py:822-879
 *          SparseSdfNetwork.upsample + lod>0 branch   reconstruction/models/sparse_sdf_network.py:198-219,336-374
 * ------------------------------------------------------------------------------------------ */

/* sdf_vol[i] = SDF MLP at voxel i of the D^3 lattice for every i with occ[i] > 0, else 1.0.  The point is
 * coord * voxel_size + origin (rounded fp32 multiply, then add) and the latent is row i of vol_cl [D^3,16] as it is
 * (no trilinear fetch).  precision: O2345_SDF_FP32 or O2345_SDF_TC_SPLIT, as in o2345_sdf_query. */
int o2345_sdf_voxels(const float* occ, const float* vol_cl, int D, const float* origin, float voxel_size,
                     const float* wpack, int precision, float* sdf_vol, o2345_stream_t stream);

/* minabs[i] = occ[i] > 0 ? min |sdf| over the 7^3 window around i (clipped at the border) : +inf, so that
 * avg_pool3d(|sdf| < t, 7, 1, 3) > 0 && occ > 0  <=>  minabs < t for every t.  counts[r] (device int32) = number of
 * voxels with minabs < ladder[r]; ladder is a HOST array of 1..16 fp32 thresholds.  scratch: float [D^3].
 * sdf, scratch and minabs must be three distinct buffers (O2345_EINVAL otherwise). */
int o2345_prune_by_sdf(const float* sdf, const float* occ, int D, const float* ladder, int n_ladder, float* scratch,
                       float* minabs, int32_t* counts, o2345_stream_t stream);
/* keep[i] = minabs[i] < threshold. */
int o2345_prune_select(const float* minabs, int64_t n, float threshold, uint8_t* keep, o2345_stream_t stream);
/* flags[rows[idx[i]]] = 0 for i < n (drops chosen survivors of a compaction). */
int o2345_clear_flags(const int32_t* rows, const int32_t* idx, int64_t n, uint8_t* flags, o2345_stream_t stream);
/* For the n lattice indices rows[i] of a D^3 lattice: coords[i] = (0, x, y, z) as floats, feats[i] = the C channels of
 * vol_cf [C, D^3] at rows[i]. */
int o2345_gather_rows(const int32_t* rows, int64_t n, int D, const float* vol_cf, int C, float* coords, float* feats,
                      o2345_stream_t stream);

/* pre_coords [n,4] float (batch, x, y, z), already in D1 lattice units: marks the 8 children (x+a, y+b, z+c),
 * a,b,c in {0,1}, keep[lin] = frustum_keep[lin] (o2345_frustum_mask at D1 with min_views = 1, i.e. > 1 views), and
 * parent[lin] = i (-1 elsewhere).  keep [D1^3] and parent [D1^3] are overwritten.  Returns O2345_EINVAL for a
 * coordinate that is not an integer with both children in [0, D1), or for duplicate parents: this call synchronises
 * the stream to read the device-side check (err_scratch: one int32 on the device). */
int o2345_lod_children(const float* pre_coords, int64_t n, int D1, const uint8_t* frustum_keep, uint8_t* keep,
                       int32_t* parent, int32_t* err_scratch, o2345_stream_t stream);

/* o2345_costvol_gather for C = 8 or 16 channels per view; cost rows are [var(C), mean(C)] or, with parent / pre_feats
 * (both or neither), [var(C), mean(C), pre_feats[parent[rows[k]]] (16)].  o2345_costvol_gather is C = 16 without parent. */
int o2345_costvol_gather_lod(const float* feats_nhwc, int C, int V, int h, int w, int sizeH, int sizeW, const float* proj,
                             const float* origin, float voxel_size, int D, const int32_t* rows, const int32_t* count,
                             int64_t max_rows, const uint32_t* mask_bits, const int32_t* parent, const float* pre_feats,
                             float* cost, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * B6: sparse 3-D convolution stack (torchsparse v1.4.0 semantics) + BatchNorm(batch stats) + ReLU.
 * Replaces spnn.Conv3d / spnn.BatchNorm / spnn.ReLU as used by SparseCostRegNet:
 *          reconstruction/tsparse/modules.py:94-124,259-304.
 * A level is described by a dense lattice index[E^3] (row id or -1), its row list rows[n] (cell
 * ids, ascending) and a device-side count.  Level l+1 has extent E/2+1.
 * ------------------------------------------------------------------------------------------ */

/* Flags the cells of the next coarser level (k=3, stride 2 down-sampling rule). cmin_scratch: int32[3]. */
int o2345_sp_coarsen(const int32_t* fine_index, int Ef, const int32_t* fine_rows, const int32_t* fine_count,
                     int64_t max_fine, int Ec, uint8_t* coarse_flags, int32_t* cmin_scratch,
                     o2345_stream_t stream);

/* mode 0: same level; 1: stride-2 down (in = fine, out = coarse); 2: transposed stride-2 (in = coarse,
 * out = fine).  kernel [27,Cin,Cout] (x-fastest offsets).  Writes raw outputs [rows,Cout] and the
 * per-channel sum / sum of squares into stats[2*Cout] (float64, zeroed by the call). */
int o2345_sp_conv(const float* in_feats, const int32_t* in_index, int Ein, const int32_t* out_rows,
                  const int32_t* out_count, int64_t max_out, int Eout, int mode, const float* kernel, int Cin,
                  int Cout, float* out_raw, double* stats, o2345_stream_t stream);

/* out = relu(batchnorm(x; batch stats, gamma, beta, eps)) (+ skip).  out may alias x. */
int o2345_sp_bn_relu(const float* x, const int32_t* count, int64_t max_rows, int C, const double* stats,
                     const float* gamma, const float* beta, float eps, const float* skip, float* out,
                     o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * B10: marching cubes on the dense u = -sdf grid.
 * Replaces mcubes.marching_cubes(u, 0): reconstruction/models/sparse_neus_renderer.py:932.
 * Case tables come from the host (o2345/mc_tables.py): tri_table int8[256,16], n_tri uint8[256],
 * edge_owner int8[12,4] = (dx,dy,dz,axis) of the lattice edge that carries cell edge e.
 * ------------------------------------------------------------------------------------------ */
int o2345_mc_classify(const float* u, int R, float iso, uint8_t* cases, uint8_t* cell_flags, uint8_t* edge_flags,
                      o2345_stream_t stream);
int o2345_mc_vertices(const float* u, int R, float iso, const int32_t* edges, const int32_t* count,
                      int64_t max_verts, double* verts, o2345_stream_t stream);
int64_t o2345_scan_scratch_ints(int64_t n);
int o2345_mc_tri_offsets(const uint8_t* cases, const int32_t* cells, const int32_t* count, int64_t max_cells,
                         const uint8_t* n_tri_table, int32_t* offsets, int32_t* total, int32_t* scratch,
                         o2345_stream_t stream);
int o2345_mc_triangles(const uint8_t* cases, int R, const int32_t* cells, const int32_t* count, int64_t max_cells,
                       const int32_t* tri_offsets, const int8_t* tri_table, const uint8_t* n_tri_table,
                       const int8_t* edge_owner, const int32_t* vert_index, int32_t* tris, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * B1 / B2: FeatureNet + compress layer primitives.
 * Replaces nn.Conv2d + InPlaceABN + F.interpolate in reconstruction/models/featurenet.py:12-91,
 *          reconstruction/models/trainer_generic.py:1104-1125, sparse_sdf_network.py:171-173.
 * ------------------------------------------------------------------------------------------ */
typedef struct o2345_view4 {
  float* ptr;               /* element (n,c,h,w) lives at ptr[n*sn + (c+c0)*sc + h*sh + w*sw] */
  int64_t sn, sc, sh, sw;
  int c0;
} o2345_view4;

/* in [N,Cin,H,W] NCHW, weight [Cout,Cin,K,K], bias NULL or [Cout]; out NCHW raw.  If stats != NULL the
 * per-channel sum / sum of squares of the output are accumulated into stats[2*Cout] (zeroed first). */
int o2345_conv2d(const float* in, int N, int Cin, int H, int W, const float* weight, const float* bias, int Cout,
                 int K, int stride, int pad, float* out, double* stats, o2345_stream_t stream);
/* InPlaceABN forward with batch statistics: (x-mean)/sqrt(var+eps)*(|gamma|+eps)+beta, leaky-ReLU(slope). */
int o2345_abn_apply(const float* x, int N, int C, int H, int W, const double* stats, const float* gamma,
                    const float* beta, float eps, float slope, const o2345_view4* out, o2345_stream_t stream);
/* Bilinear up-sampling by an integer factor, align_corners=True, optional add [N,C,H*f,W*f]. */
int o2345_upsample_bilinear(const float* x, int N, int C, int H, int W, int factor, const float* add,
                            const o2345_view4* out, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * B11 - B14: volume rendering.
 * Replaces SparseNeuSRenderer.up_sample / cat_z_vals / render_core / render
 *              reconstruction/models/sparse_neus_renderer.py:73-151,171-455,457-635
 *          sample_pdf, sample_ptsFeatures_from_feature{Volume,Maps}
 *              reconstruction/models/render_utils.py:8-120
 *          Projector.compute / compute_view_independent / compute_angle*
 *              reconstruction/models/projector.py:15-62,96-425
 *          GeneralRenderingNetwork.forward
 *              reconstruction/models/rendering_network.py:75-129
 * ------------------------------------------------------------------------------------------ */

/* One importance round: new_z [R,n_new] drawn by deterministic inverse-CDF sampling (u [n_new] =
 * linspace(0.5/n, 1-0.5/n, n)) from the NeuS section weights of the current samples z/sdf [R,S]. */
int o2345_ray_upsample(const float* rays_o, const float* rays_d, int64_t R, const float* z, const float* sdf,
                       int S, float inv_s, const float* occ, int D, const float* u, int n_new, float* new_z,
                       o2345_stream_t stream);
/* Merge the sorted lists (z,sdf) [R,S] and (new_z,new_sdf) [R,n_new] into out_* [R,S+n_new]. */
int o2345_ray_merge(const float* z, const float* sdf, int S, const float* new_z, const float* new_sdf, int n_new,
                    int64_t R, float* out_z, float* out_sdf, o2345_stream_t stream);
/* mid_z = z + dists/2, dists = forward differences (last = sample_dist), active = nearest occupancy. */
int o2345_ray_midpoints(const float* rays_o, const float* rays_d, int64_t R, const float* z, int S,
                        float sample_dist, const float* occ, int D, float* mid_z, float* dists, uint8_t* active,
                        o2345_stream_t stream);
/* o2345_ray_midpoints with a last section of its own per ray: sample_dist [R] (device), so that one launch can hold
 * rays of cameras with different near / far.  Same result per ray as o2345_ray_midpoints with that ray's value. */
int o2345_ray_midpoints_per_ray(const float* rays_o, const float* rays_d, int64_t R, const float* z, int S,
                                const float* sample_dist, const float* occ, int D, float* mid_z, float* dists,
                                uint8_t* active, o2345_stream_t stream);

#define O2345_MAP_CH 60 /* channel-last source maps: rgb(3) + pyramid features(56) + 1 pad */
#define O2345_RNET_PACK_FLOATS 19664

typedef struct o2345_views {
  int V, H, W;          /* source views and map size                                        */
  const float* maps;    /* [V,H,W,60] channel-last: [0..2] colour, [3..58] features, [59] 0  */
  const float* proj;    /* [V,3,4] = intrinsics @ w2c[:3,:4]                                 */
  const float* centers; /* [V,3] camera centres (c2w translation)                           */
  float sizeW, sizeH;   /* img_wh used to normalise pixel coordinates                       */
} o2345_views;

/* Per sample point: geometry feature, per-view colour+feature fetch, ray-difference, view-blending
 * MLP -> rgb [n,3]; nvalid [n] = number of views whose mask is set (may be NULL).  dir_mode 0: target
 * direction = normalised (query_center - p) (Projector.compute); 1: dirs [n,3] given
 * (compute_view_independent, surface normals); 2: normalised (rays_o[ray] - p), the origin of the sample's own ray
 * (O2345_PTS_RAYS only; the same bits as mode 0 with query_center = that origin: rays of many cameras in one
 * launch; query_center and dirs are ignored).  rnet_pack: O2345_RNET_PACK_FLOATS floats, every
 * matrix stored [in][out] in the order documented in csrc/blend_common.cuh. */
#define O2345_BLEND_FP32 0     /* fp32 FMA mat-vecs in the reference's operation order (tight oracle parity)            */
#define O2345_BLEND_TC_FP16 1  /* per-(sample, view) MLPs as mma.sync products: fp16 operands, fp32 accumulate / statistics */
int o2345_render_blend(const o2345_points* src, int64_t n, const uint8_t* active, const float* vol_cl,
                       const float* occ, int D, const o2345_views* views, int dir_mode, const float* query_center,
                       const float* dirs, const float* rnet_pack, int precision, float* rgb, int32_t* nvalid,
                       o2345_stream_t stream);

/* NeuS alpha from (sdf, grad), transmittance, colour/depth compositing.  Outputs: color [R,3], depth [R],
 * optional weights [R,S], cdf [R,S], alpha [R,S], weights_sum [R], color_mask [R] (uint8). */
int o2345_ray_composite(const float* rays_d, int64_t R, int S, const float* mid_z, const float* dists,
                        const float* sdf, const float* grad, const float* color, const uint8_t* active,
                        const int32_t* nvalid, float inv_s, float alpha_inter_ratio, int has_background,
                        float background, float* color_out, float* depth_out, float* weights_out, float* cdf_out,
                        float* alpha_out, float* weights_sum_out, uint8_t* color_mask_out, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Path A (rows A2-A4, A6): fp16 tensor-core GEMM, wgmma.mma_async + register accumulators + TMA operands.
 * Replaces the cuBLAS / cuDNN calls behind nn.Linear, 1x1 and (im2col'd) 3x3 nn.Conv2d and the
 * attention einsums of the Zero123 UNet and VAE:
 *          ldm/modules/diffusionmodules/openaimodel.py:745-777, ldm/modules/attention.py:170-193,
 *          ldm/modules/diffusionmodules/model.py:535-568.
 * C[b] = act(alpha * A[b] . B[b]^T + bias + rowbias) + residual[b];  A [M,K] (row stride lda), B [N,K] (row
 * stride ldb), fp16, K contiguous; C and residual [M,N] (row stride ldc), C fp16 or fp32.  nh = 0: plain GEMM;
 * nh > 0: nh * nb independent products, operand z = b * nh + h lives at ptr + h * stride_*_h + b * stride_*_b
 * (e.g. heads inside a [B, N, H*d] tensor).  lda, ldb and the A/B batch strides must be multiples of 8 elements
 * (TMA: 16-byte strides).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const float* bias;     /* [N] fp32 or NULL */
  const void* residual;  /* fp16 [M, ldc] or NULL, added after the activation (ResBlock / attention skip) */
  const void* rowbias;   /* fp16 or NULL: element [(row / rows_per_group) * rowbias_ld + col] is added before the
                            activation (the ResBlock's per-image emb_layers output, openaimodel.py:266-273) */
  int64_t rowbias_ld;
  int rows_per_group;
  int act;               /* 0 none, 1 SiLU, 2 GELU(erf), 4 QuickGELU x*sigmoid(1.702x) (CLIP), 3 GEGLU (attention.py:37-44): the N columns come in chunks of
                            32 = 16 values followed by their 16 gates, C gets N/2 columns value * gelu(gate) */
  float alpha;           /* scale on the accumulator */
  int out_f32;           /* C is fp32 instead of fp16 */
} o2345_epilogue;

int o2345_gemm_f16(const void* A, const void* B, void* C, int M, int N, int K, int64_t lda, int64_t ldb,
                   int64_t ldc, int nh, int nb, int64_t stride_a_h, int64_t stride_a_b, int64_t stride_b_h,
                   int64_t stride_b_b, int64_t stride_c_h, int64_t stride_c_b, const o2345_epilogue* ep /* NULL: plain */,
                   float* splitk_ws, int64_t ws_floats, o2345_stream_t stream);
/* splitk_ws (optional, may be NULL): fp32 scratch of ws_floats elements, no initialisation needed.  When the output tiles
 * alone cannot fill the GPU the K range is split over up to min(8, ws_floats / (M*N)) CTAs per tile that run as one
 * thread-block cluster: each stores its partial tile in its own [M, N] plane of the scratch, a cluster barrier publishes the
 * planes, and every split sums them and applies the epilogue to its share of the tile.  One workspace serves one stream at
 * a time. */

/* Every mbarrier wait inside the GEMM kernel is bounded (4 s).  If one expires the kernel records which barrier of which CTA
 * of which problem stalled in a host-mapped buffer and traps (the CUDA context then reports a launch failure at the next
 * synchronisation).  o2345_last_trap copies a description of that record into buf and returns 1, or returns 0 if no wait
 * has ever expired in this process.  Safe to call after the context has failed. */
int o2345_last_trap(char* buf, size_t n);

/* Tuning hook (tools/gemm_sweep.py; not part of the data path): force the tile configuration of the following non-batched
 * GEMM / conv calls: bn in {64, 128, 160, 256}, splits 1..8; 0 keeps the heuristic's choice of that field.  ctas is accepted and
 * ignored: every tile is one CTA. */
void o2345_debug_gemm_force(int ctas, int bn, int splits);
/* Tuning hook: the persistent launch of the kernel (at most one CTA per SM walking the tiles; launch and prologue paid once
 * per SM).  mode 0: heuristic (at least min_tiles tiles; min_tiles 0 = default),
 * 1: wherever it is available (staged fp16 epilogue, no split-K, no head batches), 2: never. */
void o2345_debug_gemm_persist(int mode, int min_tiles);
/* Tuning hook: the seven constants of the tile-configuration cost model (per-SM ingest B/clk, multi-wave bonus, fabric B/clk,
 * fixed us, epilogue us per 160 columns, split-K us, split-K us per split and 128 columns); see gemm_tc.cu predict_us. */
void o2345_debug_gemm_model(const float* seven);

/* Diagnostic hook (not part of the data path): when device_buf16 != NULL, CTA (0,0,0) of every following GEMM
 * launch stores clock64() stamps of its phases into device_buf16[0..8] (entry, prologue done, first TMA issued, last TMA
 * issued, first operands landed, last MMA issued, epilogue start, epilogue done, exit) of its last tile; in a persistent
 * launch device_buf16[9] also receives the previous tile's "last MMA issued" stamp, so [4] - [9] is the gap between two
 * tiles' MMAs.  NULL switches it off. */
void o2345_debug_gemm_trace(long long* device_buf16);

/* Implicit-GEMM 3x3 convolution, stride 1, zero padding 1 (nn.Conv2d(C, N, 3, padding=1) of the UNet ResBlocks and the
 * VAE ResnetBlocks): x channel-last [B,H,W,C] fp16, weight [N, 9*C] fp16 in (ky,kx,c) order, out [B*H*W, N] (row stride
 * ldc).  No im2col buffer exists: the nine shifted windows are fetched by 4-D TMA boxes whose out-of-bounds zero fill is
 * the padding.  W must divide 128 or be a multiple of 128; C a multiple of 8.  Epilogue as o2345_gemm_f16. */
int o2345_conv3x3_f16(const void* x, int B, int H, int W, int C, const void* weight, int N, void* out, int64_t ldc,
                      const o2345_epilogue* ep, float* splitk_ws, int64_t ws_floats, o2345_stream_t stream);

/* Nearest-neighbour 2x up-sampling followed by a 3x3 convolution (zero padding 1) -- the Upsample layers of the UNet and the
 * VAE decoder (reference ldm/modules/diffusionmodules/openaimodel.py:118-129 `Upsample.forward`, model.py:43-53) -- WITHOUT
 * materialising the up-sampled map or a patch matrix: every output pixel (2y+a, 2x+b) sees the 3x3 kernel collapse onto a
 * 2x2 window of the low-resolution input, so the layer is four 2x2 implicit convolutions, one per phase (a, b).
 * x [B, H, W, C] channel-last fp16 (the LOW-resolution map, same tiling rule as o2345_conv3x3_f16); weight4 [4][N][4*C] fp16:
 * phase 2a+b, taps in (ty, tx, c) order with the collapsed kernel rows / columns summed (a = 0: {k0, k1+k2}, a = 1: {k0+k1, k2});
 * out [B*2H*2W, ldc] fp16.  Epilogue: bias / activation only. */
int o2345_conv_up2x_f16(const void* x, int B, int H, int W, int C, const void* weight4, int N, void* out, int64_t ldc,
                        const o2345_epilogue* ep, float* splitk_ws, int64_t ws_floats, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Path A glue (rows A1, A3, A4, A6): channel-last fp16 activations [B, H*W, C]; fp32 statistics.
 * GroupNorm32 / SiLU / conv patch gather: ldm/modules/diffusionmodules/openaimodel.py:92-161,256-276,
 *   ldm/modules/diffusionmodules/util.py:214-216; LayerNorm / softmax / GEGLU: ldm/modules/attention.py:37-64,
 *   170-193,214-218; timestep embedding: util.py:151-171; CFG + DDIM update: ldm/models/diffusion/ddim.py:196-243.
 * ------------------------------------------------------------------------------------------ */
/* GroupNorm statistics folded into a per-(image, channel) affine: GroupNorm(x)[b, p, c] = x * scale[b, c] + shift[b, c]
 * (scale = rstd * gamma, shift = beta - mean * rstd * gamma; gamma / beta may be NULL).  x [B, HW, C] fp16, C a multiple
 * of 8.  scratch: o2345_groupnorm_scratch_floats(B, G) fp32 words, ALL ZERO on entry and left zeroed. */
int64_t o2345_groupnorm_scratch_floats(int B, int G);
int o2345_groupnorm_stats(const void* x, int B, int HW, int C, int G, float eps, const float* gamma, const float* beta,
                          float* scratch, float* scale, float* shift, o2345_stream_t stream);
/* GroupNorm(x) (+SiLU if act) of a channel-last activation x [B, HW, C] -> out [B, HW, C], statistics and apply in ONE kernel:
 * each image is handled by a thread-block cluster whose CTAs exchange their partial sums through distributed shared memory
 * (no scratch, no global atomics).  Same result as o2345_groupnorm_stats + o2345_norm_act_im2col(ksize 1). */
int o2345_groupnorm_apply(const void* x, int B, int HW, int C, int G, float eps, const float* gamma, const float* beta, int act,
                          void* out, o2345_stream_t stream);
/* Tuning hook (tools/gn_bench.py): CTAs per image (cluster size, a power of two <= 16) of o2345_groupnorm_apply; 0 = the launcher's rule. */
void o2345_debug_groupnorm_cluster(int cl);
/* out [B*Ho*Wo, k*k*C] (column order ky,kx,c) = patches of f(x), f = x * scale + shift (+SiLU if act) when scale != NULL.
 * upsample != 0: nearest x2 replication of x before the convolution.  Zero padding k/2 on the high side and
 * pad_lo on the low side (pad_lo < 0: k/2; pad_lo = 0 reproduces the VAE encoder's F.pad(x, (0,1,0,1))). */
int o2345_norm_act_im2col(const void* x, int B, int H, int W, int C, int ksize, int stride, int upsample, int pad_lo,
                          const float* scale, const float* shift, int act, void* out, o2345_stream_t stream);
int o2345_layernorm_rows(const void* x, int64_t M, int C, float eps, const float* gamma, const float* beta, void* y,
                         o2345_stream_t stream);
int o2345_softmax_rows(const void* s, int64_t rows, int n, void* p, o2345_stream_t stream);
/* Fused multi-head self-attention (ldm/modules/attention.py:170-193): out[b, n, h*d + j] = softmax(q k^T * scale) v.
 * q, k, v: fp16 [B*N, >= H*d] views with a common row stride ld (e.g. column blocks of a fused qkv projection);
 * d in {40, 64, 80, 160} (64: CLIP ViT-L/14); scores stay on chip (mma.sync m16n8k16, fp32 online softmax).
 * scale must be positive and finite (O2345_EINVAL otherwise). */
int o2345_attention_f16(const void* q, const void* k, const void* v, int B, int N, int H, int d, int ld, void* out,
                        int ldo, float scale, o2345_stream_t stream);
/* y[M,I] = x[:, :I] * gelu(x[:, I:2I]) */
int o2345_geglu(const void* x, int64_t M, int I, void* y, o2345_stream_t stream);
int o2345_silu(const void* x, int64_t n, void* y, o2345_stream_t stream);
int o2345_transpose_tokens(const void* x, int B, int N, int C, void* y, o2345_stream_t stream);
int o2345_timestep_embedding(const float* t, int B, int dim, void* out, o2345_stream_t stream);
/* y[b, p, c] += e[b * lde + c] */
int o2345_add_channel_bias(void* y, const void* e, int B, int HW, int C, int lde, o2345_stream_t stream);
int o2345_copy_channels(const void* src, int64_t M, int C, void* dst, int ldd, int off, o2345_stream_t stream);
int o2345_nchw_f32_to_cl_f16(const float* x, int B, int C, int HW, void* y, int ldy, int off, o2345_stream_t stream);
int o2345_cl_f16_to_nchw_f32(const void* x, int B, int C, int HW, int ldx, float* y, o2345_stream_t stream);
/* eps = [unconditional | conditional] halves of n elements each; writes x_prev and (optionally) pred_x0. */
int o2345_cfg_ddim_update(const float* x, const float* eps, const float* noise, int64_t n, float scale, float a_t,
                          float a_prev, float sigma_t, float sqrt_one_minus_at, float* x_prev, float* pred_x0,
                          o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Row A8: front end of the CLIP ViT-L/14 image tower (FrozenCLIPImageEmbedder.preprocess + the patch embedding's patch
 * gather, ldm/modules/encoders/modules.py:362-370).  mean3 / std3 are HOST pointers to three floats.
 * out [B * (res/patch)^2, kp] fp16: row (b, py, px), column (c, ky, kx) = bicubic(align_corners) resize of x [B,3,H,W]
 * (fp32, [-1,1]) to res x res, mapped to [0,1] and normalised; columns 3 patch^2 .. kp-1 zero.
 * ------------------------------------------------------------------------------------------ */
int o2345_clip_patches(const float* x, int B, int H, int W, int res, int patch, const float* mean3, const float* std3, int kp,
                       void* out, o2345_stream_t stream);
/* tok [B*N, d] fp16: row 0 of every image := class_embedding + pos[0]; rows n >= 1 += pos[n] (cls, pos fp32 on the device) */
int o2345_clip_add_positions(void* tok, const float* cls, const float* pos, int B, int N, int d, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Mesh rasterizer (render_eval.py): V views of one triangle mesh, one sample at every pixel centre, bit-reproducible.
 * Stands in for the reference's Blender / BlenderProc evaluation renderer (render/single_render_eval.py) for geometry,
 * silhouette and depth; colour is the defined model below, not Cycles.  oracle/raster_oracle.py restates every rule.
 *   vertices   camera space c = R p + t (OpenCV: x right, y down, z forward), pixel x = fx * c.x / c.z + cx (y alike),
 *              snapped to fixed point with 8 subpixel bits (round to nearest even); every float op rounded to nearest in
 *              the order of csrc/raster.cu, without FMA contraction;
 *   triangles  int64 edge functions, top-left fill rule, pixel (i, j) sampled at (i + 0.5, j + 0.5); no back-face culling.
 *              Dropped: zero screen area, any vertex at camera z <= near, any vertex projecting 2^21 pixels or more
 *              from the image origin;
 *   depth      perspective-correct camera z; per pixel the smallest (z bits << 32 | triangle id) wins, so equal depths go
 *              to the lower id and the result does not depend on execution order.
 * ------------------------------------------------------------------------------------------ */
typedef struct o2345_raster_mesh {
  const float* verts;      /* [nv,3] world positions                                                               */
  const float* colors;     /* [nv,3] base colour per vertex, or NULL (white)                                       */
  const float* uvs;        /* [nv,2] texture coordinates (glTF: origin at the image's top-left), or NULL           */
  const int32_t* faces;    /* [nf,3] vertex indices; a face with an index outside [0, nv) is dropped               */
  const int32_t* face_tex; /* [nf] texture of each face (-1 or >= n_tex: none), or NULL                            */
  const uint8_t* texels;   /* RGBA8 texels of every texture, row-major, packed one after another                    */
  const int32_t* tex_info; /* [n_tex,5]: first texel, width, height, wrap s, wrap t (O2345_WRAP_*)                  */
  const float* normals;    /* [nv,3] vertex normals, or NULL (used only with tangents and face_ntex)                */
  const float* tangents;   /* [nv,4] tangent xyz and handedness w (glTF TANGENT), or NULL                          */
  const int32_t* face_ntex;/* [nf] tangent-space normal texture of each face (-1 or >= n_tex: none), or NULL       */
  int64_t nv, nf;
  int n_tex;
} o2345_raster_mesh;

#define O2345_WRAP_REPEAT 0
#define O2345_WRAP_CLAMP 1
#define O2345_WRAP_MIRROR 2
#define O2345_SHADE_UNLIT 0    /* colour = base colour as stored                                                     */
#define O2345_SHADE_LAMBERT 1  /* colour = base colour * (0.4 + 0.6 * max(n.z, 0)), n the camera-facing world normal */

/* Bytes of scratch o2345_raster needs (-1 for negative sizes). */
int64_t o2345_raster_scratch_bytes(int64_t nv, int64_t nf, int V, int W, int H);
/* w2c [V,3,4] (row-major [R | t]), intr [V,4] = (fx, fy, cx, cy).  Outputs (any may be NULL), pixel (v, j, i) at
 * index (v * H + j) * W + i: color [.,3] (perspective-correct vertex colour times the bilinear texture sample of the
 * face's texture, then the shading term), alpha (1 covered, 0 background), depth (camera z, 0 background), normal [.,3]
 * (unit world-space face normal turned toward the camera centre), tri (face index, -1 background).  Background pixels
 * are all zero.
 * Normal maps: for a face with a valid face_ntex when normals and tangents are given, with the perspective-correct weights
 * of colour and uv (fp32, rounded to nearest, no contraction):
 *   N = normalize(interpolated normal), T = normalize(interpolated tangent xyz), w = -1 if the interpolated tangent w < 0
 *   else 1, B = (N x T) * w, t = 2 * bilinear sample of texture face_ntex - 1, n = normalize((t.x T + t.y B) + t.z N),
 * and s * n replaces the face normal in `normal` and in the shading term, s = +1 or -1 the sign that turns the face's
 * normal in its own corner order toward the camera (as the face normal output is turned).
 * A face whose N, T or n has zero or non-finite length keeps its face normal; so does every other face. */
int o2345_raster(const o2345_raster_mesh* mesh, int V, const float* w2c, const float* intr, int W, int H, float near,
                 int shading, void* scratch, int64_t scratch_bytes, float* color, float* alpha, float* depth,
                 float* normal, int32_t* tri, o2345_stream_t stream);
/* Tuning hook (tools/time_raster.py): triangles whose clipped bounding box holds more than `pixels` pixel centres are
 * walked by a warp instead of one thread; 0 restores the default (64). */
void o2345_debug_raster_split(int pixels);

/* ------------------------------------------------------------------------------------------
 * Mesh scoring (eval_mesh.py, o2345/mesh_metrics.py): F-Score and Chamfer distance between two surfaces from area-uniform
 * samples and exact nearest neighbours.  The reference has no metric code; oracle/metrics_oracle.py restates every rule.
 * ------------------------------------------------------------------------------------------ */
/* Bytes of scratch o2345_surface_sample needs (-1 for nf < 1). */
int64_t o2345_surface_sample_scratch_bytes(int64_t nf);
/* n points drawn area-uniformly on the triangles faces [nf,3] (int32) of verts [nv,3] -> pts [n,3], face_id [n] (int32).
 *   weight of face t   |(B - A) x (C - A)| in fp64 from the fp32 vertices, every operation rounded to nearest, no
 *                      contraction; 0 for a face with an index outside [0, nv) or a non-finite weight;
 *   CDF                sequential fp64 cumulative sums inside chunks of 1024 faces, a sequential scan of the chunk
 *                      totals, each chunk's offset added to its entries;
 *   sample i           u_k = top 53 bits of output 3i + k of splitmix64 seeded with `seed` (z = seed + (c + 1) *
 *                      0x9E3779B97F4A7C15, then the splitmix64 finaliser), times 2^-53; the face is the first whose CDF
 *                      exceeds u_0 * total (the first that reaches the total if the product rounds up to it); with
 *                      s = sqrt(u_1): p = ((1 - s) A + s (1 - u_2) B) + s u_2 C in fp64, rounded once to fp32.
 * Returns O2345_EINVAL when the weights sum to zero: that check reads the total on the host, so this call synchronises
 * the stream once (after the CDF, before the sampling kernel).  scratch: 8-byte aligned. */
int o2345_surface_sample(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t n, uint64_t seed,
                         void* scratch, int64_t scratch_bytes, float* pts, int32_t* face_id, o2345_stream_t stream);
/* Bytes of scratch o2345_nearest needs (-1 for sizes out of range); a function of n_ref only (n_query is checked). */
int64_t o2345_nn_scratch_bytes(int64_t n_ref, int64_t n_query);
/* Exact nearest neighbour: for every query point (query [n_query,3]) the reference point (ref [n_ref,3]) with the least
 * d2 = (dx*dx + dy*dy) + dz*dz, d = query - ref, every fp32 operation rounded to nearest; equal d2 go to the lower
 * reference index.  -> dist2 [n_query] (that d2), index [n_query] (int32).  A uniform grid of cubic cells is built over
 * the reference bbox on the device (at most 256 cells per axis); its search bound is conservative under rounding, so
 * the result equals a brute-force search bit for bit.  Coordinates must be finite.  scratch: 16-byte aligned. */
int o2345_nearest(const float* ref, int64_t n_ref, const float* query, int64_t n_query, void* scratch, int64_t scratch_bytes,
                  float* dist2, int32_t* index, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Mesh simplification (simplify_mesh.py, run.py --target_faces, o2345/mesh_simplify.py): parallel half-edge collapse
 * driven by quadric error.  Every output vertex is an input vertex.  The reference has no simplifier;
 * oracle/simplify_oracle.py restates every rule.
 * ------------------------------------------------------------------------------------------ */
/* Bytes of scratch o2345_simplify needs (-1 for sizes out of range). */
int64_t o2345_simplify_scratch_bytes(int64_t nv, int64_t nf);
/* Reduces the triangles faces [nf,3] (int32) of verts [nv,3] to target_faces or target_faces - 1 faces, unless no legal
 * collapse is left first.  Faces with a repeated index are dropped first.  Works in rounds on the mesh as it stood at the
 * round's start:
 *   quadrics   once: n = (B - A) x (C - A) in fp64, p = (n / |n|, -(n / |n|) . A), Q_f = |n| / 2 * p p^T (0 for |n| = 0);
 *              a vertex sums its faces' Q_f in ascending face order;
 *   locks      a vertex is kept when an edge at it does not have exactly two faces or its faces are not one closed fan;
 *   u -> v     u unlocked, v a neighbour; the vertices adjacent to both are exactly the two opposite uv, each of valence
 *              >= 4, val(u) + val(v) - 4 >= 3, and no face of u without v flips or collapses (n' . n > 0, fp64);
 *   cost       (v, 1)^T (Q_u + Q_v) (v, 1) in fp64, rounded to fp32, non-positive results as +0; u proposes the legal v
 *              with the least (cost, v) under the key (bits(cost) << 32) | u;
 *   selection  each key is min-reduced onto the closed 1-rings of u and v and accepted where it holds every one of them
 *              (at most ceil((F - target) / 2): the least keys); accepted collapses apply together: u -> v in u's faces
 *              (winding kept), the two faces of uv deleted, Q_v += Q_u.
 * Every floating-point operation is rounded to nearest in the order of csrc/simplify.cu, without FMA contraction.
 * Outputs: vertex_index [nv] (capacity; the first out_counts[0] entries are the input indices of the referenced vertices,
 * ascending), out_faces [nf,3] (capacity; the first out_counts[1] faces, renumbered into vertex_index, in ascending input
 * order), out_counts [3] (int32: vertices, faces, rounds).  Returns O2345_EINVAL for a face index outside [0, nv) or a
 * non-finite coordinate.  This call synchronises the stream once to read those checks and once per round to read the
 * number of accepted collapses.  scratch: 16-byte aligned. */
int o2345_simplify(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t target_faces, void* scratch,
                   int64_t scratch_bytes, int32_t* vertex_index, int32_t* out_faces, int32_t* out_counts, o2345_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Texture baking (o2345/mesh_texture.py, run.py / simplify_mesh.py --texture_size): one isometric chart per face packed
 * into an N x N atlas, the surface point behind every texel a chart owns, push-pull fill of the rest, and colours taken
 * from a source mesh.  The reference has no texture baking; oracle/texture_oracle.py restates every rule.
 * N is a power of two in [64, 8192].  Every floating-point operation is rounded to nearest in the order of
 * csrc/texture.cu, without FMA contraction.
 * ------------------------------------------------------------------------------------------ */
/* Bytes of scratch o2345_texture_atlas needs (-1 for sizes out of range). */
int64_t o2345_texture_atlas_scratch_bytes(int64_t nf);
/* The atlas of the triangles faces [nf,3] (int32) of verts [nv,3]:
 *   chart    base = the longest of the edges (v0v1, v1v2, v2v0) by fp32 squared length, the first on ties; a = its first
 *            vertex, b its second, c the third; L = |b - a|, d = (c - a).(b - a) / L, h = |(b - a) x (c - a)| / L in fp64
 *            from the fp32 vertices, rounded once to fp32 (d and h are 0 for L = 0; d is clamped to [0, L]);
 *   box      w = ceil(L rho) + 4, hgt = ceil(h rho) + 4 texels (a padding of 2 on each side);
 *   packing  boxes sorted by height descending, then face index; next-fit shelves: a box goes at the cursor unless it
 *            would cross x = N, when a new shelf opens below the tallest box of the current one; it fits when every box
 *            lies inside N x N;
 *   scale    rho0 = sqrt(0.5 N^2 / S), S = the sum of L h in fp64 (sequential inside chunks of 1024 faces, then over the
 *            chunk totals); rho_j = rho0 * j / 64; j = 1 must fit (else O2345_EINVAL), then a binary search over
 *            lo = 1, hi = 257 keeps the largest j that fits.
 * Outputs: uv [nf,3,2] (row k for corner faces[f,k]: a at (x+2, y+2), b at (x+2+L rho, y+2), c at (x+2+d rho, y+2+h rho),
 * divided by N; texel i's centre is at (i + 0.5) / N), boxes [nf,4] int32 (x, y, w, hgt), owner [N*N] int32 (the face whose
 * box holds the texel, -1 where none does), *rung_host = j and *rho_host = rho_j (either may be NULL).  Returns
 * O2345_EINVAL for a face index outside [0, nv), a non-finite coordinate, faces without area or charts that do not fit
 * at j = 1.  This call synchronises the stream once to read the checks and the sum, then once per trial of the search
 * (about 9 times).  scratch: 16-byte aligned. */
int o2345_texture_atlas(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int N, void* scratch,
                        int64_t scratch_bytes, float* uv, int32_t* boxes, int32_t* owner, int32_t* rung_host,
                        double* rho_host, o2345_stream_t stream);
/* Bytes of scratch o2345_chart_atlas needs (-1 for sizes out of range); it includes 8 N^2 bytes for the owner keys. */
int64_t o2345_chart_atlas_scratch_bytes(int64_t nv, int64_t nf, int N);
/* A second atlas of the same triangles, with multi-face charts (--atlas charts).  Its uv and owner follow the contract of
 * o2345_texture_atlas, so o2345_texel_points, o2345_texture_fill and the writers take it unchanged.  In fp64 from the fp32
 * vertices, every operation rounded to nearest in the order of csrc/texture.cu:
 *   label    n = (P1 - P0) x (P2 - P0); axis a = the largest |n_a| (the lower axis on ties); label = 2a + (n_a < 0);
 *            a zero or non-finite n gives label 6, a chart of the face's own;
 *   project  (u, v) = (p[(a+1) % 3], p[(a+2) % 3]) in fp32, u negated when n_a < 0 (so every face of a label has positive
 *            uv area and |n . axis| >= |n| / sqrt(3): no face flips, stretch <= sqrt(3)); label 6 projects along z;
 *   charts   connected components of the faces that share an edge with exactly two (face, edge) uses, on two faces, and
 *            the same key (round 0: the label); boundary, non-manifold and degenerate edges cut; a chart's id is its
 *            least face index;
 *   overlap  faces f, g of a chart overlap when their projected triangles share an interior point: with
 *            orient(a, b, p) = (bx - ax)(py - ay) - (by - ay)(px - ax), a triangle of orient 0 has no interior; for each
 *            edge (t_k, t_k+1) of either triangle, s = orient(t_k, t_k+1, t_k+2) and o_j = the other triangle's three
 *            orients; they are separated when max o_j <= min(0, s) or min o_j >= max(0, s);
 *   cut      a chart with an overlap ranks its m faces by (x0 + x1) + x2 of their corners along its longer extent (u on
 *            ties), ties by face index; the first m / 2 take side 0, the rest side 1; the next round's key is
 *            2 id + side (side 0 for charts without overlap); rounds repeat until no chart overlaps;
 *   extent   per chart, min and max of its corners' u and v; e = max - min in fp64 rounded up to fp32;
 *   packing  box = ceil(e_u rho) + 4 by ceil(e_v rho) + 4, the shelves and the rung search of o2345_texture_atlas over the
 *            charts in id order, with S = the sum of e_u e_v (fp64, the same chunked order);
 *   uv       (box origin + 2 + (p - chart min) rho) / N per coordinate in fp64, rounded to fp32;
 *   owner    a texel of a chart's box is a candidate of each face of the chart whose uv bounding box (uv * N in fp32) grown
 *            by 2 holds its centre; key = (fp32 of the squared distance of the centre to the face's uv triangle, f), the
 *            least key wins.  The distance is 0 when the three edge orients (b, c), (c, a), (a, b) of the centre are all
 *            >= 0 or all <= 0 on a triangle of non-zero orient, else |q - ((la a + lb b) + lc c)|^2 with the barycentrics
 *            of the 7-region test of o2345_texel_points (corners in face order).  A texel without candidate is -1.
 * Outputs: uv [nf,3,2], boxes [nf,4] int32 (the box of the face's chart), owner [N*N], labels [nf] int32, chart [nf] int32
 * (its chart's id), *rung_host, *rho_host, *rounds_host (the cut rounds) and *charts_host (the chart count); any of the
 * host pointers may be NULL.  Returns O2345_EINVAL for a face index outside [0, nv), a non-finite coordinate, charts
 * without area or charts that do not fit at j = 1.  Synchronises to read the checks, one flag per component pass, the
 * chart count and the overlap flag per round, the sum and a fit flag per trial.  scratch: 16-byte aligned. */
int o2345_chart_atlas(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int N, void* scratch,
                      int64_t scratch_bytes, float* uv, int32_t* boxes, int32_t* owner, int32_t* labels, int32_t* chart,
                      int32_t* rung_host, double* rho_host, int32_t* rounds_host, int32_t* charts_host,
                      o2345_stream_t stream);
/* Bytes of scratch o2345_texel_points needs (-1 for an invalid N). */
int64_t o2345_texel_points_scratch_bytes(int N);
/* For the faces and the uv / owner of o2345_texture_atlas: texel_index [N*N] (capacity; the first *count entries are the
 * owned texels, ascending), texel_face [N*N] their faces and points [N*N,3] their surface points: the point of the chart's
 * triangle (uv * N, corners a, b, c as in the atlas) closest to the texel centre as barycentrics (la, lb, lc) in fp64
 * (the 7-region test), then (la A + lb B) + lc C in fp32 with the weights rounded to fp32.  A texel whose closest point
 * is a corner gets that vertex's position exactly.  count: one int32 on the device.  Faces must be ones the atlas
 * accepted (a face index outside [0, nv) gives NaN points).  scratch: 16-byte aligned. */
int o2345_texel_points(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                       const int32_t* owner, int N, void* scratch, int64_t scratch_bytes, int32_t* texel_index,
                       float* points, int32_t* texel_face, int32_t* count, o2345_stream_t stream);
/* Bytes of scratch o2345_texture_fill needs (-1 for an invalid N). */
int64_t o2345_texture_fill_scratch_bytes(int N);
/* texture [N,N,3] fp32 := rgb [*count,3] at texel_index (as o2345_texel_points lists them); every texel with owner < 0 is
 * filled by push-pull: pull builds levels N/2 .. 1 where a texel's weight is the sum of its 2 x 2 children's (an owned
 * texel weighs 1) and its colour their weight-normalised mean (((w0 c0 + w1 c1) + w2 c2) + w3 c3) / (((w0 + w1) + w2) + w3)
 * in fp32 (children row-major), 0 without weight; push, from coarse to fine, gives every texel of weight 0 its parent's
 * colour.  Owned texels are never changed.  scratch: 16-byte aligned. */
int o2345_texture_fill(const int32_t* texel_index, const int32_t* count, const float* rgb, const int32_t* owner, int N,
                       void* scratch, int64_t scratch_bytes, float* texture, o2345_stream_t stream);
/* Colour transfer from a source mesh verts [nv,3], faces [nf,3], colors [nv,3] fp32: for point i of points [n,3], face f =
 * sample_face[nn_index[i]] (the face of its nearest surface sample, o2345_surface_sample + o2345_nearest), the closest
 * point of f to the point as in o2345_texel_points (corners in face order) and rgb [n,3] = (l0 C0 + l1 C1) + l2 C2 in fp32.
 * An index out of range gives NaN. */
int o2345_transfer_colors(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* colors,
                          const float* points, int64_t n, const int32_t* nn_index, const int32_t* sample_face,
                          int64_t n_samples, float* rgb, o2345_stream_t stream);

/* Normal maps (o2345/mesh_texture.py, run.py / simplify_mesh.py --normal_map; mesh_io's writers and o2345_raster read the
 * same frame).  For a face with corners P0, P1, P2 (in face order) and uv rows (u_k, v_k) (glTF: v down the image), in fp64
 * from the fp32 inputs, every operation rounded to nearest in the order of csrc/texture.cu:
 *   e1 = P1 - P0, e2 = P2 - P0, (du1, dv1) = uv1 - uv0, (du2, dv2) = uv2 - uv0, det = du1 dv2 - du2 dv1,
 *   dp/du = (dv2 e1 - dv1 e2) / det, dp/dv = (du1 e2 - du2 e1) / det (per component),
 *   T = dp/du / |dp/du|, B = -dp/dv / |dp/dv| (+Y up the image), N = (e1 x e2) / |e1 x e2|, |a| = sqrt((ax ax + ay ay) + az az);
 *   a world normal n is coded as (n.T, n.B, n.N) / |n|, rounded to fp32.
 * The atlas's charts are isometric, so T, B, N are orthonormal and t.x T + t.y B + t.z N decodes exactly.  A face with
 * det = 0 (or not finite) or no area, and a normal that is zero or not finite, give (0, 0, 1).  The texel's byte code is
 * round_half_even((c + 1) * 127.5) per component of v / |v| in fp32 (|v| as above in fp32); a vector of zero or non-finite
 * length is (0, 0, 1), i.e. (128, 128, 255).
 * out [n,3] fp32 := the code of normals [n,3] in the frame of face texel_face[i] with the atlas uv [nf,3,2] (a face index
 * out of range gives NaN). */
int o2345_tangent_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                          const int32_t* texel_face, const float* normals, int64_t n, float* out, o2345_stream_t stream);
/* As o2345_tangent_normals, in the frame a decoder builds from NORMAL and TANGENT (T, w): B = w (N x T) with
 * w = sign((N x T) . (-dp/dv)) (+1 on 0), N x T in the operation order of (b - a) x (c - a) with a = 0.  For the charts
 * of o2345_chart_atlas, where dp/du and dp/dv are not orthogonal; on an isometric chart it is the frame above. */
int o2345_tangent_normals_decoded(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* uv,
                                  const int32_t* texel_face, const float* normals, int64_t n, float* out,
                                  o2345_stream_t stream);
/* out [n,3] uint8 := the byte codes of texture [n,3] fp32 (after o2345_texture_fill), as above; n <= 8192^2. */
int o2345_normal_quantise(const float* texture, int64_t n, uint8_t* out, o2345_stream_t stream);
/* Bytes of scratch o2345_vertex_normals needs (-1 for sizes out of range). */
int64_t o2345_vertex_normals_scratch_bytes(int64_t nv, int64_t nf);
/* normals [nv,3] fp32: per vertex the sum of (B - A) x (C - A) (fp64) over its faces in ascending face order, divided by
 * its length and rounded once to fp32; (0, 0, 0) for a vertex without faces or with a zero sum.  Returns O2345_EINVAL for
 * a face index outside [0, nv) or a non-finite coordinate: this call synchronises the stream once to read that check.
 * scratch: 16-byte aligned. */
int o2345_vertex_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, void* scratch,
                         int64_t scratch_bytes, float* normals, o2345_stream_t stream);

/* Input-view projection (o2345/mesh_texture.py, run.py --project_input; csrc/project.cu).  The constants are not tuned on
 * real outputs: no released checkpoint is available to the tests. */
#define O2345_PROJECT_COS_LO 0.3f   /* facing weight 0 at or below this cosine ... */
#define O2345_PROJECT_COS_HI 0.7f   /* ... and 1 at or above this one */
#define O2345_PROJECT_TAU_PIX 2.0f  /* depth-test slack, in depth-buffer pixels of slope */
/* For point i of points [n,3] with normal normals[i] (any length) and colour base[i] (fp32), the camera w2c [3,4] (device,
 * OpenCV) with (fx, fy, cx, cy), the photo RGB uint8 [H,W,3], alpha uint8 [H,W] (or null: opaque) and the depth buffer
 * [scale H, scale W] fp32 of the mesh rendered by o2345_raster with (scale fx, scale fy, scale (cx + 0.5), scale (cy + 0.5)),
 * every operation in fp32 rounded to nearest in this order:
 *   q_r = ((M[r][0] p.x + M[r][1] p.y) + M[r][2] p.z) + M[r][3]; weight 0 unless near < q.z <= FLT_MAX;
 *   x = (fx q.x) / q.z + cx, y = (fy q.y) / q.z + cy (pixel i's centre at i); weight 0 unless 0 <= x <= W-1, 0 <= y <= H-1;
 *   weight 0 unless 0 < |n| <= FLT_MAX, |a| = sqrt((a.x a.x + a.y a.y) + a.z a.z);
 *   c_k = -((M[0][k] M[0][3] + M[1][k] M[1][3]) + M[2][k] M[2][3]), d = c - p,
 *   cos = ((n.x/|n|)(d.x/|d|) + (n.y/|n|)(d.y/|d|)) + (n.z/|n|)(d.z/|d|);
 *   w_a = t clamped to [0, 1] (NaN -> 0), t = (cos - COS_LO) / (COS_HI - COS_LO); weight 0 unless w_a > 0;
 *   the buffer pixel (j, k) = (min(floor(scale (x + 0.5)), scale W - 1), min(floor(scale (y + 0.5)), scale H - 1)) holds D;
 *   tau = ((TAU_PIX q.z) / (scale fx)) / max(cos, COS_LO); weight 0 unless D <= 0 (background) or q.z - D <= tau;
 *   weight = w_a a, a = min(bilinear(alpha) / 255, 1) (1 without alpha);
 *   out = base + weight (bilinear(photo) / 255 - base) per channel where weight > 0, else base bit for bit.
 * bilinear(img) at (x, y): x0 = floor(x), x1 = x0 + 1 (y alike), taps nw, ne, sw, se with weights (x1 - x)(y1 - y),
 * (x - x0)(y1 - y), (x1 - x)(y - y0), (x - x0)(y - y0), summed as ((v_nw w_nw + v_ne w_ne) + v_sw w_sw) + v_se w_se on the
 * byte values; a tap past the last column or row has weight 0 and reads the last one.  weight [n] and out [n,3] fp32. */
int o2345_project_view(const float* points, const float* normals, const float* base, int64_t n, const float* w2c,
                       float fx, float fy, float cx, float cy, float near, const uint8_t* photo, const uint8_t* alpha,
                       int W, int H, const float* depth, int scale, float* out, float* weight, o2345_stream_t stream);
/* normals [n,3] fp32 := the unit normal of face face_index[i] of verts [nv,3], faces [nf,3]: (B - A) x (C - A) in fp64,
 * divided by its length and rounded once; (0, 0, 0) for an index out of range or a face without area. */
int o2345_face_normals(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const int32_t* face_index,
                       int64_t n, float* normals, o2345_stream_t stream);

/* Mesh cleaning (o2345/mesh_clean.py, run.py / simplify_mesh.py --min_component; csrc/clean.cu).  For verts [nv,3] fp32
 * and faces [nf,3] int32 (welded first: components follow vertex indices) and 0 < min_component <= 1:
 *   components  two faces belong to one component when they share a vertex index (a bowtie vertex joins its fans);
 *               components are numbered by their least face: label [nf] int32 := the component of each face, nc of them;
 *   area        of a face: 0.5 sqrt(n . n), n = (B - A) x (C - A) in fp64 from the fp32 positions; of component c (area [nc]
 *               fp64): its faces' areas in ascending face order, summed sequentially inside chunks of 1024 faces and then
 *               sequentially over the chunk totals, each sum from +0.0;
 *   largest     L: the greatest area, the least component on ties;
 *   winding     of c != L (winding [nc] fp64, 0 at L): at the centroid p = ((A + B) + C) / 3 (fp64) of c's least face,
 *               (the sum of the solid angles of L's faces, in ascending face order and chunked as the area) / (4 pi); the
 *               solid angle of ABC is 2 atan2(a . (b x c), ((|a||b|)|c| + (a . b)|c| + (a . c)|b|) + (b . c)|a|), a = A - p
 *               etc., |a| = sqrt((a.x a.x + a.y a.y) + a.z a.z), with the atan2 of csrc/clean.cu (+, -, *, /, sqrt only);
 *               c is enclosed when |winding| >= 0.5 (either face orientation);
 *   keep        keep [nc] uint8 := c == L, or c is not enclosed and area[c] >= min_component area[L] (fp64 product);
 *   output      vertex_index [nv'] := the input indices of the vertices a kept face references, ascending; faces_out
 *               [nf',3] := the kept faces in input order, renumbered into vertex_index.
 * counts_host [6] := (nc, L, kept components, enclosed components, nv', nf').  Every float operation rounds to nearest
 * in the stated order, so the outputs do not depend on scheduling.  Synchronises (see the conventions above). */
int64_t o2345_clean_mesh_scratch_bytes(int64_t nv, int64_t nf);
int o2345_clean_mesh(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, double min_component, void* scratch,
                     int64_t scratch_bytes, int32_t* label, double* area, double* winding, uint8_t* keep,
                     int32_t* vertex_index, int32_t* faces_out, int32_t* counts_host, o2345_stream_t stream);

/* Ambient occlusion (o2345/mesh_texture.py, run.py / simplify_mesh.py --ambient_occlusion; csrc/ao.cu).  For point p with
 * normal n and the occluder mesh verts [nv,3] fp32, faces [nf,3] int32, AO(p) is the share of the k directions of dirs
 * [k,3] (fp32, turned into n's frame) for which the segment p + t w, t in [t_min, t_max], hits no face.  The library's
 * callers pass K = 256 points of a golden-angle spiral on the unit disk lifted to the hemisphere (Malley's method, so they
 * are cosine-distributed): d_k = (r cos phi, r sin phi, sqrt(1 - r^2)), r = sqrt((k + 1/2) / K), phi = k pi (3 - sqrt 5),
 * computed in fp64 and rounded once to fp32 on the host (no device sin / cos), the same table at every point: the result
 * moves in steps of 1/256, below one 8-bit code, so there is no per-point rotation.  t_min = 1e-3 D and t_max = 0.1 D,
 * D the diagonal of the box of the nv vertices (fp64, rounded once); t_min drops the hits at t = 0 on the faces around
 * a vertex the ray starts from.  Every fp32 operation is rounded to nearest in this order, without FMA contraction:
 *   frame     |n| = sqrt((n.x n.x + n.y n.y) + n.z n.z), u = n / |n| per component; s = copysign(1, u.z),
 *             a = -1 / (s + u.z), b = (u.x u.y) a, T = (1 + ((s u.x) u.x) a, s b, -(s u.x)), B = (b, s + (u.y u.y) a, -u.y)
 *             (Duff et al. 2017), w = (d.x T + d.y B) + d.z u per component.  A normal of zero or non-finite length, or a
 *             point with a non-finite coordinate, gives AO = 1;
 *   box test  of a box [lo, hi] on the segment [0, t_max]: per axis c, when 1 / w_c rounds to a finite i_c the slab gives
 *             t1 = (lo_c - p_c) i_c, t2 = (hi_c - p_c) i_c and the interval [min(t1, t2), max(t1, t2)]; otherwise the axis
 *             passes when lo_c <= p_c <= hi_c and gives no interval.  The box passes when every axis passes and
 *             max(0, the interval starts) <= min(t_max, the interval ends);
 *   face      the face's box is the min / max of its corners' coordinates grown by pad = D' 2^-13 on every side (D' the
 *             diagonal above, rounded to fp32; lo - pad, hi + pad rounded), and a face is hit when its box passes and the
 *             watertight test (Woop, Benthin and Wald, JCGT 2013; no culling) accepts:
 *               kz = the axis of the largest |w_c| (the lower on ties), kx = kz + 1, ky = kx + 1 (mod 3), kx and ky
 *               swapped when w_kz < 0; Sx = w_kx / w_kz, Sy = w_ky / w_kz, Sz = 1 / w_kz;
 *               per corner V (A, B, C in face order): P = V - p, x = P_kx - Sx P_kz, y = P_ky - Sy P_kz;
 *               U = Cx By - Cy Bx, V = Ax Cy - Ay Cx, W = Bx Ay - By Ax; if any of them is 0 all three are recomputed as
 *               fp32(fp64 product - fp64 product) of the same terms;
 *               no hit if one of U, V, W is < 0 and one is > 0; det = (U + V) + W, no hit if det = 0;
 *               T = ((U Sz A_kz + V Sz B_kz) + W Sz C_kz) with each Sz P_kz rounded first, T' and |det| the values with
 *               det's sign taken off both; hit when t_min |det| <= T' <= t_max |det|.
 *             The box stops the fp32 edge functions of a nearly degenerate face from accepting rays that pass far from
 *             it; a ray through a shared edge or vertex is decided the same way by both faces' edge functions, so a
 *             closed mesh lets none through.
 *   result    out[i] = (number of directions without a hit) / k in fp32.  The count is a count of any-hits, so it does not
 *             depend on which face is found first.
 * The faces are searched through an LBVH built on the device (30-bit Morton codes of face-box centres, ties by face index;
 * Karras 2012); a node's box is the exact min / max of the padded face boxes below it, and the box test only moves
 * with its bounds through rounded subtractions and products, so a node never rejects a ray one of its faces passes and
 * the result equals the brute-force search over all faces bit for bit.  Returns O2345_EINVAL for a face index outside
 * [0, nv) or a non-finite vertex: the call synchronises the stream once to read that check.  nf = 0 gives AO = 1
 * everywhere; n = 0 does nothing.  scratch: 16-byte aligned. */
int64_t o2345_ambient_occlusion_scratch_bytes(int64_t nv, int64_t nf);
int o2345_ambient_occlusion(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* points,
                            const float* normals, int64_t n, const float* dirs, int k, float t_min, float t_max,
                            void* scratch, int64_t scratch_bytes, float* out, o2345_stream_t stream);

/* Closest points and isotropic remeshing (o2345/mesh_remesh.py, simplify_mesh.py --remesh; csrc/remesh.cu).
 *
 * Closest point.  For a point p (fp32, taken to fp64) and the reference mesh verts [nv,3], faces [nf,3]: over every face,
 * the barycentrics (la, lb, lc) of the 7-region test of o2345_texel_points (corners A, B, C in face order, fp64), the
 * point q = (la A + lb B) + lc C per component in fp64, d = q - p, d2 = (d.x d.x + d.y d.y) + d.z d.z; the face with the
 * least (d2, face index) wins (so of duplicated faces the lowest index), and the point is q rounded to fp32.  The faces
 * are searched through the LBVH of o2345_ambient_occlusion (padded face boxes, exact node boxes).  A node is skipped when
 * its lower bound b > the best d2 so far, where per axis g = (lo - p) or (p - hi) outside the box (0 inside), minus the
 * slack s = M 2^-44 (M the largest |coordinate| of the vertex box), floored at 0, and b = (gx gx + gy gy) + gz gz, every
 * operation of g and b rounded downward.  Why this skips no face the brute force would pick: the computed q of a face
 * lies within a few fp64 ulps of M of the face's box (the weights are in [0, 1] and sum to 1 within 2^-51), far inside
 * s; the face's box is inside the node's; so the real |q_c - p_c| >= g_c per axis, rounding to nearest is monotone, and
 * the face's computed d2 >= b > best.  Nodes with b = best are visited, so ties are decided by the face index as in the
 * brute force, and the result equals it bit for bit.  A point with a non-finite coordinate, or nf = 0, gives NaN and
 * face -1.  Returns O2345_EINVAL for a face index outside [0, nv) or a non-finite vertex (one synchronisation). */
int64_t o2345_closest_points_scratch_bytes(int64_t nv, int64_t nf);
int o2345_closest_points(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* points, int64_t n,
                         void* scratch, int64_t scratch_bytes, float* out_points, int32_t* out_face, o2345_stream_t stream);

/* Remesh.  verts [nv,3] fp32, faces [nf,3] int32 (faces with a repeated index are dropped; an index outside [0, nv) or a
 * non-finite coordinate is refused), target edge length L (fp32; the library's callers pass L = sqrt(4 A / (sqrt(3) N))
 * rounded once to fp32, A the input's area summed in fp64 in ascending face order, N the target face count).  In fp64:
 * hi = L (4/3), lo = L 0.8, hi2 = hi hi, lo2 = lo lo; len2(a, b) = (d.x d.x + d.y d.y) + d.z d.z, d = b - a from the fp32
 * positions; an edge is long when len2 > hi2 and short when len2 < lo2.  Locks are the simplifier's (o2345_simplify),
 * recomputed from the current faces at every round; a vertex without faces is locked.  The edge id of an edge is 3 g + k,
 * its half-edge in its least face g.  Each of `iterations` iterations runs, on the mesh as the previous step left it:
 *   split     rounds (at most 64 per iteration, fewer when a round splits nothing): each face's key is the greatest of
 *             (bits(fp32(len2)) << 32) | edge id over its long edges with one or two faces; an edge splits when it is the
 *             key of each of its faces.  The new vertices, numbered nv + i in edge-id order, are the fp32 midpoints
 *             (a + b) * 0.5f (so a boundary edge's new vertex lies on it and is locked); a split face (p, q, r) on edge pq
 *             (corners k, k + 1) becomes (p, m, r) and the face appended in face order is (m, q, r).  A round that would
 *             exceed the capacities returns O2345_ENOSPC with counts_host[0..1] = the vertices and faces it needs;
 *   collapse  rounds until none is accepted (each removes two faces per collapse: at most nf / 2 rounds): every unlocked
 *             u proposes the neighbour v with the least (bits(fp32(len2(u, v))), v) among its short neighbours where u -> v
 *             is the simplifier's legal collapse and every other neighbour x of u has len2(v, x) <= hi2; the key is
 *             (bits << 32) | u, claims and acceptance are the simplifier's, and every accepted u -> v applies (u's faces
 *             take v, the two faces of uv are deleted, the rest keep their order);
 *   flip      rounds until none is accepted (every flip lowers the integer sum of (val - t)^2 over the mesh, t = 4 for a
 *             locked vertex and 6 otherwise, so the rounds end): for the edge ab of a face f = (a, b, c) that is its
 *             least face, with exactly two faces, the other holding b -> a with third vertex d: legal when d != c, cd is
 *             not an edge, val(a), val(b) > 3 and the new faces (a, d, c), (d, b, c) have normals (B - A) x (C - A) whose
 *             dot with both old faces' normals is > 0 (fp64, so no new face is degenerate or folded); the gain is the drop
 *             of the sum over a, b, c, d, and a flip with gain > 0 claims its four vertices with the least key
 *             ((2^30 - gain) << 32) | edge id; flips holding all four apply together: f := (a, d, c), the other := (d, b, c);
 *   relax     every unlocked vertex p moves to p + (e - n (e . n)), e = c - p, c = (the sum of its neighbours' positions in
 *             ascending index order, fp64, from 0) / their count, n its o2345_vertex_normals normal (fp32, taken to fp64),
 *             e . n = (e.x n.x + e.y n.y) + e.z n.z, each component p + (e - n t) rounded to fp32; all from the positions
 *             before the step (Jacobi);
 *   project   every unlocked vertex moves to its closest point on the input mesh (as given, repeated-index faces included).
 * Every floating-point operation is rounded to nearest in that order, without FMA contraction.  Outputs: out_verts
 * [vertex_capacity,3] (the first counts_host[0] are the referenced vertices in index order: the input's, then the split
 * vertices in creation order), out_faces [face_capacity,3] (the first counts_host[1], in their final order, renumbered),
 * counts_host [5] (int64: vertices, faces, split rounds, collapse rounds, flip rounds).  The result does not depend on the
 * capacities; capacities below nv, nf give O2345_ENOSPC at once.  L must be >= 2^-60 (+inf: no edge is long, every edge
 * short: the mesh collapses as far as the rules allow).  scratch: 16-byte aligned. */
int64_t o2345_remesh_scratch_bytes(int64_t nv, int64_t nf, int64_t vertex_capacity, int64_t face_capacity);
int o2345_remesh(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float target_length, int iterations,
                 int64_t vertex_capacity, int64_t face_capacity, void* scratch, int64_t scratch_bytes, float* out_verts,
                 int32_t* out_faces, int64_t* counts_host, o2345_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* O2345_H_ */
