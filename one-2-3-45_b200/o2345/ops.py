"""Tensor-level wrappers over the C-ABI: torch owns device memory and streams, the library does the work.

Every function takes CUDA fp32 (or the stated integer) tensors, allocates the outputs and scratch the
C-ABI asks for, and enqueues on torch's current stream.  Nothing here computes on the host or with
PyTorch kernels (only allocation / zero-fill / pointer plumbing).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L
from . import mc_tables

_f32, _i32, _u8 = torch.float32, torch.int32, torch.uint8


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t, dtype=None):
    if t is None:
        return None
    if not t.is_cuda:
        raise L.O2345Error("expected a CUDA tensor (the o2345 kernels have no CPU path)")
    if t.device.index != torch.cuda.current_device():
        # the C-ABI launches on the current device's current stream: a tensor of another GPU would be read through a pointer that
        # is not valid there (wrap the call in `with torch.cuda.device(t.device)`, as one process per GPU does by construction)
        raise L.O2345Error(f"tensor on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}")
    if dtype is not None and t.dtype != dtype:
        raise L.O2345Error(f"expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise L.O2345Error("expected a contiguous tensor")
    return C.c_void_p(t.data_ptr())


def _f(t):
    return _p(t, _f32)


def cf32(t):
    """fp32 + contiguous view/copy of a CUDA tensor."""
    return t.detach().to(_f32).contiguous()


# ----------------------------------------------------------------------------- point sources
class PointSource:
    """Keeps the tensors alive that an o2345_points struct points to."""

    def __init__(self, struct, n, keep):
        self.struct, self.n, self._keep = struct, n, keep

    @staticmethod
    def explicit(pts):
        pts = cf32(pts).view(-1, 3)
        s = L.Points(mode=L.PTS_EXPLICIT, pts=pts.data_ptr())
        return PointSource(s, pts.shape[0], (pts,))

    @staticmethod
    def lattice(lin):
        lin = cf32(lin)
        R = lin.numel()
        return PointSource(L.Points(mode=L.PTS_LATTICE, lin=lin.data_ptr(), R=R), R ** 3, (lin,))

    @staticmethod
    def rays(rays_o, rays_d, z):
        rays_o, rays_d, z = cf32(rays_o), cf32(rays_d), cf32(z)
        R, S = z.shape
        s = L.Points(mode=L.PTS_RAYS, rays_o=rays_o.data_ptr(), rays_d=rays_d.data_ptr(), z=z.data_ptr(), S=S,
                     z_stride=S)
        return PointSource(s, R * S, (rays_o, rays_d, z))


# ----------------------------------------------------------------------------- SDF query (B8/B9)
def sdf_pack_weights(w0, b0, w1, b1, w2, b2):
    pack = torch.empty(L.SDF_PACK_FLOATS, dtype=_f32, device=w0.device)
    L.call("o2345_sdf_pack_weights", _f(cf32(w0)), _f(cf32(b0)), _f(cf32(w1)), _f(cf32(b1)), _f(cf32(w2)),
           _f(cf32(b2)), _f(pack), _stream())
    return pack


# SDF MLP kernel used when a call does not say otherwise: forward GEMMs on tensor cores with split-fp16 operands
# (fp32-grade values); L.SDF_FP32 selects the fp32 FMA kernel.
SDF_PRECISION = L.SDF_TC_SPLIT


def sdf_query(src: PointSource, vol_cl, pack, active=None, inactive_sdf=100.0, negate=False, want_feat=False,
              want_latent=False, want_grad=False, precision=None):
    """Returns dict(sdf [n,1], feat [n,127]?, latent [n,16]?, grad [n,3]?)."""
    precision = SDF_PRECISION if precision is None else precision
    n, dev = src.n, vol_cl.device
    D = vol_cl.shape[0]
    out = {"sdf": torch.empty(n, 1, dtype=_f32, device=dev)}
    if want_feat:
        out["feat"] = torch.empty(n, 127, dtype=_f32, device=dev)
    if want_latent:
        out["latent"] = torch.empty(n, 16, dtype=_f32, device=dev)
    if want_grad:
        out["grad"] = torch.empty(n, 3, dtype=_f32, device=dev)
    L.call("o2345_sdf_query", C.byref(src.struct), n, _f(vol_cl), D, _f(pack), _p(active, _u8),
           float(inactive_sdf), int(bool(negate)), int(precision), _f(out["sdf"]), _f(out.get("feat")), _f(out.get("latent")),
           _f(out.get("grad")), _stream())
    return out


# ----------------------------------------------------------------------------- cost volume (B3-B7)
def compact(flags):
    """flags uint8 [n] -> rows int32 [n] (first *count valid), index int32 [n], count int32 [1]."""
    n = flags.numel()
    dev = flags.device
    rows = torch.empty(n, dtype=_i32, device=dev)
    index = torch.empty(n, dtype=_i32, device=dev)
    count = torch.empty(1, dtype=_i32, device=dev)
    scratch = torch.empty(L.load().o2345_compact_scratch_ints(n), dtype=_i32, device=dev)
    L.call("o2345_compact", _p(flags, _u8), n, _p(rows, _i32), _p(index, _i32), _p(count, _i32), _p(scratch, _i32),
           _stream())
    return rows, index, count


def frustum_mask(proj, origin, voxel_size, D, sizeH, sizeW, min_views):
    V = proj.shape[0]
    bits = torch.empty(D ** 3, dtype=_i32, device=proj.device)
    keep = torch.empty(D ** 3, dtype=_u8, device=proj.device)
    L.call("o2345_frustum_mask", _f(proj), V, _f(origin), float(voxel_size), D, int(sizeH), int(sizeW),
           int(min_views), _p(bits, _i32), _p(keep, _u8), _stream())
    return bits, keep


def costvol_gather(feats_nhwc, proj, origin, voxel_size, D, sizeH, sizeW, rows, count, bits, max_rows):
    V, h, w, c = feats_nhwc.shape
    assert c == 16
    cost = torch.empty(max_rows, 32, dtype=_f32, device=proj.device)
    L.call("o2345_costvol_gather", _f(feats_nhwc), V, h, w, int(sizeH), int(sizeW), _f(proj), _f(origin),
           float(voxel_size), D, _p(rows, _i32), _p(count, _i32), max_rows, _p(bits, _i32), _f(cost), _stream())
    return cost


def costvol_gather_lod(feats_nhwc, proj, origin, voxel_size, D, sizeH, sizeW, rows, count, bits, max_rows, parent, pre_feats):
    """Cost rows [max_rows, 2C + 16] = [var(C), mean(C), pre_feats[parent[lin]]] for C = feats_nhwc.shape[-1] (8 or 16)."""
    V, h, w, c = feats_nhwc.shape
    cost = torch.empty(max_rows, 2 * c + 16, dtype=_f32, device=proj.device)
    L.call("o2345_costvol_gather_lod", _f(feats_nhwc), c, V, h, w, int(sizeH), int(sizeW), _f(proj), _f(origin),
           float(voxel_size), D, _p(rows, _i32), _p(count, _i32), max_rows, _p(bits, _i32), _p(parent, _i32), _f(pre_feats),
           _f(cost), _stream())
    return cost


def sdf_voxels(occ, vol_cl, origin, voxel_size, pack, precision=None):
    """[D^3] SDF of every occupied voxel (own latent row, no trilinear fetch), 1.0 elsewhere."""
    precision = SDF_PRECISION if precision is None else precision
    D = vol_cl.shape[0]
    out = torch.empty(D ** 3, dtype=_f32, device=vol_cl.device)
    L.call("o2345_sdf_voxels", _f(occ), _f(vol_cl), D, _f(origin), float(voxel_size), _f(pack), int(precision), _f(out),
           _stream())
    return out


MAX_RUNGS = 16


def prune_by_sdf(sdf, occ, D, ladder):
    """-> minabs [D^3] (window minimum of |sdf|, +inf where occ == 0) and the host list of survivor counts per rung of
    `ladder` (fp32 thresholds; one device-to-host copy per 16 rungs)."""
    dev = sdf.device
    minabs = torch.empty(D ** 3, dtype=_f32, device=dev)
    scratch = torch.empty(D ** 3, dtype=_f32, device=dev)
    counts = []
    for k in range(0, len(ladder), MAX_RUNGS):
        part = ladder[k:k + MAX_RUNGS]
        arr = (C.c_float * len(part))(*part)
        dcounts = torch.empty(len(part), dtype=_i32, device=dev)
        L.call("o2345_prune_by_sdf", _f(sdf), _f(occ), D, arr, len(part), _f(scratch), _f(minabs), _p(dcounts, _i32),
               _stream())
        counts += dcounts.tolist()
    return minabs, counts


def prune_select(minabs, threshold):
    keep = torch.empty(minabs.numel(), dtype=_u8, device=minabs.device)
    L.call("o2345_prune_select", _f(minabs), minabs.numel(), float(threshold), _p(keep, _u8), _stream())
    return keep


def clear_flags(flags, rows, idx):
    L.call("o2345_clear_flags", _p(rows, _i32), _p(idx, _i32), idx.numel(), _p(flags, _u8), _stream())


def gather_rows(rows, n, D, vol_cf):
    """coords [n,4] (0, x, y, z) and the channels of vol_cf [C, D^3] at the first n lattice indices of rows."""
    Cc = vol_cf.shape[0]
    coords = torch.empty(n, 4, dtype=_f32, device=rows.device)
    feats = torch.empty(n, Cc, dtype=_f32, device=rows.device)
    L.call("o2345_gather_rows", _p(rows, _i32), n, D, _f(vol_cf), Cc, _f(coords), _f(feats), _stream())
    return coords, feats


def lod_children(pre_coords, D1, frustum_keep):
    """-> keep uint8 [D1^3] (children seen by > 1 views), parent int32 [D1^3].  Synchronises (argument check)."""
    dev = pre_coords.device
    keep = torch.empty(D1 ** 3, dtype=_u8, device=dev)
    parent = torch.empty(D1 ** 3, dtype=_i32, device=dev)
    err = torch.empty(1, dtype=_i32, device=dev)
    L.call("o2345_lod_children", _f(pre_coords), pre_coords.shape[0], D1, _p(frustum_keep, _u8), _p(keep, _u8),
           _p(parent, _i32), _p(err, _i32), _stream())
    return keep, parent


def dense_scatter(feat, rows, count, D, max_rows, want_cf=True):
    dev = feat.device
    vol_cl = torch.empty(D, D, D, 16, dtype=_f32, device=dev)
    vol_cf = torch.empty(1, 16, D, D, D, dtype=_f32, device=dev) if want_cf else None
    occ = torch.empty(1, 1, D, D, D, dtype=_f32, device=dev)
    L.call("o2345_dense_scatter", _f(feat), _p(rows, _i32), _p(count, _i32), max_rows, D, _f(vol_cl), _f(vol_cf),
           _f(occ), _stream())
    return vol_cl, vol_cf, occ


def occ_nearest(src: PointSource, occ):
    D = occ.shape[-1]
    out = torch.empty(src.n, dtype=_u8, device=occ.device)
    L.call("o2345_occ_nearest", C.byref(src.struct), src.n, _f(occ), D, _p(out, _u8), _stream())
    return out


# ----------------------------------------------------------------------------- sparse conv (B6)
class SparseLevel:
    """index lattice [E^3], row list, device-side count and a host-side upper bound of the rows."""

    def __init__(self, E, rows, index, count, max_rows):
        self.E, self.rows, self.index, self.count, self.max_rows = E, rows, index, count, max_rows


def sp_coarsen(level: SparseLevel) -> SparseLevel:
    Ec = level.E // 2 + 1
    dev = level.rows.device
    flags = torch.empty(Ec ** 3, dtype=_u8, device=dev)
    cmin = torch.empty(3, dtype=_i32, device=dev)
    L.call("o2345_sp_coarsen", _p(level.index, _i32), level.E, _p(level.rows, _i32), _p(level.count, _i32),
           level.max_rows, Ec, _p(flags, _u8), _p(cmin, _i32), _stream())
    rows, index, count = compact(flags)
    return SparseLevel(Ec, rows, index, count, Ec ** 3)


def sp_conv_bn_relu(x, lin: SparseLevel, lout: SparseLevel, mode, kernel, gamma, beta, skip=None, eps=1e-5):
    """One BasicSparse(De)ConvolutionBlock: conv -> BatchNorm(batch stats) -> ReLU (+ skip)."""
    cin, cout = kernel.shape[1], kernel.shape[2]
    dev = x.device
    raw = torch.empty(lout.max_rows, cout, dtype=_f32, device=dev)
    stats = torch.empty(2 * cout, dtype=torch.float64, device=dev)
    L.call("o2345_sp_conv", _f(x), _p(lin.index, _i32), lin.E, _p(lout.rows, _i32), _p(lout.count, _i32),
           lout.max_rows, lout.E, mode, _f(kernel), cin, cout, _f(raw), _p(stats, torch.float64), _stream())
    L.call("o2345_sp_bn_relu", _f(raw), _p(lout.count, _i32), lout.max_rows, cout, _p(stats, torch.float64),
           _f(gamma), _f(beta), float(eps), _f(skip), _f(raw), _stream())
    return raw


# ----------------------------------------------------------------------------- marching cubes (B10)
_MC_CACHE = {}


def _mc_tables(dev):
    key = str(dev)
    if key not in _MC_CACHE:
        _, tri, ntri = mc_tables.tables()
        _MC_CACHE[key] = (torch.from_numpy(tri.copy()).to(dev), torch.from_numpy(ntri.copy()).to(dev),
                          torch.from_numpy(mc_tables.EDGE_OWNER.astype(np.int8)).to(dev).contiguous())
    return _MC_CACHE[key]


def marching_cubes(u, iso=0.0):
    """u float32 [R,R,R] (device) -> verts float64 [nv,3] (index units), tris int32 [nt,3], cases uint8."""
    R = u.shape[0]
    dev = u.device
    u = cf32(u)
    tri, ntri, owner = _mc_tables(dev)
    cases = torch.empty((R - 1) ** 3, dtype=_u8, device=dev)
    cell_flags = torch.empty((R - 1) ** 3, dtype=_u8, device=dev)
    edge_flags = torch.empty(3 * R ** 3, dtype=_u8, device=dev)
    L.call("o2345_mc_classify", _f(u), R, float(iso), _p(cases, _u8), _p(cell_flags, _u8), _p(edge_flags, _u8),
           _stream())
    edges, vert_index, nv_d = compact(edge_flags)
    cells, _, nc_d = compact(cell_flags)
    nv, nc = int(nv_d.item()), int(nc_d.item())  # the mesh size has to reach the host anyway
    verts = torch.empty(nv, 3, dtype=torch.float64, device=dev)
    L.call("o2345_mc_vertices", _f(u), R, float(iso), _p(edges, _i32), _p(nv_d, _i32), nv,
           _p(verts, torch.float64), _stream())
    if nc == 0:
        return verts, torch.empty(0, 3, dtype=_i32, device=dev), cases.view(R - 1, R - 1, R - 1)
    offs = torch.empty(nc, dtype=_i32, device=dev)
    total = torch.empty(1, dtype=_i32, device=dev)
    scratch = torch.empty(L.load().o2345_scan_scratch_ints(nc), dtype=_i32, device=dev)
    L.call("o2345_mc_tri_offsets", _p(cases, _u8), _p(cells, _i32), _p(nc_d, _i32), nc, _p(ntri, _u8),
           _p(offs, _i32), _p(total, _i32), _p(scratch, _i32), _stream())
    nt = int(total.item())
    tris = torch.empty(nt, 3, dtype=_i32, device=dev)
    L.call("o2345_mc_triangles", _p(cases, _u8), R, _p(cells, _i32), _p(nc_d, _i32), nc, _p(offs, _i32),
           _p(tri, torch.int8), _p(ntri, _u8), _p(owner, torch.int8), _p(vert_index, _i32), _p(tris, _i32),
           _stream())
    return verts, tris, cases.view(R - 1, R - 1, R - 1)


# ----------------------------------------------------------------------------- FeatureNet (B1/B2)
def view_of(t, layout, c0=0):
    """View4 over tensor t laid out as 'nchw' or 'nhwc' (channel offset c0 for concatenation)."""
    if layout == "nchw":
        N, Cc, H, W = t.shape
        v = L.View4(ptr=t.data_ptr(), sn=Cc * H * W, sc=H * W, sh=W, sw=1, c0=c0)
    else:
        N, H, W, Cc = t.shape
        v = L.View4(ptr=t.data_ptr(), sn=H * W * Cc, sc=1, sh=W * Cc, sw=Cc, c0=c0)
    return v


def conv2d(x, weight, bias, stride, pad, want_stats):
    N, Cin, H, W = x.shape
    Cout, _, K, _ = weight.shape
    Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
    out = torch.empty(N, Cout, Ho, Wo, dtype=_f32, device=x.device)
    stats = torch.empty(2 * Cout, dtype=torch.float64, device=x.device) if want_stats else None
    L.call("o2345_conv2d", _f(x), N, Cin, H, W, _f(weight), _f(bias), Cout, K, stride, pad, _f(out),
           _p(stats, torch.float64), _stream())
    return out, stats


def abn_apply(x, stats, gamma, beta, out_view, eps=1e-5, slope=0.01):
    N, Cc, H, W = x.shape
    L.call("o2345_abn_apply", _f(x), N, Cc, H, W, _p(stats, torch.float64), _f(gamma), _f(beta), float(eps),
           float(slope), C.byref(out_view), _stream())


def upsample_bilinear(x, factor, out_view, add=None):
    N, Cc, H, W = x.shape
    L.call("o2345_upsample_bilinear", _f(x), N, Cc, H, W, int(factor), _f(add), C.byref(out_view), _stream())


# ----------------------------------------------------------------------------- rendering (B11-B14)
def ray_upsample(rays_o, rays_d, z, sdf, inv_s, occ, u):
    R, S = z.shape
    n_new = u.numel()
    new_z = torch.empty(R, n_new, dtype=_f32, device=z.device)
    L.call("o2345_ray_upsample", _f(rays_o), _f(rays_d), R, _f(z), _f(sdf), S, float(inv_s), _f(occ),
           occ.shape[-1], _f(u), n_new, _f(new_z), _stream())
    return new_z


def ray_merge(z, sdf, new_z, new_sdf):
    R, S = z.shape
    n_new = new_z.shape[1]
    oz = torch.empty(R, S + n_new, dtype=_f32, device=z.device)
    osdf = torch.empty_like(oz)
    L.call("o2345_ray_merge", _f(z), _f(sdf), S, _f(new_z), _f(new_sdf), n_new, R, _f(oz), _f(osdf), _stream())
    return oz, osdf


def ray_midpoints(rays_o, rays_d, z, sample_dist, occ):
    """sample_dist: the last section length of every ray (a number), or a CUDA fp32 tensor [R] with one per ray."""
    R, S = z.shape
    mid = torch.empty_like(z)
    dists = torch.empty_like(z)
    active = torch.empty(R * S, dtype=_u8, device=z.device)
    if torch.is_tensor(sample_dist):
        if sample_dist.numel() != R:
            raise L.O2345Error(f"per-ray sample_dist has {sample_dist.numel()} values for {R} rays")
        L.call("o2345_ray_midpoints_per_ray", _f(rays_o), _f(rays_d), R, _f(z), S, _f(sample_dist), _f(occ), occ.shape[-1],
               _f(mid), _f(dists), _p(active, _u8), _stream())
    else:
        L.call("o2345_ray_midpoints", _f(rays_o), _f(rays_d), R, _f(z), S, float(sample_dist), _f(occ), occ.shape[-1],
               _f(mid), _f(dists), _p(active, _u8), _stream())
    return mid, dists, active


class SourceViews:
    """Channel-last colour+feature maps and camera data of the source views (o2345_views)."""

    def __init__(self, maps_nhwc, proj34, centers, sizeW, sizeH):
        V, H, W, c = maps_nhwc.shape
        assert c == L.MAP_CH
        self.maps, self.proj, self.centers = maps_nhwc, cf32(proj34), cf32(centers)
        self.struct = L.Views(V=V, H=H, W=W, maps=self.maps.data_ptr(), proj=self.proj.data_ptr(),
                              centers=self.centers.data_ptr(), sizeW=float(sizeW), sizeH=float(sizeH))


def render_blend(src: PointSource, active, vol_cl, occ, views: SourceViews, rnet_pack, query_center=None, dirs=None,
                 precision=L.BLEND_TC_FP16, ray_origins=False):
    """Target direction: towards query_center, along dirs, or (ray_origins=True, ray points only) towards each sample's own
    ray origin, for rays of several cameras in one call.
    precision: L.BLEND_TC_FP16 (mma.sync MLPs, fp16 operands / fp32 accumulate; the default) or L.BLEND_FP32 (fp32 FMA, the
    reference the parity tests compare against).  Any other value is refused."""
    n, dev = src.n, vol_cl.device
    rgb = torch.empty(n, 3, dtype=_f32, device=dev)
    nvalid = torch.empty(n, dtype=_i32, device=dev)
    mode = 2 if ray_origins else 0 if dirs is None else 1
    L.call("o2345_render_blend", C.byref(src.struct), n, _p(active, _u8), _f(vol_cl), _f(occ), vol_cl.shape[0],
           C.byref(views.struct), mode, _f(query_center), _f(dirs), _f(rnet_pack), int(precision), _f(rgb), _p(nvalid, _i32),
           _stream())
    return rgb, nvalid


def ray_composite(rays_d, mid, dists, sdf, grad, color, active, nvalid, inv_s, ratio, background):
    R, S = mid.shape
    dev = mid.device
    out = {"color": torch.empty(R, 3, dtype=_f32, device=dev), "depth": torch.empty(R, 1, dtype=_f32, device=dev),
           "weights": torch.empty(R, S, dtype=_f32, device=dev), "cdf": torch.empty(R, S, dtype=_f32, device=dev),
           "alpha": torch.empty(R, S, dtype=_f32, device=dev),
           "weights_sum": torch.empty(R, 1, dtype=_f32, device=dev),
           "color_mask": torch.empty(R, 1, dtype=_u8, device=dev)}
    has_bg = background is not None
    L.call("o2345_ray_composite", _f(rays_d), R, S, _f(mid), _f(dists), _f(sdf), _f(grad), _f(color),
           _p(active, _u8), _p(nvalid, _i32), float(inv_s), float(ratio), int(has_bg),
           float(background if has_bg else 0.0), _f(out["color"]), _f(out["depth"]), _f(out["weights"]),
           _f(out["cdf"]), _f(out["alpha"]), _f(out["weights_sum"]), _p(out["color_mask"], _u8), _stream())
    return out


# ----------------------------------------------------------------------------- mesh rasterizer
def raster(verts, faces, w2c, intr, W, H, near=0.1, shading=L.SHADE_UNLIT, colors=None, uvs=None, face_tex=None, texels=None,
           tex_info=None, normals=None, tangents=None, face_ntex=None):
    """V views of one triangle mesh (csrc/raster.cu): verts [nv,3] world, faces [nf,3] int32, w2c [V,3,4] OpenCV, intr
    [V,4] = (fx, fy, cx, cy); optional colors [nv,3], uvs [nv,2] with face_tex [nf] int32, texels RGBA8 uint8 and tex_info
    [n_tex,5] int32; optional normal maps: normals [nv,3], tangents [nv,4] and face_ntex [nf] int32 (textures of the same
    pool).  Returns device tensors color [V,H,W,3], alpha [V,H,W], depth [V,H,W], normal [V,H,W,3], tri [V,H,W] int32 (-1
    background)."""
    verts, w2c, intr = cf32(verts).view(-1, 3), cf32(w2c).view(-1, 3, 4), cf32(intr).view(-1, 4)
    faces = faces.contiguous().view(-1, 3)
    V, nv, nf, dev = w2c.shape[0], verts.shape[0], faces.shape[0], verts.device
    if intr.shape[0] != V:
        raise ValueError(f"{V} w2c matrices but {intr.shape[0]} intrinsics")
    colors = None if colors is None else cf32(colors).view(-1, 3)
    uvs = None if uvs is None else cf32(uvs).view(-1, 2)
    normals = None if normals is None else cf32(normals).view(-1, 3)
    tangents = None if tangents is None else cf32(tangents).view(-1, 4)
    for name, t, rows in (("colors", colors, nv), ("uvs", uvs, nv), ("face_tex", face_tex, nf), ("normals", normals, nv),
                          ("tangents", tangents, nv), ("face_ntex", face_ntex, nf)):
        if t is not None and t.shape[0] != rows:
            raise ValueError(f"{name} has {t.shape[0]} rows, expected {rows}")
    mesh = L.RasterMesh(verts=_f(verts).value, colors=_f(colors).value if colors is not None else None,
                        uvs=_f(uvs).value if uvs is not None else None, faces=_p(faces, _i32).value,
                        face_tex=_p(face_tex, _i32).value if face_tex is not None else None,
                        texels=_p(texels, _u8).value if texels is not None else None,
                        tex_info=_p(tex_info, _i32).value if tex_info is not None else None,
                        normals=_f(normals).value if normals is not None else None,
                        tangents=_f(tangents).value if tangents is not None else None,
                        face_ntex=_p(face_ntex, _i32).value if face_ntex is not None else None,
                        nv=nv, nf=nf, n_tex=0 if tex_info is None else tex_info.shape[0])
    nbytes = L.load().o2345_raster_scratch_bytes(nv, nf, V, W, H)
    scratch = torch.empty(nbytes, dtype=_u8, device=dev)
    out = {"color": torch.empty(V, H, W, 3, dtype=_f32, device=dev), "alpha": torch.empty(V, H, W, dtype=_f32, device=dev),
           "depth": torch.empty(V, H, W, dtype=_f32, device=dev), "normal": torch.empty(V, H, W, 3, dtype=_f32, device=dev),
           "tri": torch.empty(V, H, W, dtype=_i32, device=dev)}
    L.call("o2345_raster", C.byref(mesh), V, _f(w2c), _f(intr), int(W), int(H), float(near), int(shading), _p(scratch), nbytes,
           _f(out["color"]), _f(out["alpha"]), _f(out["depth"]), _f(out["normal"]), _p(out["tri"], _i32), _stream())
    return out


# ----------------------------------------------------------------------------- mesh scoring
def surface_sample(verts, faces, n, seed=0):
    """n points drawn area-uniformly on a triangle mesh (csrc/metrics.cu): verts [nv,3] fp32, faces [nf,3] int32 (faces with
    an index outside [0, nv) and zero-area faces get no samples) -> pts [n,3] fp32, face_id [n] int32.  Deterministic in
    (mesh, n, seed).  Synchronises once; raises O2345Error when the faces have no area."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    n, seed = int(n), int(seed) & (2 ** 64 - 1)
    nbytes = L.load().o2345_surface_sample_scratch_bytes(nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    pts = torch.empty(max(n, 0), 3, dtype=_f32, device=dev)
    face_id = torch.empty(max(n, 0), dtype=_i32, device=dev)
    L.call("o2345_surface_sample", _f(verts), nv, _p(faces, _i32), nf, n, seed, _p(scratch), nbytes, _f(pts), _p(face_id, _i32),
           _stream())
    return pts, face_id


def nearest(query, ref):
    """Exact nearest neighbour of every query point among the reference points (csrc/metrics.cu): query [nq,3], ref [nr,3]
    fp32 -> dist2 [nq] fp32 ((dx*dx + dy*dy) + dz*dz, rounded as written), index [nq] int32 (ties: the lower index)."""
    query, ref = cf32(query).view(-1, 3), cf32(ref).view(-1, 3)
    nq, nr, dev = query.shape[0], ref.shape[0], query.device
    nbytes = L.load().o2345_nn_scratch_bytes(nr, nq)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    dist2 = torch.empty(nq, dtype=_f32, device=dev)
    index = torch.empty(nq, dtype=_i32, device=dev)
    L.call("o2345_nearest", _f(ref), nr, _f(query), nq, _p(scratch), nbytes, _f(dist2), _p(index, _i32), _stream())
    return dist2, index


# ----------------------------------------------------------------------------- mesh simplification
def simplify_mesh(verts, faces, target_faces):
    """Quadric-driven half-edge collapse down to target_faces or target_faces - 1 faces (csrc/simplify.cu): verts [nv,3]
    fp32, faces [nf,3] int32 -> vertex_index [nv'] int32 (the input indices of the kept vertices, ascending; every output
    vertex is an input vertex), faces [nf',3] int32 renumbered into vertex_index, in ascending input order, and the number
    of rounds.  Fewer faces than asked for are left only when no legal collapse remains.  Deterministic.  Synchronises
    once per round; raises O2345Error for an index outside [0, nv) or a non-finite coordinate."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    nbytes = L.load().o2345_simplify_scratch_bytes(nv, nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    vertex_index = torch.empty(max(nv, 1), dtype=_i32, device=dev)
    out = torch.empty(max(nf, 1), 3, dtype=_i32, device=dev)
    counts = torch.empty(3, dtype=_i32, device=dev)
    L.call("o2345_simplify", _f(verts), nv, _p(faces, _i32), nf, int(target_faces), _p(scratch), nbytes, _p(vertex_index, _i32),
           _p(out, _i32), _p(counts, _i32), _stream())
    n_v, n_f, rounds = counts.tolist()
    return vertex_index[:n_v], out[:n_f], rounds


# ----------------------------------------------------------------------------- texture baking
def texture_atlas(verts, faces, N):
    """One isometric chart per face packed into an N x N atlas (csrc/texture.cu): verts [nv,3] fp32, faces [nf,3] int32
    -> dict(uv [nf,3,2] fp32 (row k for corner k, glTF convention: texel i's centre at (i + 0.5) / N), boxes [nf,4] int32
    (x, y, w, hgt), owner [N*N] int32 (-1 where no box is), j (the ladder rung), rho (texels per unit length)).
    Synchronises about 9 times; raises O2345Error for bad input or charts that do not fit."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    nbytes = L.load().o2345_texture_atlas_scratch_bytes(nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    uv = torch.empty(max(nf, 1), 3, 2, dtype=_f32, device=dev)
    boxes = torch.empty(max(nf, 1), 4, dtype=_i32, device=dev)
    owner = torch.empty(int(N) * int(N), dtype=_i32, device=dev)
    j, rho = C.c_int32(0), C.c_double(0.0)
    L.call("o2345_texture_atlas", _f(verts), nv, _p(faces, _i32), nf, int(N), _p(scratch), nbytes, _f(uv), _p(boxes, _i32),
           _p(owner, _i32), C.byref(j), C.byref(rho), _stream())
    return {"uv": uv[:nf], "boxes": boxes[:nf], "owner": owner, "j": j.value, "rho": rho.value}


def chart_atlas(verts, faces, N):
    """Multi-face charts packed into an N x N atlas (csrc/texture.cu; the rules are in include/o2345.h): faces with the
    same dominant normal axis and sign, joined across edges of two faces, projected along that axis and cut at their
    median until no chart overlaps itself.  -> the dict of texture_atlas (boxes: each face's chart box) plus label [nf]
    int32, chart [nf] int32 (the chart's least face), rounds (cut rounds) and charts (chart count).  Synchronises per
    component pass, per round and per trial; raises O2345Error for bad input or charts that do not fit."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    nbytes = L.load().o2345_chart_atlas_scratch_bytes(nv, nf, int(N))
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    uv = torch.empty(max(nf, 1), 3, 2, dtype=_f32, device=dev)
    boxes = torch.empty(max(nf, 1), 4, dtype=_i32, device=dev)
    owner = torch.empty(int(N) * int(N), dtype=_i32, device=dev)
    label = torch.empty(max(nf, 1), dtype=_i32, device=dev)
    chart = torch.empty(max(nf, 1), dtype=_i32, device=dev)
    j, rho, rounds, charts = C.c_int32(0), C.c_double(0.0), C.c_int32(0), C.c_int32(0)
    L.call("o2345_chart_atlas", _f(verts), nv, _p(faces, _i32), nf, int(N), _p(scratch), nbytes, _f(uv), _p(boxes, _i32),
           _p(owner, _i32), _p(label, _i32), _p(chart, _i32), C.byref(j), C.byref(rho), C.byref(rounds), C.byref(charts),
           _stream())
    return {"uv": uv[:nf], "boxes": boxes[:nf], "owner": owner, "j": j.value, "rho": rho.value, "label": label[:nf],
            "chart": chart[:nf], "rounds": rounds.value, "charts": charts.value}


def texel_points(verts, faces, uv, owner, N):
    """The owned texels of an atlas (texture_atlas) and the surface points behind them: -> texel_index [T] int32
    (ascending), points [T,3] fp32, texel_face [T] int32.  Reads T on the host."""
    verts, faces, uv = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3), cf32(uv).view(-1, 3, 2)
    nv, nf, dev, n = verts.shape[0], faces.shape[0], verts.device, int(N) * int(N)
    nbytes = L.load().o2345_texel_points_scratch_bytes(int(N))
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    index = torch.empty(n, dtype=_i32, device=dev)
    points = torch.empty(n, 3, dtype=_f32, device=dev)
    face = torch.empty(n, dtype=_i32, device=dev)
    count = torch.empty(1, dtype=_i32, device=dev)
    L.call("o2345_texel_points", _f(verts), nv, _p(faces, _i32), nf, _f(uv), _p(owner.contiguous(), _i32), int(N), _p(scratch),
           nbytes, _p(index, _i32), _f(points), _p(face, _i32), _p(count, _i32), _stream())
    T = int(count.item())
    return index[:T], points[:T], face[:T]


def texture_fill(texel_index, rgb, owner, N):
    """texture [N,N,3] fp32: rgb [T,3] at texel_index [T] and push-pull fill of every texel with owner < 0."""
    rgb, dev = cf32(rgb).view(-1, 3), owner.device
    if rgb.shape[0] != texel_index.shape[0]:
        raise ValueError(f"{rgb.shape[0]} colours for {texel_index.shape[0]} texels")
    count = torch.tensor([texel_index.shape[0]], dtype=_i32, device=dev)
    nbytes = L.load().o2345_texture_fill_scratch_bytes(int(N))
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    tex = torch.empty(int(N), int(N), 3, dtype=_f32, device=dev)
    L.call("o2345_texture_fill", _p(texel_index.contiguous(), _i32), _p(count, _i32), _f(rgb), _p(owner.contiguous(), _i32),
           int(N), _p(scratch), nbytes, _f(tex), _stream())
    return tex


def transfer_colors(verts, faces, colors, points, nn_index, sample_face):
    """Colours [n,3] fp32 of a source mesh (verts [nv,3], faces [nf,3], colors [nv,3] fp32) at points [n,3]: each point is
    projected onto the face of its nearest surface sample (nn_index [n] into sample_face [m]) and the face's vertex
    colours are interpolated there."""
    verts, faces, colors = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3), cf32(colors).view(-1, 3)
    points = cf32(points).view(-1, 3)
    n, dev = points.shape[0], points.device
    rgb = torch.empty(n, 3, dtype=_f32, device=dev)
    if n == 0:
        return rgb
    L.call("o2345_transfer_colors", _f(verts), verts.shape[0], _p(faces, _i32), faces.shape[0], _f(colors), _f(points), n,
           _p(nn_index.contiguous(), _i32), _p(sample_face.contiguous(), _i32), sample_face.shape[0], _f(rgb), _stream())
    return rgb


# ----------------------------------------------------------------------------- normal maps
def tangent_normals(verts, faces, uv, texel_face, normals):
    """World normals [T,3] at texels of faces texel_face [T] int32 -> their tangent-space unit vectors [T,3] fp32 in each
    face's frame from its corners and atlas uv [nf,3,2] (csrc/texture.cu; the rule is in include/o2345.h).  Degenerate
    faces and zero or non-finite normals give (0, 0, 1)."""
    verts, faces, uv = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3), cf32(uv).view(-1, 3, 2)
    normals = cf32(normals).view(-1, 3)
    n, dev = normals.shape[0], normals.device
    if texel_face.shape[0] != n:
        raise ValueError(f"{n} normals for {texel_face.shape[0]} texels")
    out = torch.empty(n, 3, dtype=_f32, device=dev)
    if n == 0:
        return out
    L.call("o2345_tangent_normals", _f(verts), verts.shape[0], _p(faces, _i32), faces.shape[0], _f(uv),
           _p(texel_face.contiguous(), _i32), _f(normals), n, _f(out), _stream())
    return out


def tangent_normals_decoded(verts, faces, uv, texel_face, normals):
    """As tangent_normals, in the frame decoders build from NORMAL and TANGENT: B = w (N x T), w = sign((N x T) . -dp/dv)
    (for chart_atlas, whose dp/du and dp/dv are not orthogonal)."""
    verts, faces, uv = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3), cf32(uv).view(-1, 3, 2)
    normals = cf32(normals).view(-1, 3)
    n, dev = normals.shape[0], normals.device
    if texel_face.shape[0] != n:
        raise ValueError(f"{n} normals for {texel_face.shape[0]} texels")
    out = torch.empty(n, 3, dtype=_f32, device=dev)
    if n == 0:
        return out
    L.call("o2345_tangent_normals_decoded", _f(verts), verts.shape[0], _p(faces, _i32), faces.shape[0], _f(uv),
           _p(texel_face.contiguous(), _i32), _f(normals), n, _f(out), _stream())
    return out


def normal_quantise(texture):
    """Tangent-space texture [N,N,3] fp32 (texture_fill) -> uint8 [N,N,3]: renormalised in fp32, each component coded as
    round_half_even((c + 1) * 127.5); an empty vector becomes (128, 128, 255)."""
    texture = cf32(texture)
    out = torch.empty(texture.shape, dtype=_u8, device=texture.device)
    L.call("o2345_normal_quantise", _f(texture), texture.numel() // 3, _p(out, _u8), _stream())
    return out


def vertex_normals(verts, faces):
    """Unit vertex normals [nv,3] fp32 of verts [nv,3], faces [nf,3] int32: each vertex's sum of its faces'
    (B - A) x (C - A) in ascending face order in fp64, normalised and rounded once ((0, 0, 0) for a zero sum).
    Synchronises once; raises O2345Error for an index outside [0, nv) or a non-finite coordinate."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    nbytes = L.load().o2345_vertex_normals_scratch_bytes(nv, nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    out = torch.empty(nv, 3, dtype=_f32, device=dev)
    L.call("o2345_vertex_normals", _f(verts), nv, _p(faces, _i32), nf, _p(scratch), nbytes, _f(out), _stream())
    return out


# ----------------------------------------------------------------------------- input-view projection
def face_normals(verts, faces, face_index):
    """Unit normals [n,3] fp32 of faces face_index [n] int32 of verts [nv,3], faces [nf,3] (csrc/project.cu): (B - A) x
    (C - A) in fp64, normalised and rounded once; (0, 0, 0) for an index out of range or a face without area."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    n, dev = face_index.shape[0], verts.device
    out = torch.empty(n, 3, dtype=_f32, device=dev)
    if n == 0:
        return out
    L.call("o2345_face_normals", _f(verts), verts.shape[0], _p(faces, _i32), faces.shape[0], _p(face_index.contiguous(), _i32),
           n, _f(out), _stream())
    return out


def project_view(points, normals, base, w2c, intr, photo, alpha, depth, near=0.1):
    """The input photo blended into base colours (csrc/project.cu; the rule is in include/o2345.h): points [T,3], normals
    [T,3] (any length; zero or non-finite: not seen), base [T,3] fp32; w2c [3,4] (OpenCV) and intr (fx, fy, cx, cy) of
    the photo's camera; photo uint8 [H,W,3], alpha uint8 [H,W] or None; depth [s H, s W] fp32: the mesh's depth from
    raster with (s fx, s fy, s (cx + 0.5), s (cy + 0.5)), s an integer >= 1.  -> (colours [T,3], weight [T]) fp32."""
    points, normals, base = cf32(points).view(-1, 3), cf32(normals).view(-1, 3), cf32(base).view(-1, 3)
    w2c, depth = cf32(w2c).view(3, 4), cf32(depth)
    T, dev = points.shape[0], points.device
    H, W = photo.shape[0], photo.shape[1]
    if photo.shape != (H, W, 3) or (alpha is not None and alpha.shape != (H, W)):
        raise ValueError(f"photo must be [H,W,3] and alpha [H,W], got {tuple(photo.shape)} and "
                         f"{None if alpha is None else tuple(alpha.shape)}")
    s = depth.shape[1] // W
    if depth.dim() != 2 or s < 1 or depth.shape[1] != s * W or depth.shape[0] != s * H:
        raise ValueError(f"depth {tuple(depth.shape)} is not an integer multiple of the photo's {H} x {W}")
    if normals.shape[0] != T or base.shape[0] != T:
        raise ValueError(f"{T} points, {normals.shape[0]} normals and {base.shape[0]} colours")
    out = torch.empty(T, 3, dtype=_f32, device=dev)
    weight = torch.empty(T, dtype=_f32, device=dev)
    if T == 0:
        return out, weight
    fx, fy, cx, cy = (float(v) for v in intr)
    L.call("o2345_project_view", _f(points), _f(normals), _f(base), T, _f(w2c), fx, fy, cx, cy, float(near),
           _p(photo.contiguous(), _u8), None if alpha is None else _p(alpha.contiguous(), _u8), W, H, _f(depth), s, _f(out),
           _f(weight), _stream())
    return out, weight


# ----------------------------------------------------------------------------- mesh cleaning
def clean_mesh(verts, faces, min_component):
    """Drops the components that are small next to the largest one or enclosed by it (csrc/clean.cu; the rules are in
    include/o2345.h): verts [nv,3] fp32, faces [nf,3] int32 (welded: faces sharing a vertex index form one component),
    0 < min_component <= 1 -> (vertex_index [nv'] int32, the input indices of the kept vertices (those a kept face
    references), ascending; faces [nf',3] int32, the kept faces in input order renumbered into vertex_index; stats).
    stats: components, largest, dropped (components), dropped_faces, enclosed (components) as ints, and the tensors
    label [nf] int32 (each face's component, numbered by least face), area [nc] fp64, winding [nc] fp64 (0 at the largest)
    and keep [nc] uint8.  Deterministic.  Synchronises once per union-find pass and three more times; raises O2345Error
    for min_component outside (0, 1], an index outside [0, nv) or a non-finite coordinate."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    if not 0.0 < float(min_component) <= 1.0:
        raise L.O2345Error(f"min_component must lie in (0, 1], got {min_component}")
    if nf == 0:                      # no face: no component, and every vertex is unreferenced
        empty = torch.empty(0, dtype=_i32, device=dev)
        return empty, torch.empty(0, 3, dtype=_i32, device=dev), {
            "components": 0, "largest": -1, "dropped": 0, "dropped_faces": 0, "enclosed": 0, "label": empty,
            "area": torch.empty(0, dtype=torch.float64, device=dev), "winding": torch.empty(0, dtype=torch.float64, device=dev),
            "keep": torch.empty(0, dtype=_u8, device=dev)}
    nbytes = L.load().o2345_clean_mesh_scratch_bytes(nv, nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    label = torch.empty(nf, dtype=_i32, device=dev)
    area = torch.empty(nf, dtype=torch.float64, device=dev)
    winding = torch.empty(nf, dtype=torch.float64, device=dev)
    keep = torch.empty(nf, dtype=_u8, device=dev)
    vertex_index = torch.empty(max(nv, 1), dtype=_i32, device=dev)
    out = torch.empty(nf, 3, dtype=_i32, device=dev)
    counts = (C.c_int32 * 6)()
    L.call("o2345_clean_mesh", _f(verts), nv, _p(faces, _i32), nf, float(min_component), _p(scratch), nbytes,
           _p(label, _i32), _p(area, torch.float64), _p(winding, torch.float64), _p(keep, _u8), _p(vertex_index, _i32),
           _p(out, _i32), counts, _stream())
    nc, largest, kept, enclosed, n_v, n_f = list(counts)
    stats = {"components": nc, "largest": largest, "dropped": nc - kept, "dropped_faces": nf - n_f, "enclosed": enclosed,
             "label": label, "area": area[:nc], "winding": winding[:nc], "keep": keep[:nc]}
    return vertex_index[:n_v], out[:n_f], stats


# ----------------------------------------------------------------------------- ambient occlusion
def ambient_occlusion(verts, faces, points, normals):
    """AO [n] fp32 of points [n,3] with normals [n,3] (any length; zero or non-finite: 1) against the mesh verts [nv,3],
    faces [nf,3] int32 (csrc/ao.cu; the rule is in include/o2345.h): the share of the mesh_texture.AO_RAYS directions of
    mesh_texture.ao_directions, turned into each normal's frame, whose segment [t_min, t_max] (mesh_texture.ao_distances)
    hits no face.  Deterministic.  Synchronises once; raises O2345Error for an index outside [0, nv) or a non-finite
    coordinate."""
    from .mesh_texture import ao_directions, ao_distances
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    points, normals = cf32(points).view(-1, 3), cf32(normals).view(-1, 3)
    nv, nf, n, dev = verts.shape[0], faces.shape[0], points.shape[0], points.device
    if normals.shape[0] != n:
        raise ValueError(f"{n} points and {normals.shape[0]} normals")
    dirs = torch.from_numpy(ao_directions()).to(dev)
    t_min, t_max = ao_distances(verts.cpu().numpy())
    nbytes = L.load().o2345_ambient_occlusion_scratch_bytes(nv, nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    out = torch.empty(n, dtype=_f32, device=dev)
    L.call("o2345_ambient_occlusion", _f(verts), nv, _p(faces, _i32), nf, _f(points), _f(normals), n, _f(dirs), dirs.shape[0],
           float(t_min), float(t_max), _p(scratch), nbytes, _f(out), _stream())
    return out


# ----------------------------------------------------------------------------- remeshing
def closest_points(verts, faces, points):
    """Closest points of points [n,3] on the mesh verts [nv,3] fp32, faces [nf,3] int32 (csrc/remesh.cu; the rule is in
    include/o2345.h): per point the least (squared distance, face index) of the 7-region closest point over all faces in
    fp64, searched through an LBVH and equal to the search over all faces bit for bit -> (points [n,3] fp32, face [n]
    int32); NaN and -1 for a non-finite point or no faces.  Synchronises once; raises O2345Error for an index outside
    [0, nv) or a non-finite vertex."""
    verts, faces, points = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3), cf32(points).view(-1, 3)
    nv, nf, n, dev = verts.shape[0], faces.shape[0], points.shape[0], points.device
    nbytes = L.load().o2345_closest_points_scratch_bytes(nv, nf)
    scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
    out = torch.empty(n, 3, dtype=_f32, device=dev)
    face = torch.empty(n, dtype=_i32, device=dev)
    L.call("o2345_closest_points", _f(verts), nv, _p(faces, _i32), nf, _f(points), n, _p(scratch), nbytes, _f(out),
           _p(face, _i32), _stream())
    return out, face


def remesh_mesh(verts, faces, target_length, iterations, vertex_capacity=None, face_capacity=None):
    """Isotropic remesh of verts [nv,3] fp32, faces [nf,3] int32 (nf >= 1) at target edge length target_length (fp32)
    for `iterations` iterations of split, collapse, flip, tangential relaxation and projection onto the input (csrc/
    remesh.cu; the rules are in include/o2345.h) -> (verts [nv',3] fp32, faces [nf',3] int32, (split, collapse, flip
    rounds)).  The buffers start at the given capacities (default: twice the input, at least 1024) and are regrown to
    what a run reports it needs (O2345_ENOSPC) until it fits; the result does not depend on them.  Deterministic.
    Synchronises once per round; raises O2345Error for an index outside [0, nv) or a non-finite coordinate."""
    verts, faces = cf32(verts).view(-1, 3), faces.contiguous().view(-1, 3)
    nv, nf, dev = verts.shape[0], faces.shape[0], verts.device
    vcap = max(nv, int(vertex_capacity) if vertex_capacity is not None else max(2 * nv, 1024))
    fcap = max(nf, int(face_capacity) if face_capacity is not None else max(2 * nf, 1024))
    lib = L.load()
    counts = (C.c_int64 * 5)()
    while True:
        nbytes = lib.o2345_remesh_scratch_bytes(nv, nf, vcap, fcap)
        if nbytes < 0:
            raise L.O2345Error(f"o2345_remesh_scratch_bytes: sizes out of range (nv {nv}, nf {nf}, capacities {vcap}, {fcap})")
        scratch = torch.empty(max(nbytes, 1), dtype=_u8, device=dev)
        out_v = torch.empty(vcap, 3, dtype=_f32, device=dev)
        out_f = torch.empty(fcap, 3, dtype=_i32, device=dev)
        rc = lib.o2345_remesh(_f(verts), nv, _p(faces, _i32), nf, float(target_length), int(iterations), vcap, fcap,
                              _p(scratch), nbytes, _f(out_v), _p(out_f, _i32), counts, _stream())
        if rc == L.ENOSPC:
            vcap, fcap = max(int(counts[0]), 2 * vcap), max(int(counts[1]), 2 * fcap)
            del scratch, out_v, out_f
            continue
        if rc != 0:
            raise L.O2345Error(f"o2345_remesh failed with {rc}: {L.last_error()}")
        L.add_launches(1)
        return out_v[:counts[0]], out_f[:counts[1]], (int(counts[2]), int(counts[3]), int(counts[4]))
