"""Texture baking on host arrays (run.py / simplify_mesh.py --texture_size, GenericTrainer.export_mesh_step): every face
gets its own chart in an N x N atlas (ops.texture_atlas; or, with atlas="charts", faces share projected multi-face charts:
ops.chart_atlas), the surface point behind every texel a chart owns is evaluated
by a colour function (ops.texel_points), and the texels no chart owns are filled by push-pull (ops.texture_fill), all in
csrc/texture.cu.  The colour function is the reconstruction's (SparseNeuSRenderer.blend_points, the one that colours the
vertices) or, for a mesh without a reconstruction, the colours of a source mesh (transfer_fn).

A normal map shares the atlas and the texel points: a normal function gives the world normal at every texel's point (the
SDF gradient, or a source mesh's interpolated vertex normals: normal_transfer_fn), ops.tangent_normals codes it in the
face's tangent frame (the rule of include/o2345.h, which mesh_io's writers and the rasterizer decode), the same push-pull
fills the rest and ops.normal_quantise codes it to uint8.

The input photo can be projected onto the mesh (view=, prepare_view, project_vertex_colors): ops.raster renders the
mesh's depth from the photo's camera once, and ops.project_view blends the photo into the colours of every vertex
(ops.vertex_normals) and texel (ops.face_normals of its face) that camera sees squarely.

An occlusion map (ao_fn=, vertex_ao, ao_transfer_fn) shares the atlas too: ops.ambient_occlusion gives the AO of every
vertex of the full mesh, the texels take it interpolated on the face of their nearest source sample (as transfer_fn does
colours), and the same push-pull fills the rest.  The glTF occlusionTexture reads it."""
from __future__ import annotations

import numpy as np
import torch

from . import ops

MIN_SIZE, MAX_SIZE = 64, 8192
ATLASES = ("faces", "charts")  # ops.texture_atlas (the default) and ops.chart_atlas
TRANSFER_SEED = 0          # seed of the source surface samples of transfer_fn
TRANSFER_SAMPLES = 4       # source samples per texel of the atlas
DEPTH_SCALE = 4            # depth-buffer pixels per photo pixel and side (a 256^2 photo: 1024^2) ...
DEPTH_MAX = 4096           # ... at most this many per side
NEAR = 0.1                 # near plane of the depth buffer and of the projection
AO_RAYS = 256              # ambient occlusion: directions per point (steps of 1/256, below one 8-bit code) ...
AO_T_MIN = 1e-3            # ... on segments from AO_T_MIN to AO_T_MAX times the diagonal of the occluder's box;
AO_T_MAX = 0.1             # AO_T_MIN drops the hits at t = 0 on the faces around the vertex a ray starts from


def check_size(texture_size):
    """Raises ValueError unless texture_size is a power of two in [64, 8192]."""
    n = int(texture_size)
    if n != texture_size or n < MIN_SIZE or n > MAX_SIZE or n & (n - 1):
        raise ValueError(f"texture_size must be a power of two in [{MIN_SIZE}, {MAX_SIZE}], got {texture_size}")
    return n


def _device(device):
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def quantise(rgb):
    """The vertex-colour rule of GenericTrainer.validate_colored_mesh: (rgb * 255).astype(uint8)."""
    return (rgb.cpu() * 255).numpy().astype(np.uint8)


def check_atlas(atlas):
    """Raises ValueError unless atlas is one of ATLASES."""
    if atlas not in ATLASES:
        raise ValueError(f"atlas must be one of {', '.join(ATLASES)}, got {atlas!r}")
    return atlas


def depth_scale(W, H):
    """Depth-buffer pixels per photo pixel (per side) for a W x H photo: DEPTH_SCALE, less where the buffer would exceed
    DEPTH_MAX on a side, at least 1."""
    return max(1, min(DEPTH_SCALE, DEPTH_MAX // max(int(W), int(H))))


def depth_intrinsics(intr, s):
    """(fx, fy, cx, cy) of the depth buffer at s buffer pixels per photo pixel.  The rasterizer samples pixel j at
    fx X / Z + cx = j + 0.5 and the photo puts pixel i's centre at i, so the buffer pixel under photo coordinate x is
    floor(s (x + 0.5)) and photo pixel i covers buffer pixels s i .. s i + s - 1."""
    fx, fy, cx, cy = (float(v) for v in intr)
    return (s * fx, s * fy, s * (cx + 0.5), s * (cy + 0.5))


def rescale_intrinsics(intr, from_wh, to_wh):
    """(fx, fy, cx, cy) of a camera whose W x H image (from_wh) is resized to to_wh, with pixel i's centre at i (the
    projector's convention; the image spans [-0.5, W - 0.5]): f' = f W' / W, c' = (c + 0.5) W' / W - 0.5 (y alike)."""
    fx, fy, cx, cy = (float(v) for v in intr)
    sx, sy = to_wh[0] / from_wh[0], to_wh[1] / from_wh[1]
    return (fx * sx, fy * sy, (cx + 0.5) * sx - 0.5, (cy + 0.5) * sy - 0.5)


def prepare_view(vt, ft, view):
    """view: dict(photo uint8 [H,W,3] composited on white, alpha uint8 [H,W] or None, w2c [3,4] or [4,4] (OpenCV),
    intr (fx, fy, cx, cy)) in the frame of the mesh vt [n,3] fp32, ft [m,3] int32 (device tensors).  Returns the view
    with its arrays on the mesh's device and the mesh's depth buffer from that camera (ops.raster at depth_scale
    pixels per photo pixel, depth_intrinsics); a view that already has its depth buffer is returned as it is, so one
    buffer serves the vertices and the texels of the same mesh."""
    if "depth" in view:
        return view
    dev = vt.device

    def as_dev(a, dt):
        return (a if torch.is_tensor(a) else torch.from_numpy(np.require(a, requirements="CW"))).to(dev, dt).contiguous()
    photo = as_dev(view["photo"], torch.uint8)
    alpha = None if view.get("alpha") is None else as_dev(view["alpha"], torch.uint8)
    w2c = as_dev(view["w2c"], torch.float32)[:3, :4].contiguous()
    intr = tuple(float(v) for v in view["intr"])
    H, W = photo.shape[:2]
    s = depth_scale(W, H)
    with torch.cuda.device(dev):
        depth = ops.raster(vt, ft, w2c[None], torch.tensor([depth_intrinsics(intr, s)], device=dev), s * W, s * H,
                           near=NEAR)["depth"][0]
    return {"photo": photo, "alpha": alpha, "w2c": w2c, "intr": intr, "depth": depth}


def project(points, normals, rgb, view):
    """ops.project_view of a prepared view (prepare_view) -> (colours [T,3], weight [T])."""
    return ops.project_view(points, normals, rgb, view["w2c"], view["intr"], view["photo"], view["alpha"], view["depth"],
                            near=NEAR)


def project_vertex_colors(vt, ft, rgb, view):
    """The photo of view (prepare_view's dict, or one it accepts) blended into vertex colours rgb [n,3] fp32 of the mesh
    vt, ft (device tensors) with its vertex normals (ops.vertex_normals) -> (colours [n,3], weight [n])."""
    view = prepare_view(vt, ft, view)
    with torch.cuda.device(vt.device):
        return project(vt, ops.vertex_normals(vt, ft), rgb, view)


def ao_directions(k=AO_RAYS):
    """The golden-angle spiral on the unit disk lifted to the hemisphere by Malley's method (cosine-distributed):
    d_i = (r cos phi, r sin phi, sqrt(1 - r^2)), r = sqrt((i + 1/2) / k), phi = i pi (3 - sqrt 5), in fp64 and rounded
    once -> float32 [k,3]."""
    i = np.arange(k, dtype=np.float64)
    r2 = (i + 0.5) / k
    r, phi = np.sqrt(r2), i * (np.pi * (3.0 - np.sqrt(5.0)))
    return np.stack([r * np.cos(phi), r * np.sin(phi), np.sqrt(1.0 - r2)], 1).astype(np.float32)


def ao_distances(verts):
    """(t_min, t_max) float32 of the occluder verts [n,3]: AO_T_MIN and AO_T_MAX times the diagonal of their box,
    sqrt((dx dx + dy dy) + dz dz) in fp64, each rounded once (0 without vertices)."""
    v = np.asarray(verts, np.float32).reshape(-1, 3)
    if len(v) == 0:
        return np.float32(0.0), np.float32(0.0)
    e = v.max(0).astype(np.float64) - v.min(0).astype(np.float64)
    d = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
    return np.float32(AO_T_MIN * d), np.float32(AO_T_MAX * d)


def vertex_ao(vt, ft):
    """AO [n] fp32 at the vertices of the mesh vt [n,3], ft [m,3] int32 (device tensors) against the mesh itself, with
    its vertex normals (ops.vertex_normals; a vertex without faces gets 1)."""
    with torch.cuda.device(vt.device):
        return ops.ambient_occlusion(vt, ft, vt, ops.vertex_normals(vt, ft))


def ao_transfer_fn(src_v, src_f, texture_size=None, device=None, seed=TRANSFER_SEED):
    """An ao_fn for bake from a source mesh src_v [n,3], src_f [m,3]: its vertex AO (vertex_ao, computed now),
    interpolated at each point's closest point on the face of its nearest source sample, with the same seeded samples
    and search as transfer_fn."""
    dev = _device(device)
    sv = torch.from_numpy(np.ascontiguousarray(src_v, np.float32).reshape(-1, 3)).to(dev)
    sf = torch.from_numpy(np.ascontiguousarray(src_f, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        fn = _transfer(sv, sf, vertex_ao(sv, sf)[:, None].expand(-1, 3).contiguous(), texture_size, seed)
    return lambda points: fn(points)[:, 0]


def ao_quantise(ao):
    """AO [N,N] fp32 -> uint8 [N,N]: round_half_even(ao * 255) in fp32."""
    return np.rint(ao.cpu().numpy().astype(np.float32) * np.float32(255)).clip(0, 255).astype(np.uint8)


def bake(vertices, faces, texture_size, colour_fn, device=None, return_atlas=False, normal_fn=None, atlas="faces",
         view=None, ao_fn=None):
    """vertices [n,3], faces [m,3] (numpy) -> (uv float32 [m,3,2], texture uint8 [N,N,3]); uv row k belongs to corner
    faces[f, k], in glTF's convention (v down the image, texel i's centre at (i + 0.5) / N).  colour_fn(points [T,3] fp32
    device tensor) -> rgb [T,3] in [0, 1] on the device, for the surface point behind every owned texel.  A texel whose
    point is a vertex gets that vertex's position exactly.  normal_fn(points) -> world normals [T,3] (any length) adds a
    tangent-space normal map uint8 [N,N,3] in the same uv as a third result.  return_atlas: also the device tensors of the
    atlas and the texels (dict; with normal_fn also their tangent-space normals and the fp32 filled map).  atlas: "faces"
    (ops.texture_atlas, one isometric chart per face) or "charts" (ops.chart_atlas, multi-face projected charts: denser
    and far fewer seams, stretch up to sqrt(3); its normal map is coded in the decoders' frame).  view: the input photo
    and its camera (prepare_view), blended into the texel colours with their faces' normals (ops.face_normals); with
    return_atlas the dict then also holds the texels' project_weight [T].  ao_fn(points) -> AO [T] in [0, 1] (e.g.
    ao_transfer_fn) adds an occlusion map uint8 [N,N] (ao_quantise of the push-pull filled AO) as the last result."""
    N = check_size(texture_size)
    check_atlas(atlas)
    dev = _device(device)
    vt = torch.from_numpy(np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(faces, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        at = (ops.texture_atlas if atlas == "faces" else ops.chart_atlas)(vt, ft, N)
        index, points, face = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
        rgb = colour_fn(points).float().contiguous()
        extra = {}
        if view is not None:
            rgb, extra["project_weight"] = project(points, ops.face_normals(vt, ft, face), rgb, prepare_view(vt, ft, view))
        tex = ops.texture_fill(index, rgb, at["owner"], N)
        if normal_fn is not None:
            code = ops.tangent_normals if atlas == "faces" else ops.tangent_normals_decoded
            tn = code(vt, ft, at["uv"], face, normal_fn(points).float().contiguous())
            nfill = ops.texture_fill(index, tn, at["owner"], N)
            extra.update(tangent_normals=tn, normal_fill=nfill, normal_map=ops.normal_quantise(nfill))
        if ao_fn is not None:
            ao = ao_fn(points).float().reshape(-1, 1).expand(-1, 3).contiguous()
            extra.update(ao=ao[:, 0], ao_fill=ops.texture_fill(index, ao, at["owner"], N)[..., 0])
    uv, texture = at["uv"].cpu().numpy(), quantise(tex)
    res = (uv, texture) if normal_fn is None else (uv, texture, extra["normal_map"].cpu().numpy())
    res = res if ao_fn is None else (*res, ao_quantise(extra["ao_fill"]))
    if return_atlas:
        return (*res, dict(at, texel_index=index, points=points, texel_face=face, rgb=rgb, **extra))
    return res


def transfer_fn(src_v, src_f, src_c, texture_size=None, device=None, seed=TRANSFER_SEED):
    """A colour_fn for bake that takes colours from a source mesh: src_v [n,3], src_f [m,3], src_c [n,k] uint8 (the
    first three channels, / 255) or float in [0, 1].  The source surface gets 4 N^2 area-uniform samples (4 per texel;
    ops.surface_sample with a fixed seed), each point takes the face of its nearest sample (ops.nearest) and the face's
    vertex colours at its closest point on that face (ops.transfer_colors).  Without texture_size the sample count is 4
    per queried point."""
    dev = _device(device)
    c = np.asarray(src_c)
    c = c[:, :3].astype(np.float32) / np.float32(255) if c.dtype == np.uint8 else c[:, :3].astype(np.float32)
    sv = torch.from_numpy(np.ascontiguousarray(src_v, np.float32).reshape(-1, 3)).to(dev)
    sf = torch.from_numpy(np.ascontiguousarray(src_f, np.int32).reshape(-1, 3)).to(dev)
    return _transfer(sv, sf, torch.from_numpy(np.ascontiguousarray(c)).to(dev), texture_size, seed)


def normal_transfer_fn(src_v, src_f, texture_size=None, device=None, seed=TRANSFER_SEED):
    """A normal_fn for bake that takes normals from a source mesh src_v [n,3], src_f [m,3]: its vertex normals
    (ops.vertex_normals), interpolated at each point's closest point on the face of its nearest source sample, with the
    same seeded samples and search as transfer_fn."""
    dev = _device(device)
    sv = torch.from_numpy(np.ascontiguousarray(src_v, np.float32).reshape(-1, 3)).to(dev)
    sf = torch.from_numpy(np.ascontiguousarray(src_f, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        return _transfer(sv, sf, ops.vertex_normals(sv, sf), texture_size, seed)


def _transfer(sv, sf, values, texture_size, seed):
    """The function of points that interpolates values [n,3] (one row per source vertex) on the face of each point's
    nearest source sample."""
    def fn(points):
        n = TRANSFER_SAMPLES * (check_size(texture_size) ** 2 if texture_size is not None else len(points))
        samples, sample_face = ops.surface_sample(sv, sf, n, seed)
        _, nn = ops.nearest(points, samples)
        return ops.transfer_colors(sv, sf, values, points, nn, sample_face)
    return fn
