"""Texture baking on host arrays (run.py / simplify_mesh.py --texture_size, GenericTrainer.export_mesh_step): every face
gets its own chart in an N x N atlas (ops.texture_atlas; or, with atlas="charts", faces share projected multi-face charts:
ops.chart_atlas), the surface point behind every texel a chart owns is evaluated
by a colour function (ops.texel_points), and the texels no chart owns are filled by push-pull (ops.texture_fill), all in
csrc/texture.cu.  The colour function is the reconstruction's (SparseNeuSRenderer.blend_points, the one that colours the
vertices) or, for a mesh without a reconstruction, the colours of a source mesh (transfer_fn).

A normal map shares the atlas and the texel points: a normal function gives the world normal at every texel's point (the
SDF gradient, or a source mesh's interpolated vertex normals: normal_transfer_fn), ops.tangent_normals codes it in the
face's tangent frame (the rule of include/o2345.h, which mesh_io's writers and the rasterizer decode), the same push-pull
fills the rest and ops.normal_quantise codes it to uint8."""
from __future__ import annotations

import numpy as np
import torch

from . import ops

MIN_SIZE, MAX_SIZE = 64, 8192
ATLASES = ("faces", "charts")  # ops.texture_atlas (the default) and ops.chart_atlas
TRANSFER_SEED = 0          # seed of the source surface samples of transfer_fn
TRANSFER_SAMPLES = 4       # source samples per texel of the atlas


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


def bake(vertices, faces, texture_size, colour_fn, device=None, return_atlas=False, normal_fn=None, atlas="faces"):
    """vertices [n,3], faces [m,3] (numpy) -> (uv float32 [m,3,2], texture uint8 [N,N,3]); uv row k belongs to corner
    faces[f, k], in glTF's convention (v down the image, texel i's centre at (i + 0.5) / N).  colour_fn(points [T,3] fp32
    device tensor) -> rgb [T,3] in [0, 1] on the device, for the surface point behind every owned texel.  A texel whose
    point is a vertex gets that vertex's position exactly.  normal_fn(points) -> world normals [T,3] (any length) adds a
    tangent-space normal map uint8 [N,N,3] in the same uv as a third result.  return_atlas: also the device tensors of the
    atlas and the texels (dict; with normal_fn also their tangent-space normals and the fp32 filled map).  atlas: "faces"
    (ops.texture_atlas, one isometric chart per face) or "charts" (ops.chart_atlas, multi-face projected charts: denser
    and far fewer seams, stretch up to sqrt(3); its normal map is coded in the decoders' frame)."""
    N = check_size(texture_size)
    check_atlas(atlas)
    dev = _device(device)
    vt = torch.from_numpy(np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(faces, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        at = (ops.texture_atlas if atlas == "faces" else ops.chart_atlas)(vt, ft, N)
        index, points, face = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
        rgb = colour_fn(points).float().contiguous()
        tex = ops.texture_fill(index, rgb, at["owner"], N)
        extra = {}
        if normal_fn is not None:
            code = ops.tangent_normals if atlas == "faces" else ops.tangent_normals_decoded
            tn = code(vt, ft, at["uv"], face, normal_fn(points).float().contiguous())
            nfill = ops.texture_fill(index, tn, at["owner"], N)
            extra = {"tangent_normals": tn, "normal_fill": nfill, "normal_map": ops.normal_quantise(nfill)}
    uv, texture = at["uv"].cpu().numpy(), quantise(tex)
    res = (uv, texture) if normal_fn is None else (uv, texture, extra["normal_map"].cpu().numpy())
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
