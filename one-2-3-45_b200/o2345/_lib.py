"""ctypes binding of libo2345_sm90.so (the C-ABI declared in include/o2345.h).

There is deliberately NO fallback: if the shared library is missing or a call fails this module
raises, it never routes work to PyTorch or to the CPU oracle.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("O2345_LIB") or os.path.join(os.path.dirname(HERE), "lib", "libo2345_sm90.so")   # O2345_LIB: A/B against another build (tools/)

c_fp = C.c_void_p  # device pointers travel as integers
c_i64 = C.c_int64


class Points(C.Structure):
    _fields_ = [("mode", C.c_int), ("pts", c_fp), ("lin", c_fp), ("R", C.c_int), ("rays_o", c_fp),
                ("rays_d", c_fp), ("z", c_fp), ("S", C.c_int), ("z_stride", C.c_int)]


class View4(C.Structure):
    _fields_ = [("ptr", c_fp), ("sn", c_i64), ("sc", c_i64), ("sh", c_i64), ("sw", c_i64), ("c0", C.c_int)]


class Views(C.Structure):
    _fields_ = [("V", C.c_int), ("H", C.c_int), ("W", C.c_int), ("maps", c_fp), ("proj", c_fp),
                ("centers", c_fp), ("sizeW", C.c_float), ("sizeH", C.c_float)]


class Epilogue(C.Structure):
    _fields_ = [("bias", c_fp), ("residual", c_fp), ("rowbias", c_fp), ("rowbias_ld", c_i64), ("rows_per_group", C.c_int),
                ("act", C.c_int), ("alpha", C.c_float), ("out_f32", C.c_int)]


class RasterMesh(C.Structure):
    _fields_ = [("verts", c_fp), ("colors", c_fp), ("uvs", c_fp), ("faces", c_fp), ("face_tex", c_fp), ("texels", c_fp),
                ("tex_info", c_fp), ("normals", c_fp), ("tangents", c_fp), ("face_ntex", c_fp), ("nv", c_i64), ("nf", c_i64),
                ("n_tex", C.c_int)]


PTS_EXPLICIT, PTS_LATTICE, PTS_RAYS = 0, 1, 2
BLEND_FP32, BLEND_TC_FP16 = 0, 1
SDF_FP32, SDF_TC_SPLIT = 0, 1
SDF_PACK_FLOATS = 39 * 128 + 128 + 2 * (144 * 128 + 128) + 128 * 144 + 128 * 48
RNET_PACK_FLOATS = 19664
MAP_CH = 60
SHADE_UNLIT, SHADE_LAMBERT = 0, 1
WRAP_REPEAT, WRAP_CLAMP, WRAP_MIRROR = 0, 1, 2

_SIGS = {
    "o2345_abi_version": (C.c_int, []),
    "o2345_last_error": (C.c_int, [C.c_char_p, C.c_size_t]),
    "o2345_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "o2345_sdf_pack_weights": (C.c_int, [c_fp] * 7 + [c_fp]),
    "o2345_sdf_query": (C.c_int, [C.POINTER(Points), c_i64, c_fp, C.c_int, c_fp, c_fp, C.c_float, C.c_int, C.c_int,
                                  c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_frustum_mask": (C.c_int, [c_fp, C.c_int, c_fp, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, c_fp,
                                     c_fp, c_fp]),
    "o2345_compact_scratch_ints": (c_i64, [c_i64]),
    "o2345_compact": (C.c_int, [c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_costvol_gather": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp, C.c_float,
                                       C.c_int, c_fp, c_fp, c_i64, c_fp, c_fp, c_fp]),
    "o2345_dense_scatter": (C.c_int, [c_fp, c_fp, c_fp, c_i64, C.c_int, c_fp, c_fp, c_fp, c_fp]),
    "o2345_sdf_voxels": (C.c_int, [c_fp, c_fp, C.c_int, c_fp, C.c_float, c_fp, C.c_int, c_fp, c_fp]),
    "o2345_prune_by_sdf": (C.c_int, [c_fp, c_fp, C.c_int, C.POINTER(C.c_float), C.c_int, c_fp, c_fp, c_fp, c_fp]),
    "o2345_prune_select": (C.c_int, [c_fp, c_i64, C.c_float, c_fp, c_fp]),
    "o2345_clear_flags": (C.c_int, [c_fp, c_fp, c_i64, c_fp, c_fp]),
    "o2345_gather_rows": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, C.c_int, c_fp, c_fp, c_fp]),
    "o2345_lod_children": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_costvol_gather_lod": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp, C.c_float,
                                           C.c_int, c_fp, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_occ_nearest": (C.c_int, [C.POINTER(Points), c_i64, c_fp, C.c_int, c_fp, c_fp]),
    "o2345_sp_coarsen": (C.c_int, [c_fp, C.c_int, c_fp, c_fp, c_i64, C.c_int, c_fp, c_fp, c_fp]),
    "o2345_sp_conv": (C.c_int, [c_fp, c_fp, C.c_int, c_fp, c_fp, c_i64, C.c_int, C.c_int, c_fp, C.c_int, C.c_int,
                                c_fp, c_fp, c_fp]),
    "o2345_sp_bn_relu": (C.c_int, [c_fp, c_fp, c_i64, C.c_int, c_fp, c_fp, c_fp, C.c_float, c_fp, c_fp, c_fp]),
    "o2345_mc_classify": (C.c_int, [c_fp, C.c_int, C.c_float, c_fp, c_fp, c_fp, c_fp]),
    "o2345_mc_vertices": (C.c_int, [c_fp, C.c_int, C.c_float, c_fp, c_fp, c_i64, c_fp, c_fp]),
    "o2345_scan_scratch_ints": (c_i64, [c_i64]),
    "o2345_mc_tri_offsets": (C.c_int, [c_fp, c_fp, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_mc_triangles": (C.c_int, [c_fp, C.c_int, c_fp, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_conv2d": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp, C.c_int, C.c_int, C.c_int,
                               C.c_int, c_fp, c_fp, c_fp]),
    "o2345_abn_apply": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp, c_fp, C.c_float, C.c_float,
                                  C.POINTER(View4), c_fp]),
    "o2345_upsample_bilinear": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_fp,
                                          C.POINTER(View4), c_fp]),
    "o2345_ray_upsample": (C.c_int, [c_fp, c_fp, c_i64, c_fp, c_fp, C.c_int, C.c_float, c_fp, C.c_int, c_fp,
                                     C.c_int, c_fp, c_fp]),
    "o2345_ray_merge": (C.c_int, [c_fp, c_fp, C.c_int, c_fp, c_fp, C.c_int, c_i64, c_fp, c_fp, c_fp]),
    "o2345_ray_midpoints": (C.c_int, [c_fp, c_fp, c_i64, c_fp, C.c_int, C.c_float, c_fp, C.c_int, c_fp, c_fp,
                                      c_fp, c_fp]),
    "o2345_ray_midpoints_per_ray": (C.c_int, [c_fp, c_fp, c_i64, c_fp, C.c_int, c_fp, c_fp, C.c_int, c_fp, c_fp, c_fp, c_fp]),
    "o2345_render_blend": (C.c_int, [C.POINTER(Points), c_i64, c_fp, c_fp, c_fp, C.c_int, C.POINTER(Views),
                                     C.c_int, c_fp, c_fp, c_fp, C.c_int, c_fp, c_fp, c_fp]),
    "o2345_gemm_f16": (C.c_int, [c_fp, c_fp, c_fp, C.c_int, C.c_int, C.c_int, c_i64, c_i64, c_i64, C.c_int, C.c_int,
                                 c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, C.POINTER(Epilogue), c_fp, c_i64, c_fp]),
    "o2345_debug_gemm_trace": (None, [c_fp]),
    "o2345_debug_gemm_force": (None, [C.c_int, C.c_int, C.c_int]),
    "o2345_debug_gemm_persist": (None, [C.c_int, C.c_int]),
    "o2345_debug_groupnorm_cluster": (None, [C.c_int]),
    "o2345_debug_gemm_model": (None, [C.POINTER(C.c_float)]),
    "o2345_last_trap": (C.c_int, [C.c_char_p, C.c_size_t]),
    "o2345_conv3x3_f16": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, C.c_int, c_fp, c_i64,
                                    C.POINTER(Epilogue), c_fp, c_i64, c_fp]),
    "o2345_conv_up2x_f16": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, C.c_int, c_fp, c_i64,
                                      C.POINTER(Epilogue), c_fp, c_i64, c_fp]),
    "o2345_groupnorm_scratch_floats": (c_i64, [C.c_int, C.c_int]),
    "o2345_groupnorm_stats": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_fp, c_fp, c_fp, c_fp, c_fp,
                                        c_fp]),
    "o2345_groupnorm_apply": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_fp, c_fp, C.c_int, c_fp, c_fp]),
    "o2345_norm_act_im2col": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp,
                                        C.c_int, c_fp, c_fp]),
    "o2345_layernorm_rows": (C.c_int, [c_fp, c_i64, C.c_int, C.c_float, c_fp, c_fp, c_fp, c_fp]),
    "o2345_softmax_rows": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, c_fp]),
    "o2345_attention_f16": (C.c_int, [c_fp, c_fp, c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, C.c_int,
                                      C.c_float, c_fp]),
    "o2345_geglu": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, c_fp]),
    "o2345_silu": (C.c_int, [c_fp, c_i64, c_fp, c_fp]),
    "o2345_transpose_tokens": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, c_fp, c_fp]),
    "o2345_timestep_embedding": (C.c_int, [c_fp, C.c_int, C.c_int, c_fp, c_fp]),
    "o2345_add_channel_bias": (C.c_int, [c_fp, c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp]),
    "o2345_copy_channels": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, C.c_int, C.c_int, c_fp]),
    "o2345_nchw_f32_to_cl_f16": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, c_fp, C.c_int, C.c_int, c_fp]),
    "o2345_cl_f16_to_nchw_f32": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, c_fp, c_fp]),
    "o2345_cfg_ddim_update": (C.c_int, [c_fp, c_fp, c_fp, c_i64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                        c_fp, c_fp, c_fp]),
    "o2345_clip_patches": (C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                     C.c_int, c_fp, c_fp]),
    "o2345_clip_add_positions": (C.c_int, [c_fp, c_fp, c_fp, C.c_int, C.c_int, C.c_int, c_fp]),
    "o2345_raster_scratch_bytes": (c_i64, [c_i64, c_i64, C.c_int, C.c_int, C.c_int]),
    "o2345_raster": (C.c_int, [C.POINTER(RasterMesh), C.c_int, c_fp, c_fp, C.c_int, C.c_int, C.c_float, C.c_int, c_fp, c_i64,
                               c_fp, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_debug_raster_split": (None, [C.c_int]),
    "o2345_surface_sample_scratch_bytes": (c_i64, [c_i64]),
    "o2345_surface_sample": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_i64, C.c_uint64, c_fp, c_i64, c_fp, c_fp, c_fp]),
    "o2345_nn_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_nearest": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp]),
    "o2345_simplify_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_simplify": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp]),
    "o2345_texture_atlas_scratch_bytes": (c_i64, [c_i64]),
    "o2345_texture_atlas": (C.c_int, [c_fp, c_i64, c_fp, c_i64, C.c_int, c_fp, c_i64, c_fp, c_fp, c_fp,
                                      C.POINTER(C.c_int32), C.POINTER(C.c_double), c_fp]),
    "o2345_chart_atlas_scratch_bytes": (c_i64, [c_i64, c_i64, C.c_int]),
    "o2345_chart_atlas": (C.c_int, [c_fp, c_i64, c_fp, c_i64, C.c_int, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp,
                                    C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_int32),
                                    C.POINTER(C.c_int32), c_fp]),
    "o2345_texel_points_scratch_bytes": (c_i64, [C.c_int]),
    "o2345_texel_points": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, C.c_int, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp]),
    "o2345_texture_fill_scratch_bytes": (c_i64, [C.c_int]),
    "o2345_texture_fill": (C.c_int, [c_fp, c_fp, c_fp, c_fp, C.c_int, c_fp, c_i64, c_fp, c_fp]),
    "o2345_transfer_colors": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_i64, c_fp, c_fp, c_i64, c_fp, c_fp]),
    "o2345_tangent_normals": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp, c_i64, c_fp, c_fp]),
    "o2345_tangent_normals_decoded": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp, c_i64, c_fp, c_fp]),
    "o2345_normal_quantise": (C.c_int, [c_fp, c_i64, c_fp, c_fp]),
    "o2345_vertex_normals_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_vertex_normals": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_i64, c_fp, c_fp]),
    "o2345_project_view": (C.c_int, [c_fp, c_fp, c_fp, c_i64, c_fp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                     c_fp, c_fp, C.c_int, C.c_int, c_fp, C.c_int, c_fp, c_fp, c_fp]),
    "o2345_face_normals": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_i64, c_fp, c_fp]),
    "o2345_clean_mesh_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_clean_mesh": (C.c_int, [c_fp, c_i64, c_fp, c_i64, C.c_double, c_fp, c_i64, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp,
                                   c_fp, c_fp]),
    "o2345_ambient_occlusion_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_ambient_occlusion": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_i64, c_fp, C.c_int, C.c_float, C.c_float,
                                          c_fp, c_i64, c_fp, c_fp]),
    "o2345_closest_points_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "o2345_closest_points": (C.c_int, [c_fp, c_i64, c_fp, c_i64, c_fp, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp]),
    "o2345_remesh_scratch_bytes": (c_i64, [c_i64, c_i64, c_i64, c_i64]),
    "o2345_remesh": (C.c_int, [c_fp, c_i64, c_fp, c_i64, C.c_float, C.c_int, c_i64, c_i64, c_fp, c_i64, c_fp, c_fp, c_fp,
                               c_fp]),
    "o2345_ray_composite": (C.c_int, [c_fp, c_i64, C.c_int, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, C.c_float,
                                      C.c_float, C.c_int, C.c_float, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp]),
}

EXPORTED = tuple(_SIGS)
ABI_VERSION = 14         # include/o2345.h: O2345_ABI_VERSION
_lib = None


ENOSPC = -4              # include/o2345.h: O2345_ENOSPC


class O2345Error(RuntimeError):
    pass


def load():
    """Loads the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise O2345Error(f"{LIB_PATH} is missing: run `python one-2-3-45_b200/build.py` "
                             "(there is no CPU or PyTorch fallback for this path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        if lib.o2345_abi_version() != ABI_VERSION:
            raise O2345Error(f"{LIB_PATH} has ABI version {lib.o2345_abi_version()}, this binding expects {ABI_VERSION}: "
                             "rebuild with `python one-2-3-45_b200/build.py`")
        _lib = lib
    return _lib


def last_trap() -> str:
    """Description of the bounded GEMM wait that expired (and trapped) in this process, or '' if none did."""
    buf = C.create_string_buffer(512)
    return buf.value.decode(errors="replace") if load().o2345_last_trap(buf, 512) == 1 else ""


def last_error() -> str:
    buf = C.create_string_buffer(512)
    load().o2345_last_error(buf, 512)
    return buf.value.decode(errors="replace")


# kernels launched per successful entry-point call (memsets are not counted)
_KERNELS_PER_CALL = {"o2345_compact": 3, "o2345_prune_by_sdf": 3, "o2345_sp_coarsen": 3, "o2345_mc_tri_offsets": 4, "o2345_conv_up2x_f16": 4, "o2345_raster": 4, "o2345_surface_sample": 5, "o2345_nearest": 7, "o2345_texel_points": 5, "o2345_vertex_normals": 8}
_launches = 0


def reset_launches():
    global _launches
    _launches = 0


def add_launches(n: int):
    """Kernels replayed by a captured CUDA graph (counted once at capture time)."""
    global _launches
    _launches += n


def launches() -> int:
    """Number of o2345 kernels launched since reset_launches() (bench.py's gpu_launches)."""
    return _launches


def call(name, *args):
    """Calls an int-returning entry point and raises O2345Error on a negative status."""
    global _launches
    rc = getattr(load(), name)(*args)
    if rc != 0:
        raise O2345Error(f"{name} failed with {rc}: {last_error()}")
    _launches += _KERNELS_PER_CALL.get(name, 1)
    return rc


def inference_only(fn):
    """Decorator for the module methods that run o2345 kernels: the kernels are forward / inference only, so a call with
    autograd enabled on a module whose parameters require grad is refused with a clear error instead of silently
    returning tensors without a graph (SURVEY.md 8(b) note 2: training stays with the reference).  Otherwise the call
    runs under torch.no_grad()."""
    import torch

    @functools.wraps(fn)
    def wrap(self, *args, **kwargs):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError(f"o2345 {type(self).__name__}.{fn.__name__} is inference-only: call it under torch.no_grad() or "
                               "freeze the parameters (requires_grad_(False)); training stays with the reference")
        with torch.no_grad():
            return fn(self, *args, **kwargs)
    return wrap
