"""Mesh simplification on host arrays (run.py --target_faces, simplify_mesh.py, GenericTrainer.export_mesh_step): the
mesh goes to the GPU, ops.simplify_mesh reduces it (csrc/simplify.cu) and the kept vertices come back with their own
positions and colours, untouched: every output vertex is an input vertex."""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def simplify(vertices, triangles, colors, target_faces, device=None):
    """vertices [n,3], triangles [m,3], colors [n,k] or None (numpy) -> (vertices, triangles int32, colors, rounds), the
    vertices and colours gathered from the inputs (same dtypes).  The device defaults to the current CUDA device."""
    if target_faces < 0:
        raise ValueError(f"target_faces must be >= 0, got {target_faces}")
    v = np.asarray(vertices)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        index, faces, rounds = ops.simplify_mesh(vt, ft, target_faces)
    index = index.cpu().numpy()
    return v[index], faces.cpu().numpy(), None if colors is None else np.asarray(colors)[index], rounds
