"""Mesh cleaning on host arrays (run.py --min_component, simplify_mesh.py, GenericTrainer.export_mesh_step): the mesh
goes to the GPU, ops.clean_mesh drops the components that are small next to the largest one or enclosed by it
(csrc/clean.cu) and the kept vertices come back with their own positions and colours, untouched: every output vertex is
an input vertex, and a mesh that loses nothing comes back as it went in."""
from __future__ import annotations

import numpy as np
import torch

from . import ops

STATS = ("components", "largest", "dropped", "dropped_faces", "enclosed")


def clean(vertices, triangles, colors, min_component, device=None):
    """vertices [n,3], triangles [m,3] (welded: mesh_io.merge_vertices), colors [n,k] or None (numpy), 0 < min_component
    <= 1 -> (vertices, triangles int32, colors, stats), the vertices and colours gathered from the inputs (same dtypes);
    stats: dict of the ints components, largest, dropped, dropped_faces and enclosed (ops.clean_mesh).  The device
    defaults to the current CUDA device."""
    if not 0.0 < min_component <= 1.0:
        raise ValueError(f"min_component must lie in (0, 1], got {min_component}")
    v = np.asarray(vertices)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)).to(dev)
    with torch.cuda.device(dev):
        index, faces, stats = ops.clean_mesh(vt, ft, min_component)
    index = index.cpu().numpy()
    return (v[index], faces.cpu().numpy(), None if colors is None else np.asarray(colors)[index],
            {k: stats[k] for k in STATS})


def describe(stats):
    """One line for the command lines: the components found and dropped."""
    return (f"{stats['components']} components, dropped {stats['dropped']} ({stats['dropped_faces']} faces; "
            f"{stats['enclosed']} enclosed by the largest)")
