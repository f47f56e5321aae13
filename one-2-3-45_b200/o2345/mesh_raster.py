"""Meshes on the GPU from the reference's 24-view evaluation rig (reference render/single_render_eval.py, run by
render/launch_render_eval.py under Blender 3.6 + BlenderProc), restated from the script's own code.

  load_scene       .obj / .glb as Blender's importers bring them in: glTF and OBJ are Y-up, so (x, y, z) -> (x, -z, y);
                   .ply (this project's write_ply) with Blender 3.6's PLY importer defaults (no axis change).  The script
                   itself refuses .ply: accepting it is an extension.  .fbx is refused (no path here follows Blender's
                   FBX importer).
  normalize_scene  the script's normalize_scene: the bbox over the corners of every mesh object's local AABB taken to
                   world, every root object scaled by 0.8 / max extent about its own origin, the bbox taken again and
                   -(min + max) / 2 added to every root's translation.
  rig_cameras      24 views: polar 60 deg x 12 then 90 deg x 12, azimuth 0, 30, ..., 330 deg; camera at
                   (r sin(phi) cos(theta), r sin(phi) sin(theta), r cos(phi)) looking at the origin with
                   to_track_quat('-Z', 'Y'); 35 mm lens on a 32 mm sensor (fx = fy = 560 px at 512^2), principal point at
                   the image centre.  The script renders 512^2 whatever --resolution says; here the resolution is honoured.
  render           csrc/raster.cu through ops.raster: colour, alpha, depth, normal, triangle id as device tensors.

Parity unpinned: neither Blender nor BlenderProc is available, so the rig is restated from the script's code, not pinned
against renders.  Geometry, silhouette and depth follow the rig; colour is a defined model (unlit base colour, or the
Lambert stand-in of O2345_SHADE_LAMBERT for the rig's overhead area light), not Cycles' lighting or the Filmic view
transform.  A glTF normal map (normalTexture with NORMAL and TANGENT) replaces the face normal in the normal output and
the Lambert term; a NORMAL without a normal map does not (faces stay flat).  Alpha modes and metallic-roughness are
ignored: the base colour is opaque."""
from __future__ import annotations

import math
import os

import numpy as np

from . import mesh_io

Y_UP_TO_Z_UP = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])   # (x, y, z) -> (x, -z, y)
SHADINGS = {"unlit": 0, "lambert": 1}
NEAR = 0.1   # Blender's default camera clip start; the rig's objects stay beyond 1.3 - 0.8 * sqrt(3) / 2 > 0.6


def _h(R):
    M = np.eye(4)
    M[:3, :3] = R
    return M


def load_scene(path, y_up=None):
    """-> scene dict in Blender's axes: roots [4x4 world matrices], meshes (verts local, faces, colors or None, uvs or None,
    face_tex or None, normals / tangents / face_ntex or None (GLB only), root, local_to_root) and textures
    [(RGBA [h,w,4], wrap s, wrap t)].  y_up overrides the format's axis
    convention (True: apply the Y-up -> Z-up change, False: none)."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".glb":
        g = mesh_io.read_glb(path)
        roots, meshes, textures = g["roots"], g["meshes"], g["textures"]
    elif ext == ".obj":
        v, f, c = mesh_io.read_obj(path)
        roots, textures = [np.eye(4)], []
        meshes = [{"verts": v, "faces": f, "colors": c, "uvs": None, "face_tex": None, "root": 0, "local_to_root": np.eye(4)}]
    elif ext == ".ply":
        v, f, c = mesh_io.read_ply(path)
        roots, textures = [np.eye(4)], []
        meshes = [{"verts": v.astype(np.float64), "faces": f.astype(np.int64), "colors": c[:, :3] / 255.0, "uvs": None,
                   "face_tex": None, "root": 0, "local_to_root": np.eye(4)}]
    elif ext == ".fbx":
        raise ValueError(f"{path}: .fbx is not supported (only .obj, .glb and .ply)")
    else:
        raise ValueError(f"{path}: unsupported mesh format {ext!r} (only .obj, .glb and .ply)")
    if y_up is None:
        y_up = ext in (".glb", ".obj")
    if y_up:
        # Blender's importers convert every node transform (C M C^T) and the mesh data (C v)
        C = _h(Y_UP_TO_Z_UP)
        roots = [C @ R @ C.T for R in roots]
        for m in meshes:
            m["verts"] = m["verts"] @ Y_UP_TO_Z_UP.T
            m["local_to_root"] = C @ m["local_to_root"] @ C.T
            if m.get("normals") is not None:       # a rotation: normals and tangents turn like positions
                m["normals"] = m["normals"] @ Y_UP_TO_Z_UP.T
            if m.get("tangents") is not None:
                m["tangents"] = np.concatenate([m["tangents"][:, :3] @ Y_UP_TO_Z_UP.T, m["tangents"][:, 3:]], 1)
    return {"roots": [np.asarray(R, np.float64) for R in roots], "meshes": meshes, "textures": textures}


def scene_bbox(scene):
    """The script's scene_bbox: min / max over the 8 corners of every mesh object's local AABB, taken to world."""
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    for m in scene["meshes"]:
        if len(m["verts"]) == 0:
            continue
        a, b = m["verts"].min(0), m["verts"].max(0)
        corners = np.array([[x, y, z, 1.0] for x in (a[0], b[0]) for y in (a[1], b[1]) for z in (a[2], b[2])])
        w = corners @ (scene["roots"][m["root"]] @ m["local_to_root"]).T
        lo, hi = np.minimum(lo, w[:, :3].min(0)), np.maximum(hi, w[:, :3].max(0))
    if not np.isfinite(lo).all():
        raise ValueError("no mesh objects in the scene to compute a bounding box for")
    return lo, hi


def normalize_scene(scene):
    """In place, as the script's normalize_scene; returns the scene."""
    lo, hi = scene_bbox(scene)
    s = 0.8 / float((hi - lo).max())
    scene["roots"] = [R @ np.diag([s, s, s, 1.0]) for R in scene["roots"]]
    lo, hi = scene_bbox(scene)
    for R in scene["roots"]:
        R[:3, 3] += -(lo + hi) / 2
    return scene


def flatten(scene):
    """World-space arrays of ops.raster / oracle.raster_oracle.render: verts float32 [nv,3], faces int32 [nf,3], colors
    float32 [nv,3] (or None when no object has any), uvs float32 [nv,2] + face_tex int32 [nf] + texels uint8 + tex_info
    int32 [n_tex,5] (or None when no face is textured), normals float32 [nv,3] + tangents float32 [nv,4] + face_ntex int32
    [nf] (or None when no face has a normal map).  Tangents go through each object's linear part A, normals through
    A^-T, and the tangent w is multiplied by sign(det A)."""
    vs, fs, cs, us, ts, ns, gs, nts, n = [], [], [], [], [], [], [], [], 0
    any_col = any(m["colors"] is not None for m in scene["meshes"])
    for m in scene["meshes"]:
        M = scene["roots"][m["root"]] @ m["local_to_root"]
        A = M[:3, :3]
        v = m["verts"] @ A.T + M[:3, 3]
        vs.append(v)
        fs.append(m["faces"] + n)
        cs.append(m["colors"] if m["colors"] is not None else np.ones((len(v), 3)))
        us.append(m["uvs"] if m["uvs"] is not None else np.zeros((len(v), 2)))
        ts.append(m["face_tex"] if m["face_tex"] is not None else np.full(len(m["faces"]), -1))
        nts.append(m["face_ntex"] if m.get("face_ntex") is not None else np.full(len(m["faces"]), -1))
        if (nts[-1] >= 0).any():
            ns.append(m["normals"] @ np.linalg.inv(A))
            g = m["tangents"]
            gs.append(np.concatenate([g[:, :3] @ A.T, g[:, 3:] * np.sign(np.linalg.det(A))], 1))
        else:
            ns.append(np.zeros((len(v), 3)))
            gs.append(np.zeros((len(v), 4)))
        n += len(v)
    out = {"verts": np.concatenate(vs).astype(np.float32), "faces": np.concatenate(fs).astype(np.int32),
           "colors": np.concatenate(cs).astype(np.float32) if any_col else None,
           "uvs": None, "face_tex": None, "texels": None, "tex_info": None, "normals": None, "tangents": None,
           "face_ntex": None}
    face_tex = np.concatenate(ts).astype(np.int32)
    face_ntex = np.concatenate(nts).astype(np.int32)
    if scene["textures"] and (face_ntex >= 0).any():
        out.update(normals=np.concatenate(ns).astype(np.float32), tangents=np.concatenate(gs).astype(np.float32),
                   face_ntex=face_ntex)
    if scene["textures"] and ((face_tex >= 0).any() or (face_ntex >= 0).any()):
        info, first = [], 0
        for rgba, ws, wt in scene["textures"]:
            info.append([first, rgba.shape[1], rgba.shape[0], ws, wt])
            first += rgba.shape[0] * rgba.shape[1]
        out.update(uvs=np.concatenate(us).astype(np.float32), face_tex=face_tex,
                   texels=np.concatenate([t[0].reshape(-1) for t in scene["textures"]]).astype(np.uint8),
                   tex_info=np.asarray(info, np.int32))
    return out


def rig_cameras(camera_dist=1.5, resolution=512):
    """-> c2w [24,4,4] (OpenCV: x right, y down, z forward) and K [3,3] of the script's 24 views."""
    polar = np.radians([60.0] * 12 + [90.0] * 12)
    azim = np.radians([*range(0, 360, 30)] * 2)
    c2w = np.zeros((24, 4, 4))
    for i, (phi, th) in enumerate(zip(polar, azim)):
        loc = camera_dist * np.array([math.sin(phi) * math.cos(th), math.sin(phi) * math.sin(th), math.cos(phi)])
        zb = loc / np.linalg.norm(loc)                        # Blender camera +Z points away from the target
        xb = np.cross([0.0, 0.0, 1.0], zb)                    # to_track_quat('-Z', 'Y'): camera Y as close to world +Z
        xb /= np.linalg.norm(xb)
        yb = np.cross(zb, xb)
        c2w[i, :3, 0], c2w[i, :3, 1], c2w[i, :3, 2], c2w[i, :3, 3] = xb, -yb, -zb, loc
        c2w[i, 3, 3] = 1.0
    f = 35.0 / 32.0 * resolution
    K = np.array([[f, 0.0, resolution / 2.0], [0.0, f, resolution / 2.0], [0.0, 0.0, 1.0]])
    return c2w, K


def camera_arrays(c2w, K):
    """c2w [V,4,4] and K [3,3] or [V,3,3] -> w2c float32 [V,3,4], intr float32 [V,4] = (fx, fy, cx, cy)."""
    c2w = np.asarray(c2w, np.float64).reshape(-1, 4, 4)
    K = np.broadcast_to(np.asarray(K, np.float64).reshape(-1, 3, 3), (len(c2w), 3, 3))
    w2c = np.linalg.inv(c2w)[:, :3, :4]
    intr = np.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], 1)
    return w2c.astype(np.float32), intr.astype(np.float32)


def render(flat, c2w, K, W, H, shading="unlit", near=NEAR, device="cuda"):
    """Renders flatten()'s arrays from cameras c2w [V,4,4] (OpenCV) with intrinsics K -> device tensors color [V,H,W,3],
    alpha [V,H,W], depth [V,H,W] (camera z, 0 on the background), normal [V,H,W,3] (unit world face normal, or the normal
    map's, toward the camera), tri [V,H,W] int32 (face index into flat['faces'], -1 on the background)."""
    import torch
    from . import ops
    if shading not in SHADINGS:
        raise ValueError(f"shading must be one of {sorted(SHADINGS)}, got {shading!r}")
    w2c, intr = camera_arrays(c2w, K)
    dev = torch.device(device)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with torch.cuda.device(dev):
        return ops.raster(t(flat["verts"]), t(flat["faces"]), t(w2c), t(intr), int(W), int(H), near=near,
                          shading=SHADINGS[shading], colors=t(flat["colors"]), uvs=t(flat["uvs"]),
                          face_tex=t(flat["face_tex"]), texels=t(flat["texels"]), tex_info=t(flat["tex_info"]),
                          normals=t(flat.get("normals")), tangents=t(flat.get("tangents")), face_ntex=t(flat.get("face_ntex")))


def render_rig(path, camera_dist=1.5, resolution=512, shading="unlit", device="cuda"):
    """Loads, normalises and renders `path` from the 24 rig views -> render()'s dict."""
    flat = flatten(normalize_scene(load_scene(path)))
    c2w, K = rig_cameras(camera_dist, resolution)
    return render(flat, c2w, K, resolution, resolution, shading=shading, device=device)


def write_views(out, output_dir):
    """output_dir/0.png ... (RGBA, the script's names: colour over coverage), depth.npy [V,H,W], normal.npy [V,H,W,3]."""
    import torch
    from PIL import Image
    os.makedirs(output_dir, exist_ok=True)
    rgba = torch.cat([out["color"].clamp(0, 1), out["alpha"][..., None]], -1)
    rgba = (rgba * 255).round().to(torch.uint8).cpu().numpy()
    for i in range(len(rgba)):
        Image.fromarray(rgba[i], "RGBA").save(os.path.join(output_dir, f"{i}.png"))
    np.save(os.path.join(output_dir, "depth.npy"), out["depth"].cpu().numpy())
    np.save(os.path.join(output_dir, "normal.npy"), out["normal"].cpu().numpy())
