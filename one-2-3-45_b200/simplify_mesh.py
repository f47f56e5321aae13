"""Simplifies a mesh on the GPU (o2345/mesh_simplify.py, csrc/simplify.cu):

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out small.glb --target_faces 20000

Reads .ply (as run.py writes it) or .obj, welds coincident vertices first (mesh_io.merge_vertices: an OBJ written with
one vertex per face corner would otherwise be all boundary, and boundary vertices are never removed), reduces it to
--target_faces or one fewer faces by quadric-driven half-edge collapse and writes .ply, .obj or .glb by the output's
extension, in the input's own coordinates.  Every output vertex is an input vertex with its colour.  Prints the face and
vertex counts before and after and the number of rounds.

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out small.glb --target_faces 5000 --texture_size 2048

--texture_size N (.glb or .obj output) also bakes the welded input's vertex colours into an N x N texture of the
simplified mesh (o2345/mesh_texture.py: each texel takes the colour of the input surface at its nearest point) and
writes it textured: .glb with the texture embedded, .obj beside <stem>.mtl and <stem>_albedo.png.

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out small.glb --target_faces 5000 --texture_size 2048 --normal_map

--normal_map (with --texture_size) also bakes the welded input's vertex normals, taken at the same nearest points, into a
tangent-space normal map, so the simplified mesh shades like the full one: the .glb gains NORMAL, TANGENT and a
normalTexture, the .obj `vn` lines and <stem>_normal.png (`norm` in the MTL).

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out small.glb --target_faces 5000 --texture_size 2048 --ambient_occlusion

--ambient_occlusion (with --texture_size) also bakes the welded input's ambient occlusion (at its vertices, against the
input itself, transferred like the colours) into an occlusion map: the .glb gains an occlusionTexture, the .obj
<stem>_occlusion.png (`map_ao` in the MTL).

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out full.glb --target_faces 1000000 --texture_size 1024 --atlas charts

--atlas charts (with --texture_size) bakes into multi-face projected charts instead of one chart per face: meshes with
far more faces fit the texture, and only chart borders are seams.

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out small.glb --target_faces 5000 --min_component 0.05

--remesh replaces the simplification by an isotropic remesh to about --target_faces faces (o2345/mesh_remesh.py): long
edges split, short ones collapse, edges flip towards valence 6 and the vertices relax and go back onto the input surface.
Each vertex takes the input's colour at its closest point of the input.

    python one-2-3-45_b200/simplify_mesh.py --in mesh.ply --out even.glb --target_faces 20000 --remesh

--min_component F (0 < F <= 1) cleans the welded input first (o2345/mesh_clean.py): components whose area is below F
times the largest one's, and components enclosed by the largest one, are dropped.  The cleaned mesh is what is simplified
and what the texture, normal map and occlusion map are transferred from, so a dropped fragment gives no texel its colour
and occludes nothing."""
from __future__ import annotations

import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

INPUTS = (".ply", ".obj")
OUTPUTS = (".ply", ".obj", ".glb")
TEXTURED = (".obj", ".glb")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--in", dest="inp", required=True, help="input mesh (.ply or .obj)")
    ap.add_argument("--out", required=True, help="output mesh (.ply, .obj or .glb)")
    ap.add_argument("--target_faces", type=int, required=True, help="number of faces to reduce to")
    ap.add_argument("--texture_size", type=int, default=None,
                    help="bake the colours into an N x N texture (a power of two in [64, 8192]; .obj or .glb output)")
    ap.add_argument("--normal_map", action="store_true",
                    help="also bake the input's normals into a tangent-space normal map (needs --texture_size)")
    ap.add_argument("--ambient_occlusion", action="store_true",
                    help="also bake the input's ambient occlusion into an occlusion map (needs --texture_size)")
    ap.add_argument("--atlas", choices=("faces", "charts"), default="faces",
                    help="texture atlas: one chart per face (default) or multi-face projected charts (needs --texture_size)")
    ap.add_argument("--min_component", type=float, default=None,
                    help="first drop components smaller than F times the largest one's area or enclosed by it (0 < F <= 1)")
    ap.add_argument("--remesh", action="store_true",
                    help="remesh isotropically to about --target_faces near-equilateral faces instead of simplifying")
    args = ap.parse_args(argv)
    if os.path.splitext(args.inp)[1].lower() not in INPUTS:
        ap.error(f"{args.inp}: unsupported input format (only {', '.join(INPUTS)})")
    if os.path.splitext(args.out)[1].lower() not in OUTPUTS:
        ap.error(f"{args.out}: unsupported output format (only {', '.join(OUTPUTS)})")
    if args.target_faces < 0:
        ap.error("--target_faces must be >= 0")
    if args.min_component is not None and not 0.0 < args.min_component <= 1.0:
        ap.error("--min_component must lie in (0, 1]")
    if args.texture_size is not None:
        n = args.texture_size
        if n < 64 or n > 8192 or n & (n - 1):
            ap.error("--texture_size must be a power of two in [64, 8192]")
        if os.path.splitext(args.out)[1].lower() not in TEXTURED:
            ap.error(f"--texture_size needs a {' or '.join(TEXTURED)} output")
    if args.normal_map and args.texture_size is None:
        ap.error("--normal_map needs --texture_size")
    if args.ambient_occlusion and args.texture_size is None:
        ap.error("--ambient_occlusion needs --texture_size")
    if args.atlas != "faces" and args.texture_size is None:
        ap.error("--atlas needs --texture_size")
    return args


def read_mesh(path):
    """-> (vertices float32 [n,3], triangles [m,3], colors uint8 [n,4]); an OBJ without colours is white."""
    import numpy as np
    from o2345 import mesh_io
    if path.lower().endswith(".ply"):
        return mesh_io.read_ply(path)
    v, f, c = mesh_io.read_obj(path)
    c = np.ones((len(v), 3)) if c is None else c
    rgba = np.concatenate([np.round(np.clip(c, 0, 1) * 255), np.full((len(v), 1), 255)], 1).astype(np.uint8)
    return v.astype(np.float32), f, rgba


def write_mesh(path, v, f, c):
    from o2345 import mesh_io
    ext = os.path.splitext(path)[1].lower()
    {".ply": mesh_io.write_ply, ".obj": mesh_io.write_obj, ".glb": mesh_io.write_glb}[ext](path, v, f, c)


def main(argv=None):
    args = parse_args(argv)
    from o2345 import mesh_io
    from o2345.mesh_simplify import simplify
    v, f, c = read_mesh(args.inp)
    print(f"read {args.inp}: {len(v)} vertices, {len(f)} faces")
    v, f, c = mesh_io.merge_vertices(v, f, c)
    print(f"welded: {len(v)} vertices, {len(f)} faces")
    if args.min_component is not None:
        from o2345.mesh_clean import clean, describe
        v, f, c, stats = clean(v, f, c, args.min_component)
        print(f"cleaned: {describe(stats)}: {len(v)} vertices, {len(f)} faces")
    src = (v, f, c)
    if args.remesh:
        from o2345.mesh_remesh import describe, remesh, surface_colors
        v, f, stats = remesh(v, f, None, args.target_faces)
        c = surface_colors(*src, v)
        rounds = stats["rounds"]
        print(describe(v, f, stats))
    else:
        v, f, c, rounds = simplify(v, f, c, args.target_faces)
        print(f"simplified: {len(v)} vertices, {len(f)} faces in {rounds} rounds")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    if args.texture_size is not None:
        from o2345.mesh_texture import ao_transfer_fn, bake, normal_transfer_fn, transfer_fn
        nfn = normal_transfer_fn(*src[:2], texture_size=args.texture_size) if args.normal_map else None
        afn = ao_transfer_fn(*src[:2], texture_size=args.texture_size) if args.ambient_occlusion else None
        baked = bake(v, f, args.texture_size, transfer_fn(*src, texture_size=args.texture_size), normal_fn=nfn,
                     atlas=args.atlas, ao_fn=afn)
        print(f"baked a {args.texture_size} x {args.texture_size} texture" + (" and normal map" if args.normal_map else "")
              + (" and occlusion map" if args.ambient_occlusion else ""))
        mesh_io.write_textured(args.out, v, f, *baked[:2], normal_texture=baked[2] if args.normal_map else None,
                               occlusion_texture=baked[-1] if args.ambient_occlusion else None)
        print("wrote", args.out)
        return (v, f, c, rounds, *baked)
    write_mesh(args.out, v, f, c)
    print("wrote", args.out)
    return v, f, c, rounds


if __name__ == "__main__":
    main()
