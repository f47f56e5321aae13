"""`python run.py --img_path P [P ...] [--polar_angle A [A ...]] [--seed S] [--gpu_idx N] [--half_precision]
[--mesh_resolution R] [--min_component F] [--target_faces N [--remesh]] [--texture_size N [--normal_map] [--ambient_occlusion]
[--atlas charts]]
[--project_input] [--output_format .ply]`

Command-line mirror of the reference's run.py:99-119 for the two accelerated paths: Zero123 stage 1 + stage 2
(8 + 32 views, DDIM 75 / 50 steps, CFG 3) and the cost-volume reconstruction, writing the same artefacts under
./exp/<shape>/ (stage1_8/*.png, stage2_8/*.png, pose.json, mesh.ply).

Not built (SURVEY.md 8(f)): SAM / rembg foreground extraction -- the input must already be a segmented object on a
plain (or transparent) background -- and the LoFTR elevation search (`--polar_angle`, default 60).  Checkpoints: without
`--zero123_ckpt` / `--recon_ckpt` the seeded synthetic weights of o2345.synthetic are used (there is no network access to
fetch the released ones).  With `--zero123_ckpt` the file is loaded the way the reference samples from it: the UNet takes
the EMA shadow (`model_ema.*`, reference ldm/modules/ema.py:14-21 + ddpm.py:180-193), the CLIP ViT-L/14 image tower is
attached and takes `cond_stage_model.*`; a file that lacks what the sampler needs is refused.  `--output_format .obj/.glb`
follow reference utils/utils.py:31-45 (o2345/mesh_io.py).  `--target_faces N` (not in the reference) simplifies the
mesh to N faces on the GPU before mesh.ply is written (o2345/mesh_simplify.py); .obj / .glb are converted from that mesh.
`--remesh` (with `--target_faces N`) replaces that simplification by an isotropic remesh to about N near-equilateral faces
whose vertices lie on the full mesh (o2345/mesh_remesh.py); colours, the projection and the bakes are taken on it.
`--texture_size N` (not in the reference; .obj or .glb only) bakes the reconstruction's colours into an N x N texture on
the GPU (o2345/mesh_texture.py) and writes mesh.glb, or mesh.obj + mesh.mtl + mesh_albedo.png, textured; mesh.ply is
written as without it.  `--normal_map` (with `--texture_size`) also bakes the SDF's gradient into a tangent-space normal
map in the same uv: the GLB gains NORMAL, TANGENT and a normalTexture, the OBJ `vn` and mesh_normal.png (`norm`).
`--ambient_occlusion` (with `--texture_size`) bakes an ambient occlusion map in the same uv: the share of 256
cosine-distributed directions along which the full mesh (before `--target_faces`) is open within a tenth of its box
diagonal, at every vertex on the GPU (o2345/mesh_texture.py), transferred to the texels.  The GLB gains an
occlusionTexture, the OBJ mesh_occlusion.png (`map_ao`).
`--atlas charts` (with `--texture_size`) packs multi-face projected charts instead of one chart per face (the default
`faces`): the full marching-cubes mesh then fits textures of practical size, and only chart borders are seams.
`--project_input` (not in the reference) projects the input photo onto the final mesh from the input camera, so the side
the photo shows keeps its colours (o2345/mesh_texture.py): into mesh.ply's vertex colours and, with `--texture_size`, the
texture.  The photo is read at its own resolution (load_photo), not the 256 x 256 Zero123 input.
`--min_component F` (0 < F <= 1, not in the reference) drops the mesh's floating fragments and enclosed inner shells right
after the vertex merge (o2345/mesh_clean.py): every component whose area is below F times the largest one's, and every
component inside the largest one, goes before simplification, projection and baking.  The counts are printed.

Several images: `--img_path a.png b.png ...` writes exp/<basename>/ for each (basenames must differ); their Zero123
calls run packed into shared sampler batches (o2345.pipeline.images_to_meshes) and image i's noise is seeded with
`--seed` (default 0) + i.  `--polar_angle` takes one value or one per image.  With one image and no `--seed` nothing is
seeded, as in the reference.  Under torchrun (WORLD_SIZE > 1) each rank runs on cuda:LOCAL_RANK, renders the images
o2345.sharding.assign_scenes gives it, and takes its weights from rank 0 (the only collective).
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


PHOTO_MIN, PHOTO_MAX = 256, 2048   # side of the photo load_photo reads for --project_input


def _on_white(im):
    from PIL import Image
    if im.mode == "RGBA":
        bg = Image.new("RGBA", im.size, (255, 255, 255, 255))
        im = Image.alpha_composite(bg, im)
    return im.convert("RGB")


def load_input(path):
    """256 x 256 RGB uint8 on white, like the output of the reference's preprocess() (utils/zero123_utils.py:180-202)."""
    from PIL import Image
    return np.asarray(_on_white(Image.open(path)).resize((256, 256), Image.LANCZOS), np.uint8)


def photo_side(w, h):
    """Side of the square photo --project_input reads from a w x h file: max(w, h) clamped to [PHOTO_MIN, PHOTO_MAX]."""
    return min(max(int(w), int(h), PHOTO_MIN), PHOTO_MAX)


def load_photo(path):
    """The input photo for --project_input: the composite on white of load_input and the same non-uniform resize to a
    square, at side photo_side(w, h) -> dict(photo uint8 [S,S,3], alpha uint8 [S,S] (RGBA files) or None)."""
    from PIL import Image
    im = Image.open(path)
    S = photo_side(*im.size)
    alpha = np.asarray(im.getchannel("A").resize((S, S), Image.LANCZOS), np.uint8) if im.mode == "RGBA" else None
    return {"photo": np.asarray(_on_white(im).resize((S, S), Image.LANCZOS), np.uint8), "alpha": alpha}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="segmented image(s) -> textured mesh(es) on the o2345 (sm_90a) kernels")
    ap.add_argument('--img_path', type=str, nargs='+', default=["./demo/demo_examples/01_wild_hydrant.png"],
                    help='Path(s) to the input image(s)')
    ap.add_argument('--gpu_idx', type=int, default=0, help='GPU index (under torchrun: LOCAL_RANK)')
    ap.add_argument('--half_precision', action='store_true', help='accepted for compatibility: the UNet / VAE kernels are fp16')
    ap.add_argument('--mesh_resolution', type=int, default=256, help='Mesh resolution')
    ap.add_argument('--output_format', type=str, default=".ply", help='Output format: .ply, .obj, .glb')
    ap.add_argument('--target_faces', type=int, default=None,
                    help='simplify the mesh to this many faces (quadric edge collapse; default: the full marching-cubes mesh)')
    ap.add_argument('--texture_size', type=int, default=None,
                    help='bake the colours into an N x N texture (a power of two in [64, 8192]; .obj or .glb output only)')
    ap.add_argument('--normal_map', action='store_true',
                    help='also bake a tangent-space normal map from the SDF gradient (needs --texture_size; .obj or .glb output)')
    ap.add_argument('--ambient_occlusion', action='store_true',
                    help='also bake an ambient occlusion map of the full mesh (needs --texture_size; .obj or .glb output)')
    ap.add_argument('--atlas', choices=("faces", "charts"), default="faces",
                    help='texture atlas: one chart per face (default) or multi-face projected charts (needs --texture_size)')
    ap.add_argument('--project_input', action='store_true',
                    help='project the input photo onto the mesh from the input camera (vertex colours and texture)')
    ap.add_argument('--min_component', type=float, default=None,
                    help='drop mesh components smaller than F times the largest one\'s area or enclosed by it (0 < F <= 1)')
    ap.add_argument('--remesh', action='store_true',
                    help='remesh isotropically to about --target_faces near-equilateral faces instead of simplifying')
    ap.add_argument('--no_ema', action='store_true', help='sample with model.* instead of the EMA shadow model_ema.* (the reference uses EMA)')
    ap.add_argument('--polar_angle', type=float, nargs='+', default=[60.0],
                    help='elevation of the input view in degrees (not estimated): one value, or one per image')
    ap.add_argument('--seed', type=int, default=None,
                    help='base seed of the sampler noise: image i uses seed + i (default: unseeded for one image, 0 for several)')
    ap.add_argument('--zero123_ckpt', type=str, default=None, help='zero123-xl.ckpt (state_dict); default: seeded synthetic weights')
    ap.add_argument('--recon_ckpt', type=str, default=None, help='reconstruction checkpoint (ckpt_*.pth); default: seeded synthetic weights')
    args = ap.parse_args(argv)
    if args.target_faces is not None and args.target_faces < 0:
        ap.error("--target_faces must be >= 0")
    if args.min_component is not None and not 0.0 < args.min_component <= 1.0:
        ap.error("--min_component must lie in (0, 1]")
    if args.texture_size is not None:
        n = args.texture_size
        if n < 64 or n > 8192 or n & (n - 1):
            ap.error("--texture_size must be a power of two in [64, 8192]")
        if args.output_format not in (".obj", ".glb"):
            ap.error("--texture_size needs --output_format .obj or .glb")
    if args.normal_map and args.texture_size is None:
        ap.error("--normal_map needs --texture_size")
    if args.ambient_occlusion and args.texture_size is None:
        ap.error("--ambient_occlusion needs --texture_size")
    if args.atlas != "faces" and args.texture_size is None:
        ap.error("--atlas needs --texture_size")
    if args.remesh and args.target_faces is None:
        ap.error("--remesh needs --target_faces")
    return args


def plan_inputs(paths, polar_angles):
    """-> (shape directories exp/<basename>, one polar angle per image).  Refuses, before any GPU work, two images whose
    outputs would share a directory and a number of polar angles that is neither one nor one per image."""
    ids = [os.path.basename(p).split('.')[0] for p in paths]
    dup = sorted({i for i in ids if ids.count(i) > 1})
    if dup:
        raise SystemExit(f"several input images share the basename {dup[0]!r}: their outputs would both go to exp/{dup[0]}/")
    if len(polar_angles) not in (1, len(paths)):
        raise SystemExit(f"--polar_angle takes one value or one per image: {len(polar_angles)} values for {len(paths)} images")
    polars = list(polar_angles) * len(paths) if len(polar_angles) == 1 else list(polar_angles)
    return [os.path.join("exp", i) for i in ids], polars


def _write_format(shape_dir, output_format, mesh=None):
    if mesh is not None and "texture" in mesh:
        from o2345.mesh_io import to_viewer_frame, write_textured
        v, f, uv = to_viewer_frame(mesh["vertices"], mesh["triangles"], mesh["uv"])
        mesh_path = os.path.join(shape_dir, f"mesh{output_format}")
        write_textured(mesh_path, v, f, uv, mesh["texture"], mesh.get("normal_texture"), mesh.get("occlusion_texture"))
        return mesh_path
    mesh_path = os.path.join(shape_dir, "mesh.ply")
    if output_format == ".ply":          # reference run.py:113-118
        pass
    elif output_format not in (".obj", ".glb"):
        print("Invalid output format, must be one of .ply, .obj, .glb")
    else:
        from o2345.mesh_io import convert_mesh_format
        mesh_path = convert_mesh_format(shape_dir, output_format)
    return mesh_path


def _texture_kw(args):
    kw = {} if args.min_component is None else {"min_component": args.min_component}
    kw = kw if args.texture_size is None else dict(kw, texture_size=args.texture_size)
    kw = kw if args.atlas == "faces" else dict(kw, atlas=args.atlas)
    kw = dict(kw, ambient_occlusion=True) if args.ambient_occlusion else kw
    kw = dict(kw, remesh=True) if args.remesh else kw
    return dict(kw, normal_map=True) if args.normal_map else kw


def main(argv=None):
    args = parse_args(argv)
    shape_dirs, polars = plan_inputs(args.img_path, args.polar_angle)
    if not torch.cuda.is_available():
        raise SystemExit("run.py needs a CUDA device: the o2345 path has no CPU fallback")
    from o2345 import sharding, synthetic as S
    from o2345.mesh_clean import describe
    from o2345.mesh_remesh import describe as describe_remesh
    from o2345.pipeline import build_networks, image_to_mesh, images_to_meshes
    from o2345.zero123 import build_zero123
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)) if world > 1 else args.gpu_idx)
    torch.cuda.set_device(dev)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)

    if args.zero123_ckpt and rank == 0:
        from o2345.zero123 import load_zero123_checkpoint
        model = load_zero123_checkpoint(args.zero123_ckpt, dev, use_ema=not args.no_ema,
                                        report=lambda m: print(m, file=sys.stderr))
    else:
        if rank == 0:
            print("no --zero123_ckpt: seeded synthetic Zero123 weights (the generated views are noise-like)", file=sys.stderr)
        model = build_zero123(dev, seed=0, clip=True)
    model = model.half()

    states = S.all_states(0)
    if args.recon_ckpt and rank == 0:
        from o2345.checkpoints import recon_states
        ck = torch.load(args.recon_ckpt, map_location="cpu")
        states.update(recon_states(ck, report=lambda m: print(m, file=sys.stderr)))
    single = len(args.img_path) == 1 and world == 1
    trainer = build_networks(dev, vol_dim=96, states=states, perturb=0.0, base_exp_dir=shape_dirs[0] if single else None)
    sharding.broadcast_module_weights([model, trainer], src=0)       # rank 0's weights everywhere (no-op for one process)

    if single:                           # one image: exactly the single-image run
        shape_dir = shape_dirs[0]
        os.makedirs(shape_dir, exist_ok=True)
        if args.seed is not None:
            torch.cuda.manual_seed(args.seed)
        mesh = image_to_mesh(model, trainer, load_input(args.img_path[0]), polar_angle=polars[0],
                             resolution=args.mesh_resolution, exp_dir=shape_dir, target_faces=args.target_faces,
                             **_texture_kw(args),
                             **({"project_view": load_photo(args.img_path[0])} if args.project_input else {}))
        mesh_path = _write_format(shape_dir, args.output_format, mesh)
        if "clean" in mesh:
            print(describe(mesh["clean"]))
        if "remesh" in mesh:
            print(describe_remesh(mesh["vertices"], mesh["triangles"], mesh["remesh"]))
        print(f"{len(mesh['vertices'])} vertices, {len(mesh['triangles'])} triangles")
        print("Mesh saved to:", mesh_path)
        return mesh_path

    mine = sharding.assign_scenes(len(args.img_path), world, rank)
    for i in mine:
        os.makedirs(shape_dirs[i], exist_ok=True)
    paths = []
    for i, mesh in images_to_meshes(model, trainer, [load_input(args.img_path[i]) for i in mine], [polars[i] for i in mine],
                                    seed=0 if args.seed is None else args.seed, resolution=args.mesh_resolution,
                                    exp_dirs=[shape_dirs[i] for i in mine], indices=mine, target_faces=args.target_faces,
                                    **_texture_kw(args),
                                    **({"project_views": [load_photo(args.img_path[i]) for i in mine]}
                                       if args.project_input else {})):
        paths.append(_write_format(shape_dirs[i], args.output_format, mesh))
        if "clean" in mesh:
            print(f"{args.img_path[i]}: {describe(mesh['clean'])}")
        if "remesh" in mesh:
            print(f"{args.img_path[i]}: {describe_remesh(mesh['vertices'], mesh['triangles'], mesh['remesh'])}")
        print(f"{args.img_path[i]}: {len(mesh['vertices'])} vertices, {len(mesh['triangles'])} triangles")
        print("Mesh saved to:", paths[-1])
    if world > 1:
        dist.destroy_process_group()
    return paths


if __name__ == "__main__":
    main()
