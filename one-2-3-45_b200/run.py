"""`python run.py --img_path P [--gpu_idx N] [--half_precision] [--mesh_resolution R] [--output_format .ply]`

Command-line mirror of the reference's run.py:99-119 for the two accelerated paths: Zero123 stage 1 + stage 2
(8 + 32 views, DDIM 75 / 50 steps, CFG 3) and the cost-volume reconstruction, writing the same artefacts under
./exp/<shape>/ (stage1_8/*.png, stage2_8/*.png, pose.json, mesh.ply).

Not built (SURVEY.md 8(f)): SAM / rembg foreground extraction -- the input must already be a segmented object on a
plain (or transparent) background -- and the LoFTR elevation search (`--polar_angle`, default 60).  Checkpoints: without
`--zero123_ckpt` / `--recon_ckpt` the seeded synthetic weights of o2345.synthetic are used (there is no network access to
fetch the released ones).  With `--zero123_ckpt` the file is loaded the way the reference samples from it: the UNet takes
the EMA shadow (`model_ema.*`, reference ldm/modules/ema.py:14-21 + ddpm.py:180-193), the CLIP ViT-L/14 image tower is
attached and takes `cond_stage_model.*`; a file that lacks what the sampler needs is refused.  `--output_format .obj/.glb`
follow reference utils/utils.py:31-45 (o2345/mesh_io.py).
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def load_input(path):
    """256 x 256 RGB uint8 on white, like the output of the reference's preprocess() (utils/zero123_utils.py:180-202)."""
    from PIL import Image
    im = Image.open(path)
    if im.mode == "RGBA":
        bg = Image.new("RGBA", im.size, (255, 255, 255, 255))
        im = Image.alpha_composite(bg, im)
    return np.asarray(im.convert("RGB").resize((256, 256), Image.LANCZOS), np.uint8)


def main(argv=None):
    ap = argparse.ArgumentParser(description="single image -> textured mesh on the o2345 (sm_90a) kernels")
    ap.add_argument('--img_path', type=str, default="./demo/demo_examples/01_wild_hydrant.png", help='Path to the input image')
    ap.add_argument('--gpu_idx', type=int, default=0, help='GPU index')
    ap.add_argument('--half_precision', action='store_true', help='accepted for compatibility: the UNet / VAE kernels are fp16')
    ap.add_argument('--mesh_resolution', type=int, default=256, help='Mesh resolution')
    ap.add_argument('--output_format', type=str, default=".ply", help='Output format: .ply, .obj, .glb')
    ap.add_argument('--no_ema', action='store_true', help='sample with model.* instead of the EMA shadow model_ema.* (the reference uses EMA)')
    ap.add_argument('--polar_angle', type=float, default=60.0, help='elevation of the input view in degrees (not estimated)')
    ap.add_argument('--zero123_ckpt', type=str, default=None, help='zero123-xl.ckpt (state_dict); default: seeded synthetic weights')
    ap.add_argument('--recon_ckpt', type=str, default=None, help='reconstruction checkpoint (ckpt_*.pth); default: seeded synthetic weights')
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("run.py needs a CUDA device: the o2345 path has no CPU fallback")
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, image_to_mesh
    from o2345.zero123 import LatentDiffusion, build_zero123
    dev = torch.device("cuda", args.gpu_idx)
    torch.cuda.set_device(dev)

    if args.zero123_ckpt:
        from o2345.zero123 import load_zero123_checkpoint
        model = load_zero123_checkpoint(args.zero123_ckpt, dev, use_ema=not args.no_ema,
                                        report=lambda m: print(m, file=sys.stderr))
    else:
        print("no --zero123_ckpt: seeded synthetic Zero123 weights (the generated views are noise-like)", file=sys.stderr)
        model = build_zero123(dev, seed=0, clip=True)
    model = model.half()

    states = S.all_states(0)
    if args.recon_ckpt:
        from o2345.checkpoints import recon_states
        ck = torch.load(args.recon_ckpt, map_location="cpu")
        states.update(recon_states(ck, report=lambda m: print(m, file=sys.stderr)))
    shape_id = os.path.basename(args.img_path).split('.')[0]
    shape_dir = os.path.join("exp", shape_id)
    os.makedirs(shape_dir, exist_ok=True)
    trainer = build_networks(dev, vol_dim=96, states=states, perturb=0.0, base_exp_dir=shape_dir)

    mesh = image_to_mesh(model, trainer, load_input(args.img_path), polar_angle=args.polar_angle,
                         resolution=args.mesh_resolution, exp_dir=shape_dir)
    mesh_path = os.path.join(shape_dir, "mesh.ply")
    if args.output_format == ".ply":          # reference run.py:113-118
        pass
    elif args.output_format not in (".obj", ".glb"):
        print("Invalid output format, must be one of .ply, .obj, .glb")
    else:
        from o2345.mesh_io import convert_mesh_format
        mesh_path = convert_mesh_format(shape_dir, args.output_format)
    print(f"{len(mesh['vertices'])} vertices, {len(mesh['triangles'])} triangles")
    print("Mesh saved to:", mesh_path)
    return mesh_path


if __name__ == "__main__":
    main()
