"""`python exp_runner_generic_blender_val.py --specific_dataset_name <exp_dir> --mode export_mesh --conf C --resolution R`

Command-line mirror of the reference's reconstruction/exp_runner_generic_blender_val.py:596-640 for the two inference
modes of the demo configuration:
  export_mesh   <exp_dir>/{pose.json, stage1_8, stage2_8} -> <exp_dir>/mesh.ply   (what run.py's reconstruct() shells out to)
  val           volume-renders the query view -> <exp_dir>/val_color.png, val_depth.npy, val_normal.npy
  turntable     volume-renders --n_frames views (default 36) on the circle of the input view, at its elevation and radius
                -> <exp_dir>/turntable/000.png ... (RGBA), <exp_dir>/turntable.gif (on white), turntable_depth.npy [n,H,W]
A conf with `model.num_lods = 2` adds the lod-1 level (`model.sdf_network_lod1`, `model.rendering_network_lod1`):
export_mesh writes the lod-1 mesh, val also writes val_color_lod1.png, val_depth_lod1.npy and val_normal_lod1.npy, and
turntable renders the lod-1 level.
`--conf` is parsed (o2345/checkpoints.py: the HOCON subset the reference's confs use; pyhocon is not needed) and supplies
`model.sdf_network_lod0` (voxel_size, vol_dims, ...), `model.variance_network`, `model.rendering_network`, `model.trainer`
(samples, perturb) and `general.base_exp_dir`; if the file does not exist the constants of
confs/one2345_lod0_val_demo.conf are used.  Weights: `--checkpoint_path`, else -- as the reference does with
`--is_continue` (:137-149) -- the lexicographically last `<base_exp_dir>/checkpoints/ckpt*.pth`, else the seeded synthetic
weights.  Training modes stay with the reference.
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


MODES = ("export_mesh", "val", "turntable")


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--conf', type=str, default='./confs/one2345_lod0_val_demo.conf')
    ap.add_argument('--mode', type=str, default='export_mesh')
    ap.add_argument('--threshold', type=float, default=0.0)
    ap.add_argument('--is_continue', default=False, action="store_true")
    ap.add_argument('--is_restore', default=False, action="store_true")
    ap.add_argument('--is_finetune', default=False, action="store_true")
    ap.add_argument('--train_from_scratch', default=False, action="store_true")
    ap.add_argument('--restore_lod0', default=False, action="store_true")
    ap.add_argument('--local_rank', type=int, default=0)
    ap.add_argument('--specific_dataset_name', type=str, default='GSO')
    ap.add_argument('--resolution', type=int, default=360)
    ap.add_argument('--checkpoint_path', type=str, default=None, help='ckpt_*.pth of the reference (default: synthetic weights)')
    ap.add_argument('--n_frames', type=int, default=36, help='turntable: number of views around the object')
    args = ap.parse_args(argv)
    if args.mode not in MODES:
        raise SystemExit(f"mode={args.mode!r}: only 'export_mesh' and 'val' of the reference's modes, plus 'turntable', run on the "
                         "o2345 path (training stays with the reference)")
    if args.n_frames < 1:
        raise SystemExit(f"--n_frames must be at least 1, got {args.n_frames}")
    return args


def main(argv=None):
    args = parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the o2345 path has no CPU fallback")
    from o2345 import synthetic as S
    from o2345.checkpoints import latest_checkpoint, load_conf, recon_states
    from o2345.pipeline import build_networks, load_sample, render_turntable
    dev = torch.device("cuda", args.local_rank)
    torch.cuda.set_device(dev)
    exp_dir = args.specific_dataset_name
    note = lambda m: print(m, file=sys.stderr)
    conf = load_conf(args.conf) if os.path.exists(args.conf) else None
    if conf is None:
        note(f"conf {args.conf!r} not found: using the built-in constants of confs/one2345_lod0_val_demo.conf")
    num_lods = conf.get_int('model.num_lods') if conf is not None else 1
    states = S.all_states(0)
    if num_lods > 1:
        states.update(S.lod1_states(0))
    ckpt = args.checkpoint_path
    if ckpt is None and conf is not None and args.is_continue:
        ckpt = latest_checkpoint(conf['general.base_exp_dir'])
        if ckpt is not None:
            note(f"Find checkpoint: {os.path.basename(ckpt)}")
    if ckpt is not None:
        states.update(recon_states(torch.load(ckpt, map_location="cpu"), report=note, num_lods=num_lods))
    else:
        note("no checkpoint: seeded synthetic reconstruction weights")
    trainer = build_networks(dev, states=states, base_exp_dir=exp_dir, conf=conf,
                             **({} if conf is not None else {"vol_dim": 96, "perturb": 0.0}))
    if args.mode == "turntable":
        out = render_turntable(trainer, exp_dir, args.n_frames, out_dir=exp_dir)
        print(f"{args.n_frames} turntable frames written to {os.path.join(exp_dir, 'turntable')}")
        return out
    sample = load_sample(exp_dir, dev)
    if args.mode == "export_mesh":
        mesh = trainer(sample, mode="export_mesh", resolution=args.resolution)
        print(f"{len(mesh['vertices'])} vertices, {len(mesh['triangles'])} triangles -> {os.path.join(exp_dir, 'mesh.ply')}")
        return mesh
    # perturb_overwrite stays -1: the stratified jitter follows the conf's model.trainer.perturb (1.0 in the demo conf), as in
    # the reference's validate(); white background and alpha_inter_ratio 1.0 as at iter_step 215 000 (:412-418,528-540)
    # (512-ray chunks as in the reference: the host generator's draws -- jitter, then 1024 random points per chunk -- interleave
    # the same way)
    out = trainer(sample, mode="val", background_rgb=1.0, alpha_inter_ratio_lod0=1.0, alpha_inter_ratio_lod1=1.0)
    W, H = int(sample['img_wh'][0][0]), int(sample['img_wh'][0][1])
    from PIL import Image
    for suffix in ("", "_lod1")[:num_lods]:
        Image.fromarray((np.clip(out["color" + suffix].reshape(H, W, 3), 0, 1) * 255).astype(np.uint8)).save(
            os.path.join(exp_dir, f"val_color{suffix}.png"))
        np.save(os.path.join(exp_dir, f"val_depth{suffix}.npy"), out["depth" + suffix].reshape(H, W))
        np.save(os.path.join(exp_dir, f"val_normal{suffix}.npy"), out["normal" + suffix].reshape(H, W, 3))
    print("val outputs written to", exp_dir)
    return out


if __name__ == "__main__":
    main()
