"""Meshes per second of `pipeline.images_to_meshes` at the bench configuration (75 / 50 DDIM steps, CFG 3, 96^3 volume,
R = 256, seeded synthetic weights) for several pack sizes K, i.e. Zero123 calls of K images run as one sampler batch
(stage 1 at batch 16 K, stage 2 at batch 64 K).  BASELINE configs[4] when launched under torchrun.

    python tools/throughput.py [--n 8] [--packs 1 2 4 8] [--rounds 2] [--out DIR]
    python -m torch.distributed.run --nproc-per-node G tools/throughput.py ...

Prints one JSON document: the card, its power limit and SM clocks (read in the same run); for each K the meshes/s of the N
images (each rank renders its assign_scenes share; the time is the slowest rank's), the UNet iteration time at batch 16 K and
64 K and per sampled row, and the peak allocated device memory; `max_pack`: the largest K whose UNet time per image still
falls, from the previous K, by more than the run-to-run spread of both, with a peak below --mem-bound-gb.  Every shape is
warmed up first; times are CUDA events; the K values alternate across rounds.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402

STAGES = ((16, 76), (64, 49))     # (sampler batch per image, iterations) of stage 1 and stage 2 at 75 / 50 steps


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(index)], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def unet_ms(unet, B, dev, reps=10):
    """One UNet iteration at batch B in its captured graph, `reps` calls queued back to back as the sampler issues them."""
    x = torch.randn(B, 8, 32, 32, device=dev)
    t = torch.full((B,), 501, device=dev)
    ctx = torch.randn(B, 1, 768, device=dev)
    unet(x, t, ctx)
    return events(lambda: [unet(x, t, ctx) for _ in range(reps)]) / reps


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8, help="synthetic input images")
    ap.add_argument("--packs", type=int, nargs="+", default=[1, 2, 4, 8], help="pack sizes K")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--mem-bound-gb", type=float, default=40.0, help="largest peak allocation a chosen K may need")
    ap.add_argument("--out", default=None, help="also write the JSON document to DIR/throughput.json")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("throughput.py needs a CUDA device")
    import torch.distributed as dist
    from o2345 import sharding, synthetic as S
    from o2345.pipeline import build_networks, images_to_meshes
    from o2345.zero123 import build_zero123
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
    z123 = build_zero123(dev, seed=0, clip=True).half()
    sharding.broadcast_module_weights([tr.pyramid_feature_network_geometry_lod0, tr.sdf_network_lod0, tr.rendering_network_lod0,
                                       tr.variance_network_lod0, z123], src=0)
    mine = sharding.assign_scenes(args.n, world, rank)
    imgs = (S.images(args.n, bench.H, bench.W, seed=4321).transpose(0, 2, 3, 1) * 255.0).astype(np.uint8)
    unet = z123.model.diffusion_model
    info = {"card": card(local), "world": world, "n_images": args.n, "packs": args.packs, "rounds": args.rounds,
            "config": {"ddim_steps": [75, 50], "vol_dim": bench.VOL, "mesh_resolution": bench.MESH_RES, "polar_angle": 60}}

    def run(K, share):
        for _ in images_to_meshes(z123, tr, imgs[share], 60.0, seed=0, resolution=bench.MESH_RES, max_pack=K, indices=share):
            pass

    peak = {}
    for K in args.packs:                       # warm-up: every UNet shape (graph capture) and one whole pack per K
        torch.cuda.reset_peak_memory_stats(dev)
        w = time.perf_counter()
        run(K, mine[:K])
        for per_image, _ in STAGES:
            unet_ms(unet, per_image * K, dev, reps=2)
        torch.cuda.synchronize()
        peak[K] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
        bench.beat("warm-up K=%d: %.1f s, peak %.1f GB" % (K, time.perf_counter() - w, peak[K]))
    clocks = bench.ClockSampler(local)
    clocks.start()
    rows = {K: {"mesh_s": [], "unet_ms": {str(b): [] for b, _ in STAGES}} for K in args.packs}
    for r in range(args.rounds):
        order = args.packs if r % 2 == 0 else args.packs[::-1]
        for K in order:
            for per_image, _ in STAGES:
                rows[K]["unet_ms"][str(per_image)].append(unet_ms(unet, per_image * K, dev))
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            w = time.perf_counter()
            ms = events(lambda: run(K, mine))
            ms, wall = sharding.max_over_ranks([ms, (time.perf_counter() - w) * 1e3], dev)
            rows[K]["mesh_s"].append(ms * 1e-3)
            bench.beat("round %d K=%d: %d images in %.1f s (wall %.1f s)" % (r, K, args.n, ms * 1e-3, wall * 1e-3))
    info["clocks"] = clocks.stop()
    info["card_after"] = card(local)
    res = {}
    for K in args.packs:
        s = rows[K]["mesh_s"]
        u = {b: rows[K]["unet_ms"][str(b)] for b, _ in STAGES}
        per_image = [sum(u[b][i] * n for b, n in STAGES) / K for i in range(args.rounds)]   # UNet ms of one image's 125 iterations
        res[str(K)] = {"meshes_per_s": [args.n / x for x in s], "seconds": s,
                       "unet_iteration_ms": {"stage1_batch%d" % (16 * K): u[16], "stage2_batch%d" % (64 * K): u[64]},
                       "unet_ms_per_row": {"stage1": [x / (16 * K) for x in u[16]], "stage2": [x / (64 * K) for x in u[64]]},
                       "unet_ms_per_image": per_image, "peak_allocated_gb": peak[K]}
    # the largest K that still pays: its median UNet time per image below the previous K's by more than both spreads
    chosen, prev = args.packs[0], None
    for K in args.packs:
        cur = res[str(K)]["unet_ms_per_image"]
        if prev is not None:
            gain = np.median(prev) - np.median(cur)
            spread = max(max(prev) - min(prev), max(cur) - min(cur))
            if gain <= spread or peak[K] > args.mem_bound_gb:
                break
            chosen = K
        prev = cur
    info["results"] = res
    info["max_pack"] = chosen
    info["mem_bound_gb"] = args.mem_bound_gb
    if rank == 0:
        doc = json.dumps(info, indent=1)
        print(doc)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            open(os.path.join(args.out, "throughput.json"), "w").write(doc)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
