"""bench.py -- One-2-3-45 hot paths on H100: sec/mesh end to end, and volume-render M rays/sec.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--dump-outputs DIR]

Headline metric (BASELINE.json, configs[1]): "sec/mesh end-to-end (256x256 in)".  One step = one 256x256 input
image -> Zero123 stage 1 + stage 2 (the reference's 10 DDIM sampler calls = 2x76 + 8x49 = 544 UNet passes over a CFG
batch of 8, run here as the two batched calls they collapse to when the elevation is given: 76 iterations at batch 16 + 49
at batch 64, same views, same noise per view; fp16 tensor-core GEMMs with fp32 accumulate; 9 CLIP ViT-L/14 image embeddings,
9 VAE encodes, 40 VAE decodes)
-> 32 views -> FeatureNet ->
96^3 cost volume -> sparse U-Net -> 256^3 SDF grid -> marching cubes -> vertex colours -> mesh arrays on the host
(`o2345.pipeline.image_to_mesh`).  Not inside the step (out of scope, SURVEY.md section 8(f)): SAM / rembg
preprocessing and the LoFTR elevation search (polar angle 60).
`value` is timed on the device with CUDA events; `e2e` is the wall clock of the same public call starting from a
pinned host image and ending with the mesh on the host (the pipeline itself moves the generated views through the
host as uint8, as the reference's PNG hand-off does).  The second BASELINE metric, "volume-render M rays/sec", is
reported under "rays" with its own roofline (GenericTrainer mode='val' on 65 536 rays x (64+64) samples x 32 views).
N > 1: one process per GPU, one independent image per rank (weak scaling, no data-path collective).
--dump-outputs DIR: after the timed steps, fixed-shape seeded samples of the arrays the last step returned (mesh vertices,
triangles, colours, SDF grid) go to DIR/<name>.npy, so that two builds can be compared output for output on the same seeded
inputs.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H = W = 256
N_VIEWS = 32
VOL = 96
N_RAYS = H * W
CHUNK = 65536   # rays marched per launch group (the reference uses 512; results are per-ray, the chunk only sets the launch count)
MESH_RES = 256
UNET_ITERS = 2 * 76 + 8 * 49             # the reference's sampler calls: UNet passes at batch 8 (what the CPU arm extrapolates with)
UNET_SCHEDULE = ((16, 76), (64, 49))     # (batch = views x CFG, iterations): stage 1 (8 views), stage 2 (32 views)
CONFIG = {"workload": "configs[1]: single 256x256 image -> mesh: Zero123 75/50-step DDIM fp16 (the reference's 2x76 + 8x49 UNet passes "
                      "at batch 8 = 4352 sample-iterations, batched as 76 iterations at batch 16 + 49 at batch 64) "
                      "+ 96^3 cost volume + 256^3 SDF grid + marching cubes, 1 image per GPU",
          "views": N_VIEWS, "vol_dim": VOL, "mesh_resolution": MESH_RES, "ddim_steps": [75, 50], "cfg_scale": 3.0,
          "l2": "inputs larger than L2 (1.72 GB fp16 UNet weights stream every iteration; 470 MB feature maps)",
          "not_in_step": "SAM/rembg, LoFTR elevation search (polar angle 60)",
          "parallelism": "one image per GPU"}
# algorithmic work, SURVEY.md section 8(d)
UNET_FLOP_PER_SAMPLE = 176.3e9
FLOP_SDF_FWD = 2 * 41856.0
FLOP_SDF_BWD = 2 * (128 * 144 + 128 * 39)
RAY_FLOP, RAY_GATHER_BYTES = 211e6, 4.0e6
PUBLISHED_SEC_PER_MESH = 40.0   # BASELINE.md section 1 (reference README.md:154, A6000, whole run.py)


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        p = json.load(open(path))
        return {"hbm_gbs": p["hbm_gbs"], "bf16_tflops": p["bf16_tflops"], "bf16_sustained": p.get("bf16_tflops_sustained"),
                "source": "measured"}
    # NVIDIA's H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense FP16 / BF16
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_sustained": None, "source": "data sheet"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.index), "-lms", "200"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        ok = [r for r in self.rows if len(r) >= 8 and r[1].replace(".", "").isdigit()]
        sm = [float(r[1]) for r in ok]
        mx = [float(r[2]) for r in ok]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in ok for i in range(4) if r[4 + i].lower().startswith("active")})
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


def input_image(seed):
    from o2345 import synthetic as S
    return (S.images(1, H, W, seed=seed)[0].transpose(1, 2, 0) * 255.0).astype(np.uint8)


_T0 = time.perf_counter()


def beat(msg):
    """Progress line on stderr (never stdout: ONE JSON line is the contract) so that a stall is attributable."""
    sys.stderr.write("[bench %7.1f s] %s\n" % (time.perf_counter() - _T0, msg))
    sys.stderr.flush()


def ev_time(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def run_gpu(args):
    """Order of work (each phase announces itself on stderr):  [cpu baseline starts in a child process]  ->  networks  ->
    warm-up steps  ->  stage breakdown / roofline / rays (untimed extras, BEFORE the timed region so that nothing can
    stand between the timed loop and the JSON line)  ->  join the cpu baseline  ->  barrier, timed steps, barrier  ->
    the ONE JSON line, immediately."""
    import torch.distributed as dist
    from o2345 import _lib, sharding, synthetic as S
    from o2345.pipeline import build_networks, image_to_mesh
    from o2345.zero123 import build_zero123
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if world != args.gpus:
        raise SystemExit(f"bench.py --gpus {args.gpus} was launched with WORLD_SIZE={world}: start it with "
                         f"`python -m torch.distributed.run --nproc-per-node {args.gpus} bench.py --gpus {args.gpus}`")
    if args.warmup < 3:
        beat("note: fewer than 3 warm-up steps requested; the timing rules ask for W >= 3")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    cpu_job = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu_job = CpuBaselineJob()       # host cores work while the GPU side builds and warms up; joined before the timed region
    if world > 1:
        # keep NCCL's version banner / warnings off stdout: ONE JSON line is the contract
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
        dist.init_process_group("nccl", device_id=dev)
        beat("process group up: rank %d of %d on cuda:%d" % (rank, world, local))
    tr = build_networks(dev, vol_dim=VOL, states=S.all_states(0), perturb=0.0)
    z123 = build_zero123(dev, seed=0, clip=True).half()   # `--half_precision`: fp16-rounded schedule buffers; CLIP tower attached
    # the only collective on the path: weights from rank 0 over NVLink (no-op at N = 1)
    nb = sharding.broadcast_module_weights([tr.pyramid_feature_network_geometry_lod0, tr.sdf_network_lod0,
                                            tr.rendering_network_lod0, tr.variance_network_lod0, z123], src=0)
    beat("networks built (%d weight elements broadcast)" % nb)
    img_host = torch.from_numpy(input_image(4321 + rank)).pin_memory()
    step = lambda: image_to_mesh(z123, tr, img_host.numpy(), polar_angle=60, resolution=MESH_RES)

    for i in range(args.warmup):
        w = time.perf_counter()
        step()
        beat("warm-up step %d: %.2f s" % (i, time.perf_counter() - w))
    torch.cuda.synchronize()
    pk = peaks()
    # the host-side baseline must be finished before anything else is measured (its 32 threads slow this process's launches)
    cpu = cpu_job.join() if cpu_job is not None else None
    extras = stage_breakdown(z123, tr, dev, pk, world)
    # every rank renders its own image at the same time: the job's ray throughput is the per-rank rate of the slowest
    # rank times the number of ranks
    img_ms = sharding.max_over_ranks([extras["rays"]["image_ms"]], dev)[0]
    extras["rays"]["image_ms"] = img_ms
    extras["rays"]["value"] = world * N_RAYS / (img_ms * 1e-3) / 1e6
    extras["rays"]["n_gpus"] = world
    # the extras above ran other kernels and allocated / freed gigabytes (eager PyTorch UNet, 256^3 grids): one more untimed
    # step brings the allocator and the caches back to the steady state the timed steps are meant to measure
    w = time.perf_counter()
    step()
    beat("settling step after the extras: %.2f s" % (time.perf_counter() - w))
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    clocks = ClockSampler(local)
    clocks.start()
    torch.manual_seed(0)             # the timed steps draw the same sampler noise in every run with the same arguments
    _lib.reset_launches()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    t0.record()
    for i in range(args.steps):
        w = time.perf_counter()
        mesh = step()
        beat("timed step %d: %.2f s" % (i, time.perf_counter() - w))
    t1.record()
    torch.cuda.synchronize()
    wall_s = time.perf_counter() - w0
    launches = _lib.launches()
    clk = clocks.stop()
    if args.dump_outputs:
        dump_outputs(args.dump_outputs if world == 1 else os.path.join(args.dump_outputs, "rank%d" % rank), mesh)
    ms, e2e_ms = sharding.max_over_ranks([t0.elapsed_time(t1), wall_s * 1e3], dev)
    if rank == 0:
        sec_per_mesh = ms * 1e-3 / (args.steps * world)
        out = {"metric": "sec/mesh end-to-end (256x256 in)", "value": sec_per_mesh, "unit": "s/mesh", "n_gpus": world,
               "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": False,
               "scaling": "weak", "vs_baseline": sec_per_mesh / PUBLISHED_SEC_PER_MESH, "dtype": "f16", "data": "synthetic",
               "config": CONFIG, "baseline_note": "BASELINE.md section 1: 40 s per image for run.py --half_precision on an A6000 "
                                                  "(reference README.md:154), which also covers SAM, the LoFTR elevation "
                                                  "search, model loading and a second process start -- not in this step",
               "clocks": clk, "gpu_launches": launches,
               "e2e": {"value": e2e_ms * 1e-3 / (args.steps * world), "unit": "s/mesh", "h2d_bytes_per_step": int(img_host.numel()),
                       "d2h_bytes_per_step": int(mesh["vertices"].nbytes + mesh["triangles"].nbytes + mesh["colors"].nbytes)},
               "mesh": {"vertices": int(len(mesh["vertices"])), "triangles": int(len(mesh["triangles"]))},
               "peaks": pk["source"]}
        out.update(extras)
        if cpu is not None:
            out["cpu_baseline"] = cpu
        emit(json.dumps(out))
        beat("JSON line written")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


class CpuBaselineJob:
    """`cpu_baseline` of the main arm: the CPU port timed in a CHILD process (`bench.py --cpu-baseline-child`) that starts
    with the bench and runs while this process builds the networks and warms the GPU up; it is joined (or, past its
    deadline, killed and reported as such) before the timed region starts, so it can neither perturb nor delay the
    timed steps and the JSON line."""

    DEADLINE_S = 300.0

    def __init__(self):
        self.t0 = time.perf_counter()
        env = dict(os.environ)
        for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "OMP_NUM_THREADS", "MKL_NUM_THREADS"):
            env.pop(k, None)            # torchrun pins OMP_NUM_THREADS=1 for its workers; the CPU arm uses the host cores
        env["CUDA_VISIBLE_DEVICES"] = ""
        self.proc = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--cpu-baseline-child"],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, env=env)
        beat("cpu baseline started in child process %d" % self.proc.pid)

    def join(self):
        left = self.DEADLINE_S - (time.perf_counter() - self.t0)
        try:
            out, _ = self.proc.communicate(timeout=max(left, 1.0))
            res = json.loads(out.strip().splitlines()[-1])
            beat("cpu baseline joined: %.0f s/mesh on %d threads" % (res["value"], res["cores"]))
            return res
        except Exception as e:   # the baseline is a reported extra: never let it take the bench line down
            self.proc.kill()
            beat("cpu baseline unavailable: %r" % (e,))
            return {"value": None, "unit": "s/mesh", "cores": host_threads(), "kind": "port",
                    "sample": "unavailable: %s" % type(e).__name__}


def stage_breakdown(z123, tr, dev, pk, world=1):
    """Per-stage device times, the tensor-core roofline of the dominant kernel (the wgmma GEMM inside the UNet)
    and the volume-rendering throughput with its own roofline.  Untimed extras; every rank runs them (symmetric)."""
    beat("stage breakdown: UNet iterations")
    from o2345 import ops_a
    from o2345.pipeline import synthetic_sample
    unet, vae = z123.model.diffusion_model, z123.first_stage_model

    def unet_profile(B):
        """(ms per iteration in the captured graph, ms of its GEMM launches alone, their FLOPs, their count, inputs)."""
        x = torch.randn(B, 8, 32, 32, device=dev)
        t = torch.full((B,), 501, device=dev)
        ctx = torch.randn(B, 1, 768, device=dev)
        unet(x, t, ctx)
        # 10 calls queued behind each other, as the sampler issues them (a call timed alone on an idle GPU would include
        # its own host-side launch latency, which the sampler hides behind the previous iteration)
        ms_unet = ev_time(lambda: [unet(x, t, ctx) for _ in range(10)])[0] / 10.0
        # Device time of the tensor-core kernel inside one UNet pass: every GEMM / implicit-conv call of an eager pass is
        # recorded (operands kept alive) and replayed back to back inside ONE CUDA graph, timed with events around the
        # replay -- the kernel's launches exactly as the captured UNet graph issues them, without the glue kernels between.
        rec = []
        real = {n: getattr(ops_a, n) for n in ("gemm", "bgemm", "conv3x3", "conv_up2x")}

        def spy(name):
            def wrap(*a, **k):
                rec.append((name, a, k))
                return real[name](*a, **k)
            return wrap
        for n in real:
            setattr(ops_a, n, spy(n))
        unet.use_cuda_graph = False
        try:
            unet(x, t, ctx)
            torch.cuda.synchronize()
        finally:
            for n in real:
                setattr(ops_a, n, real[n])
            unet.use_cuda_graph = True
        flops_counted, algo_bytes = 0.0, 0.0
        for name, a, k in rec:
            res = 2.0 if k.get("residual") is not None else 0.0
            if name == "gemm":
                M, K, N = a[0].shape[0], a[0].shape[1], a[1].shape[0]
                n_out = N // 2 if k.get("act", 0) == ops_a.ACT_GEGLU else N
                flops_counted += 2.0 * M * K * N
                algo_bytes += 2.0 * (M * K + N * K) + (2.0 + res) * M * n_out
            elif name == "conv3x3":
                M, C, N = a[1] * a[2] * a[3], a[4], a[5].shape[0]
                flops_counted += 2.0 * M * 9 * C * N
                algo_bytes += 2.0 * (M * C + N * 9 * C) + (2.0 + res) * M * N          # the activation is read once, not nine times
            elif name == "conv_up2x":                                                  # four 2x2 phase convolutions = four launches
                M, C, N = a[1] * a[2] * a[3], a[4], a[5].shape[1]
                flops_counted += 4 * 2.0 * M * 4 * C * N
                algo_bytes += 2.0 * (M * C + 16 * C * N) + 2.0 * 4 * M * N
            else:
                flops_counted += 2.0 * a[3] * a[4] * a[8] * a[9] * a[10]
                algo_bytes += 2.0 * a[3] * a[4] * (a[8] * a[10] + a[9] * a[10] + a[8] * a[9])
        side = torch.cuda.Stream()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            for name, a, k in rec:
                real[name](*a, **k)
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, stream=side):
                for name, a, k in rec:
                    real[name](*a, **k)
        graph.replay()
        torch.cuda.synchronize()
        ms_gemm = float(np.median([ev_time(graph.replay)[0] for _ in range(10)]))
        n = sum(4 if name == "conv_up2x" else 1 for name, a, k in rec)
        del graph, rec
        beat("stage breakdown: UNet iteration at batch %d: %.3f ms; its %d GEMM launches replay in %.3f ms (%.0f TFLOP/s)"
             % (B, ms_unet, n, ms_gemm, flops_counted / ms_gemm / 1e9))
        return ms_unet, ms_gemm, flops_counted, n, (x, t, ctx), algo_bytes

    prof = {B: unet_profile(B) for B, _ in UNET_SCHEDULE}
    B_TOP = max(UNET_SCHEDULE, key=lambda bi: prof[bi[0]][0] * bi[1])[0]       # the batch whose iterations take the larger share
    ms_unet, ms_gemm, flops_counted, n_gemm, (x, t, ctx), algo_bytes = prof[B_TOP]
    # informational (SURVEY.md 2a "beats PyTorch / cuDNN on the same box"): the plain-PyTorch restatement of the same UNet
    # (oracle/ldm_oracle.py: F.conv2d / F.linear / einsum attention -> cuDNN + cuBLAS) under fp16 autocast on this GPU, eager,
    # outside every timed region, at the same batch.  It is the reference's execution model, not the product path.
    ms_torch = None
    if int(os.environ.get("RANK", 0)) == 0:
        try:
            from o2345 import synthetic as S
            from oracle import ldm_oracle as LO
            sd_t = {k: torch.from_numpy(v).to(dev) for k, v in S.unet_state(0).items()}
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                for _ in range(2):
                    LO.unet_forward(sd_t, x, t, ctx)
                ms_torch = float(np.median([ev_time(lambda: LO.unet_forward(sd_t, x, t, ctx))[0] for _ in range(5)]))
            del sd_t
            torch.cuda.empty_cache()
            beat("stage breakdown: plain PyTorch (cuDNN / cuBLAS, fp16 autocast, eager) UNet iteration at batch %d: %.2f ms" % (B_TOP, ms_torch))
        except Exception as e:
            beat("stage breakdown: plain-PyTorch UNet timing skipped: %r" % (e,))
    z = torch.randn(4, 4, 32, 32, device=dev)
    vae.decode(z)
    ms_dec = float(np.mean([ev_time(lambda: vae.decode(z))[0] for _ in range(3)]))
    flops = B_TOP * UNET_FLOP_PER_SAMPLE
    tf = flops_counted / (ms_gemm * 1e-3) / 1e12
    roofline = {"kernel": "gemm_tc_kernel<BN, STAGES, MODE> (wgmma.mma_async m64nBNk16 f16, TMA operands; all %d GEMM / implicit-conv "
                          "launches of one UNet iteration at batch %d, the batch of the 49 stage-2 iterations)" % (n_gemm, B_TOP),
                "bound": "tensor", "achieved": tf, "peak": pk["bf16_tflops"], "unit": "TFLOP/s", "frac": tf / pk["bf16_tflops"],
                "algorithmic_bytes_per_launch": algo_bytes / max(n_gemm, 1),
                "flops_per_step": flops_counted, "gemm_ms_per_unet_iteration": ms_gemm,
                "other_batches": {str(B): {"unet_iteration_ms": prof[B][0], "gemm_ms": prof[B][1],
                                           "tflops": prof[B][2] / (prof[B][1] * 1e-3) / 1e12} for B, _ in UNET_SCHEDULE if B != B_TOP},
                "note": "algorithmic FLOPs = sum of 2 M N K over the recorded launches (%.1f GFLOP; SURVEY.md 8(d) row A2 quotes "
                        "%.1f GFLOP for the same pass including attention) / CUDA-event time of those launches replayed back to back "
                        "in one CUDA graph (split-K reductions are inside the kernel)" % (flops_counted / 1e9, flops / 1e9)}
    # ---- reconstruction stages + volume rendering
    beat("stage breakdown: reconstruction + volume rendering")
    sample = synthetic_sample(dev, n_views=N_VIEWS, H=H, W=W)
    tr._conditional_features(sample)
    ms_front, (imgs, fmaps, cond, sizeW, sizeH) = ev_time(lambda: tr._conditional_features(sample))
    tr.base_exp_dir = None
    tr(sample, mode="export_mesh", resolution=MESH_RES)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    tr(sample, mode="export_mesh", resolution=MESH_RES)
    torch.cuda.synchronize()
    s_mesh = time.perf_counter() - w0
    rays = render_throughput(tr, sample, imgs, fmaps, cond, sizeW, sizeH, dev, pk)
    stages = {"unet_iteration_ms": {"batch%d" % B: prof[B][0] for B, _ in UNET_SCHEDULE},
              "unet_total_s": sum(prof[B][0] * n for B, n in UNET_SCHEDULE) * 1e-3,
              "torch_gpu_unet_ms": ms_torch, "torch_gpu_unet_batch": B_TOP, "vae_decode4_ms": ms_dec,
              "volume_build_ms": ms_front, "export_mesh_s": s_mesh}
    return {"roofline": roofline, "stages": stages, "rays": rays}


def render_throughput(tr, sample, imgs, fmaps, cond, sizeW, sizeH, dev, pk):
    from o2345 import ops
    from o2345.sparse_sdf_network import channel_last_volume
    vol, occ = cond['dense_volume_scale0'], cond['valid_mask_volume_scale0']
    near, far = sample['query_near_far'][0, :1], sample['query_near_far'][0, 1:]
    ro = ops.cf32(sample['rays']['rays_o'][0].reshape(-1, 3))
    rd = ops.cf32(sample['rays']['rays_v'][0].reshape(-1, 3))

    def image():
        outs = []
        for a, b in zip(ro.split(CHUNK), rd.split(CHUNK)):
            o = tr.sdf_renderer_lod0.render(a, b, near, far, tr.sdf_network_lod0, tr.rendering_network_lod0,
                                            perturb_overwrite=0, background_rgb=1.0, alpha_inter_ratio=1.0, lod=0,
                                            conditional_volume=vol, conditional_valid_mask_volume=occ, feature_maps=fmaps,
                                            color_maps=imgs, w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
                                            img_wh=[sizeW, sizeH], query_c2w=sample['query_c2w'])
            outs.append(o)
        return outs
    image()
    ms_img, outs = ev_time(image)
    o = outs[0]
    # dominant kernels of the ray march, timed alone on the first KCHUNK rays (the slice round 1 reported)
    KCHUNK = 8192
    vol_cl = channel_last_volume(vol)
    pack = tr.sdf_network_lod0.sdf_layer.packed()
    mid = o['mid_z_vals'][:KCHUNK].contiguous()
    active = (o['inside_sphere'][:KCHUNK] > 0).to(torch.uint8).reshape(-1).contiguous()
    n_act = int(active.sum())
    src = ops.PointSource.rays(ro[:KCHUNK], rd[:KCHUNK], mid)
    f_sdf = lambda: ops.sdf_query(src, vol_cl, pack, active=active, want_grad=True)
    f_sdf()
    ms_sdf = float(np.mean([ev_time(f_sdf)[0] for _ in range(3)]))
    views = tr.sdf_renderer_lod0._source_views(fmaps, imgs, sample['w2cs'][0], sample['intrinsics'][0], [sizeW, sizeH])
    qc = ops.cf32(sample['query_c2w'].reshape(-1, 4, 4)[0, :3, 3])
    prec = tr.sdf_renderer_lod0.blend_precision
    f_bl = lambda: ops.render_blend(src, active, vol_cl, occ, views, tr.rendering_network_lod0.packed(), query_center=qc,
                                    precision=prec)
    f_bl()
    ms_bl = float(np.mean([ev_time(f_bl)[0] for _ in range(3)]))
    pairs = int(f_bl()[1].sum())
    f_bl32 = lambda: ops.render_blend(src, active, vol_cl, occ, views, tr.rendering_network_lod0.packed(), query_center=qc,
                                      precision=0)
    rgb32 = f_bl32()[0]
    ms_bl32 = float(np.mean([ev_time(f_bl32)[0] for _ in range(2)]))
    drift = float((f_bl()[0] - rgb32).abs().max())
    t_roof = max(RAY_FLOP / (pk["bf16_tflops"] * 1e12), RAY_GATHER_BYTES / (pk["hbm_gbs"] * 1e9)) * N_RAYS
    return {"metric": "volume-render M rays/sec", "value": N_RAYS / (ms_img * 1e-3) / 1e6, "unit": "M rays/s",
            "workload": "65536 rays x (64+64) samples x 32 views, volume + feature maps resident; SDF MLP split-fp16 tensor cores (fp32-grade), view-blending "
                        "MLPs on tensor cores (fp16 operands, fp32 accumulate / statistics)",
            "image_ms": ms_img, "frac_of_survey_contract": t_roof * 1e3 / ms_img,
            "chunk_rays": CHUNK, "kernels_first_8192_rays": {
                "sdf_query_kernel<grad>": {"ms": ms_sdf, "tflops": n_act * (FLOP_SDF_FWD + FLOP_SDF_BWD) / (ms_sdf * 1e-3) / 1e12,
                                           "active_samples": n_act},
                "render_blend_tc_kernel (mma.sync, default)" if prec == 1 else "render_blend_kernel precision %d" % prec: {"ms": ms_bl, "valid_pairs": pairs, "ms_fp32_kernel": ms_bl32,
                                           "max_colour_drift_vs_fp32_kernel": drift,
                                        "gather_gbs": (pairs * 960 + n_act * 544) / (ms_bl * 1e-3) / 1e9}}}


DUMP_ROWS = 1 << 16        # rows kept of a row array (mesh vertices, triangles, colours)
DUMP_ELEMENTS = 1 << 20    # elements kept of a grid (the SDF field)


def dump_outputs(out_dir, outputs):
    """Every array of `outputs` as out_dir/<name>.npy, float32 where that is exact (fp32 data, integers below 2^24), float64
    otherwise, with a FIXED shape.  Runs of one build are bit-identical, but a mesh's size follows the last bits of the views
    it was reconstructed from (125 stochastic DDIM steps amplify them), so two builds that round differently give meshes of
    different sizes; to compare them array by array, each array is a fixed, seeded sample -- DUMP_ROWS rows of a row array,
    DUMP_ELEMENTS elements of a grid -- taken at the same relative positions (rows in marching-cubes lattice order), with
    the sampled indices in out_dir/<name>_index.npy.  About 20 MB in all."""
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(0)
    for name, v in sorted(outputs.items()):
        v = v.detach().cpu().numpy() if torch.is_tensor(v) else v
        if not isinstance(v, np.ndarray):
            continue
        exact32 = (v.dtype.kind == "f" and v.itemsize <= 4) or (v.dtype.kind in "iub" and (v.size == 0 or np.abs(v).max() < 2 ** 24))
        rows = v.reshape(len(v), -1) if v.ndim == 2 else v.reshape(-1)
        pos = np.sort(rng.random(DUMP_ROWS if v.ndim == 2 else DUMP_ELEMENTS))
        idx = np.minimum((pos * len(rows)).astype(np.int64), max(len(rows) - 1, 0))
        out = rows[idx] if len(rows) else rows
        np.save(os.path.join(out_dir, name + ".npy"), out.astype(np.float32 if exact32 else np.float64))
        np.save(os.path.join(out_dir, name + "_index.npy"), idx.astype(np.float64))
        beat("dump: %s %s of %s" % (name, out.shape, v.shape))


def host_threads():
    """Threads for the CPU arm: every core up to 32 (the torch-CPU port stops scaling beyond that; the count actually
    used is what the JSON reports as `cores`)."""
    return max(1, min(os.cpu_count() or 1, 32))


class CpuPort:
    """The reference's own algorithm on the host cores (oracle/ port, fp32): bounded samples of every stage of one mesh,
    extrapolated to the full workload.  A path-A sample is 1 UNet iteration at batch 8 (x544 per mesh) + 1 VAE decode of
    one latent (x40) + 1 VAE encode (x10) + 1 CLIP image embedding (x10); a reconstruction sample is the full 96^3 volume
    build + a 48^3 SDF grid (scaled to 256^3 by the point count) + marching cubes on it (scaled by the cell count) + the
    colours of 2048 mesh vertices (scaled to the mesh's vertex count, estimated from the 48^3 mesh x (256/48)^2).
    bench.py is the one place outside tests/ allowed to execute oracle/ (as the CPU baseline, never as the product)."""

    def __init__(self):
        from helpers import states_torch
        from o2345 import synthetic as S
        torch.set_num_threads(host_threads())
        t = lambda x: torch.from_numpy(np.asarray(x)).float()
        w0 = time.perf_counter()
        self.sd_u = {k: torch.from_numpy(v) for k, v in S.unet_state(0).items()}
        self.sd_v = {k: torch.from_numpy(v) for k, v in S.vae_state(10).items()}
        self.sd_c = {k: torch.from_numpy(v) for k, v in S.clip_state(20).items()}
        self.st = states_torch(0)
        cams = S.scene_cameras(S.pose_json(60.0), n_src=N_VIEWS, img_wh=(W, H))
        self.imgs = torch.from_numpy(S.images(N_VIEWS + 1, H, W, seed=1234))[1:]
        self.origin, self.proj = t(cams["partial_vol_origin"]), t(cams["affine_mats"])
        self.w2cs, self.intr = t(cams["w2cs"]), t(cams["intrinsics"])
        self.t_setup = time.perf_counter() - w0
        self.g = torch.Generator().manual_seed(0)
        self.a, self.r = [], []          # per-sample stage times

    @staticmethod
    def _clock(fn):
        w0 = time.perf_counter()
        out = fn()
        return time.perf_counter() - w0, out

    @torch.no_grad()
    def path_a_sample(self, record=True):
        from oracle import clip_oracle as CO, ldm_oracle as LO, vae_oracle as VO
        g = self.g
        t_unet, _ = self._clock(lambda: LO.unet_forward(self.sd_u, torch.randn(8, 8, 32, 32, generator=g), torch.full((8,), 501),
                                                        torch.randn(8, 1, 768, generator=g)))
        t_dec, _ = self._clock(lambda: VO.decode(self.sd_v, torch.randn(1, 4, 32, 32, generator=g)))
        t_enc, _ = self._clock(lambda: VO.encode_moments(self.sd_v, torch.rand(1, 3, 256, 256, generator=g) * 2 - 1))
        t_clip, _ = self._clock(lambda: CO.embed(self.sd_c, torch.rand(1, 3, 256, 256, generator=g) * 2 - 1))
        if record:
            self.a.append((t_unet, t_dec, t_enc, t_clip))
        return t_unet + t_dec + t_enc + t_clip

    @torch.no_grad()
    def recon_sample(self, record=True):
        from oracle import recon_oracle as O
        st = self.st

        def volume():
            fm = O.pyramid_feature_maps(self.imgs, st["pyramid_feature_network"])
            return fm, O.conditional_volume(fm, self.origin, self.proj, st["sdf_network_lod0"], VOL, 2.0 / (VOL - 1), H, W)
        t_vol, (fm, cv) = self._clock(volume)
        t_grid, u = self._clock(lambda: O.sdf_grid(cv["dense"], st["sdf_network_lod0"], 48))
        t_mc, (v, tri, _) = self._clock(lambda: O.marching_cubes(u, 0.0))
        nv = max(len(v), 1)
        pts = torch.from_numpy(v[np.linspace(0, nv - 1, 2048).astype(np.int64)] / 47.0 * 2 - 1).float() if len(v) else \
            torch.zeros(2048, 3)
        t_col, _ = self._clock(lambda: O.vertex_colors(pts, cv["dense"], cv["occ"], fm, self.imgs, self.w2cs, self.intr,
                                                       st["sdf_network_lod0"], st["rendering_network_lod0"], W=W, H=H))
        k = MESH_RES / 48.0
        row = (t_vol, t_grid * k ** 3, t_mc * k ** 3, t_col * (nv * k ** 2) / 2048.0)
        if record:
            self.r.append(row)
        return t_vol + t_grid + t_mc + t_col

    def result(self):
        med = lambda rows, i: float(np.median([r[i] for r in rows]))
        tu, td, te, tc = (med(self.a, i) for i in range(4))
        tv, tg, tm, tcol = (med(self.r, i) for i in range(4))
        total = UNET_ITERS * tu + 40 * td + 10 * te + 10 * tc + tv + tg + tm + tcol
        return {"value": total, "unit": "s/mesh", "cores": torch.get_num_threads(), "kind": "port",
                "sample": f"median of {len(self.a)} path-A samples after 1 warm-up: 1 UNet iteration at batch 8 ({tu:.2f} s, x{UNET_ITERS}) + "
                          f"1 VAE decode ({td:.2f} s, x40) + 1 VAE encode ({te:.2f} s, x10) + 1 CLIP image embedding ({tc:.2f} s, x10); "
                          f"median of {len(self.r)} reconstruction samples: full 96^3 volume build ({tv:.1f} s) + 48^3 SDF grid scaled to "
                          f"256^3 ({tg:.0f} s) + marching cubes scaled by cells ({tm:.1f} s) + vertex colours scaled from 2048 vertices "
                          f"({tcol:.1f} s); weights generated in {self.t_setup:.0f} s (untimed)",
                "stages_s": {"unet_iteration": tu, "vae_decode": td, "vae_encode": te, "clip_embed": tc, "volume_build": tv,
                             "sdf_grid_256": tg, "marching_cubes_256": tm, "vertex_colours": tcol}}


def cpu_reference(n_a=3, n_recon=1, warm=True):
    """`cpu_baseline`: 1 warm-up + n_a timed path-A samples, n_recon reconstruction samples (about 30-60 s of host work)."""
    port = CpuPort()
    if warm:
        port.path_a_sample(record=False)
    for _ in range(n_a):
        port.path_a_sample()
    for _ in range(n_recon):
        port.recon_sample()
    return port.result()


def run_reference(args):
    """--impl reference: the CPU port of the reference (oracle/) on the host cores, same metric and config.  A step is one
    bounded sample of the workload: a path-A sample every step; a reconstruction sample on the first warm-up step and on
    (at most) the first 3 timed steps -- W + K steps end within a few minutes.  value = the mesh time extrapolated from
    the medians of the timed samples."""
    if int(os.environ.get("RANK", 0)) != 0:
        return
    for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS"):
        if os.environ.get(k) == "1":         # torchrun's default for its workers; this arm owns the host
            beat("note: %s=1 in the environment; torch.set_num_threads(%d) overrides it for this arm" % (k, host_threads()))
    port = CpuPort()
    beat("reference arm: weights ready (%.0f s), %d threads" % (port.t_setup, torch.get_num_threads()))
    for i in range(args.warmup):
        dt = port.path_a_sample(record=False) + (port.recon_sample(record=False) if i == 0 else 0.0)
        beat("reference warm-up sample %d: %.1f s" % (i, dt))
    w0 = time.perf_counter()
    for i in range(args.steps):
        dt = port.path_a_sample() + (port.recon_sample() if i < 3 else 0.0)
        beat("reference timed sample %d: %.1f s" % (i, dt))
    wall = time.perf_counter() - w0
    cb = port.result()
    cb["timed_samples_wall_s"] = wall
    emit(json.dumps({"impl": "reference", "metric": "sec/mesh end-to-end (256x256 in)", "value": cb["value"], "unit": "s/mesh",
                      "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["value"] * 1e3,
                      "higher_is_better": False, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                      "config": CONFIG, "cpu_baseline": cb,
                      "note": "value is one mesh extrapolated from bounded samples (see cpu_baseline.sample); the K timed samples "
                              "took %.0f s of wall clock" % wall,
                      "e2e": {"value": cb["value"], "unit": "s/mesh", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


_JSON_OUT = None


def emit(line):
    """The ONE JSON line goes to the process's original stdout; everything else printed to fd 1 (NCCL's version banner,
    library chatter) has been re-routed to stderr by main()."""
    out = _JSON_OUT if _JSON_OUT is not None else sys.stdout
    out.write(line + "\n")
    out.flush()


def main():
    global _JSON_OUT
    sys.stdout.flush()
    _JSON_OUT = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="o2345", choices=["o2345", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write fixed-shape seeded samples of the arrays the last timed step computed to DIR/<name>.npy")
    ap.add_argument("--cpu-baseline-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.cpu_baseline_child:      # child of CpuBaselineJob: the port's result as one JSON line on stdout
        return emit(json.dumps(cpu_reference()))
    if args.impl == "reference":
        return run_reference(args)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the o2345 path has no CPU fallback")
    run_gpu(args)


if __name__ == "__main__":
    main()
