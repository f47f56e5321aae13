"""Device time of the captured UNet graph under a list of knob settings, all in ONE process on ONE GPU, the graphs of the
cases replayed in turn round after round (box-to-box and over-the-run drift is larger than most of the effects):
    python tools/unet_ab.py [batch ...]           (default 16 64)
Knobs: the persistent GEMM variant (o2345_debug_gemm_persist), the GroupNorm cluster size (o2345_debug_groupnorm_cluster),
the one-kernel GroupNorm (net.gn_one_kernel)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from o2345 import _lib, ops_a
from o2345.unet import UNetModel
lib = _lib.load()
net = UNetModel().cuda().requires_grad_(False)
CASES = [("default", {}), ("up-sampling convs by gather", {"up2x": False}), ("GEMM never persistent", {"persist": (2, 0)}),
         ("GroupNorm clusters of 8", {"gn_cl": 8}), ("default again", {})]
if os.environ.get("UNET_AB_CASES"):
    CASES = eval(os.environ["UNET_AB_CASES"])
for B in [int(a) for a in sys.argv[1:]] or [16, 64]:
    x = torch.randn(B, 8, 32, 32, device="cuda"); t = torch.full((B,), 501, device="cuda"); ctx = torch.randn(B, 1, 768, device="cuda")
    graphs = []
    for label, knobs in CASES:
        lib.o2345_debug_gemm_persist(*knobs.get("persist", (0, 0)))
        lib.o2345_debug_groupnorm_cluster(knobs.get("gn_cl", 0))
        lib.o2345_debug_gemm_force(*knobs.get("force", (0, 0, 0)))
        net.gn_one_kernel = knobs.get("gn_one", True)
        ops_a.USE_CONV_UP2X = knobs.get("up2x", True)
        net._graphs.clear()
        for _ in range(2):
            net(x, t, ctx)
        torch.cuda.synchronize()
        graphs.append((label, net._graphs[next(iter(net._graphs))], []))
    lib.o2345_debug_gemm_persist(0, 0); lib.o2345_debug_groupnorm_cluster(0); lib.o2345_debug_gemm_force(0, 0, 0); net.gn_one_kernel = True; ops_a.USE_CONV_UP2X = True
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(6):
        for label, g, ts in graphs:
            a.record()
            for _ in range(5):
                g[0].replay()
            b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) / 5)
    for label, g, ts in graphs:
        print("batch %3d  %-28s %.3f ms (min %.3f)  kernels %d" % (B, label, float(np.median(ts)), min(ts), g[5]), flush=True)
