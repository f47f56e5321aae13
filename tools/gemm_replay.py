"""Device time of all GEMM / implicit-conv launches of one UNet forward (CFG batch 8) replayed back to back in one CUDA
graph -- the conditions of the live UNet graph (activations L2-resident, weights streaming, PDL chaining) -- under a list
of tile-configuration settings: forced (ctas, bn, splits) and alternative cost-model constants."""
import ctypes as C
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from o2345 import _lib as L, ops_a as A
from o2345.unet import UNetModel
lib = L.load()
net = UNetModel().cuda().requires_grad_(False)
net.use_cuda_graph = False
BATCH = int(os.environ.get("UNET_BATCH", "8"))
x = torch.randn(BATCH, 8, 32, 32, device="cuda"); t = torch.full((BATCH,), 501, device="cuda"); ctx = torch.randn(BATCH, 1, 768, device="cuda")
net(x, t, ctx); torch.cuda.synchronize()
rec = []
real = {n: getattr(A, n) for n in ("gemm", "conv3x3")}
def spy(name):
    def wrap(*a, **k):
        rec.append((name, a, k)); return real[name](*a, **k)
    return wrap
for n in real: setattr(A, n, spy(n))
net(x, t, ctx); torch.cuda.synchronize()
for n in real: setattr(A, n, real[n])
side = torch.cuda.Stream()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
def replay_ms():
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        for name, a, k in rec: real[name](*a, **k)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=side):
            for name, a, k in rec: real[name](*a, **k)
    g.replay(); torch.cuda.synchronize()
    ts = []
    for _ in range(7):
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))
# cuBLAS on the same shapes (implicit convs as plain [M, 9C] x [N, 9C]^T products), same back-to-back protocol
shapes = []
for name, a, k in rec:
    if name == "gemm":
        shapes.append((a[0].shape[0], a[1].shape[0], a[0].shape[1]))
    else:
        B_, H_, W_, C_ = a[1:5]
        shapes.append((B_ * H_ * W_, a[5].shape[0], 9 * C_))
ops = {}
for (M, N, K) in set(shapes):
    ops[(M, N, K)] = (torch.randn(M, K, device="cuda", dtype=torch.float16), torch.randn(N, K, device="cuda", dtype=torch.float16),
                      torch.empty(M, N, device="cuda", dtype=torch.float16))
def lib_pass():
    for sh in shapes:
        ta, tb, to = ops[sh]
        torch.matmul(ta, tb.t(), out=to)
g = torch.cuda.CUDAGraph()
with torch.cuda.stream(side):
    lib_pass(); torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=side):
        lib_pass()
g.replay(); torch.cuda.synchronize()
ts = []
for _ in range(7):
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
print("cuBLAS, same %d shapes back to back: %.3f ms (no bias / residual / GEGLU epilogues, distinct operands per shape only)" % (len(shapes), float(np.median(ts))))
del g, ops
DEF = [40, 0.5, 6300, 5, 3, 4, 1]
def model(v): lib.o2345_debug_gemm_model((C.c_float * 7)(*v))
print("%d launches" % len(rec))
CASES = [("default", (0, 0, 0), DEF, (0, 0)), ("never persistent", (0, 0, 0), DEF, (2, 0)), ("persistent everywhere", (0, 0, 0), DEF, (1, 0)),
         ("persistent >= 74 tiles", (0, 0, 0), DEF, (0, 74)), ("persistent >= 296 tiles", (0, 0, 0), DEF, (0, 296)),
         ("persistent >= 592 tiles", (0, 0, 0), DEF, (0, 592)), ("default again", (0, 0, 0), DEF, (0, 0))]
# one graph per case (the kernel choice is frozen at capture), then the cases are timed in turn, round after round, so that
# clock / power drift over the run hits all of them alike
def capture():
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        for name, a, k in rec: real[name](*a, **k)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=side):
            for name, a, k in rec: real[name](*a, **k)
    g.replay(); torch.cuda.synchronize()
    return g
graphs = []
for label, force, mv, pers in CASES:
    lib.o2345_debug_gemm_force(*force); model(mv); lib.o2345_debug_gemm_persist(*pers)
    graphs.append((label, capture(), []))
lib.o2345_debug_gemm_persist(0, 0)
lib.o2345_debug_gemm_force(0, 0, 0); model(DEF)
for rnd in range(6):
    for label, g, ts in graphs:
        for _ in range(3):
            e0.record(); g.replay(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
for label, g, ts in graphs:
    print("%-30s %.3f ms (min %.3f)" % (label, float(np.median(ts)), min(ts)), flush=True)
