"""Tile-configuration sweep of the wgmma GEMM over every distinct GEMM / implicit-conv shape of one UNet forward
(CFG batch 8): for each shape, the device time of the heuristic's choice, of every forced (ctas, bn, splits) candidate
(o2345_debug_gemm_force) and of cuBLAS on the same shape, all under the protocol the captured UNet graph runs under
(cold L2, no host launch gaps): a CUDA graph of REPS x (L2 flush, call) minus a graph of REPS flushes.

    python tools/gemm_sweep.py [--quick] > gpurun_out/gemm_sweep.txt
"""
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import torch
from o2345 import _lib as L
from o2345.unet import UNetModel
import o2345.ops_a as A

QUICK = "--quick" in sys.argv
REPS = 6
lib = L.load()
net = UNetModel().cuda().requires_grad_(False)
net.use_cuda_graph = False
BATCH = int(os.environ.get("UNET_BATCH", "8"))
x = torch.randn(BATCH, 8, 32, 32, device="cuda")
t = torch.full((BATCH,), 501, device="cuda")
ctx = torch.randn(BATCH, 1, 768, device="cuda")
net(x, t, ctx)
torch.cuda.synchronize()

rec = []
_gemm, _conv = A.gemm, A.conv3x3


def spy_gemm(*a, **k):
    rec.append(("gemm", _gemm, a, k))
    return _gemm(*a, **k)


def spy_conv(*a, **k):
    rec.append(("conv", _conv, a, k))
    return _conv(*a, **k)


A.gemm, A.conv3x3 = spy_gemm, spy_conv
keep = net(x, t, ctx)
torch.cuda.synchronize()
A.gemm, A.conv3x3 = _gemm, _conv


def key(kind, a, k):
    rb, res, act = int(k.get("rowbias") is not None), int(k.get("residual") is not None), int(k.get("act", 0))
    if kind == "gemm":
        return ("gemm", a[0].shape[0], a[1].shape[0], a[0].shape[1], rb, res, act)
    B, H, W, C = a[1:5]
    return ("conv", B * H * W, a[5].shape[0], 9 * C, rb, res, act)


groups = collections.OrderedDict()
for kind, fn, a, k in rec:
    groups.setdefault(key(kind, a, k), []).append((fn, a, k))

flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")   # 256 MB > L2
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
side = torch.cuda.Stream()


def graph_ms(fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=side):
            for _ in range(REPS):
                flush.zero_()
                fn()
    ts = []
    for _ in range(3):
        torch.cuda.synchronize()
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[1] / REPS


base = graph_ms(lambda: None)
tot_h = tot_best = tot_lib = 0.0
rows = []
for k, calls in groups.items():
    fn, a, kw = calls[0]
    kind, M, N, K, rb, res, act = k
    nk = (K + 63) // 64
    lib.o2345_debug_gemm_force(0, 0, 0)
    t_h = max(graph_ms(lambda: fn(*a, **kw)) - base, 1e-4)
    cands = []
    for ctas in (1,):
        for bn in (64, 128, 160, 256):
            if bn > 64 and N <= 64:
                continue
            if act == 3 and N % bn:
                continue
            for sp in (1, 2, 3, 4, 6, 8):
                if sp > 1 and (act == 3 or nk // sp < 3):
                    continue
                mblocks = (M + 127) // 128
                tiles = mblocks * ((N + bn - 1) // bn)
                if sp > 1 and tiles * sp > 700:
                    continue
                if QUICK and sp not in (1, 2, 4, 8):
                    continue
                cands.append((ctas, bn, sp))
    best = (t_h, "heur")
    res_c = {}
    for c in cands:
        lib.o2345_debug_gemm_force(*c)
        try:
            tc = max(graph_ms(lambda: fn(*a, **kw)) - base, 1e-4)
        except Exception as ex:   # a forced config the entry point refuses
            res_c["%d,%d,%d" % c] = None
            continue
        res_c["%d,%d,%d" % c] = round(tc * 1e3, 2)
        if tc < best[0]:
            best = (tc, "%d,%d,%d" % c)
    lib.o2345_debug_gemm_force(0, 0, 0)
    ta = torch.randn(M, K, device="cuda", dtype=torch.float16)
    tb = torch.randn(N, K, device="cuda", dtype=torch.float16)
    to = torch.empty(M, N, device="cuda", dtype=torch.float16)
    t_lib = max(graph_ms(lambda: torch.matmul(ta, tb.t(), out=to)) - base, 1e-4)
    del ta, tb, to
    n = len(calls)
    tot_h += t_h * n
    tot_best += best[0] * n
    tot_lib += t_lib * n
    rows.append({"kind": kind, "M": M, "N": N, "K": K, "rowbias": rb, "res": res, "act": act, "n": n, "heur_us": round(t_h * 1e3, 2),
                 "best_us": round(best[0] * 1e3, 2), "best": best[1], "lib_us": round(t_lib * 1e3, 2), "cands": res_c})
    print(json.dumps(rows[-1]), flush=True)
print(json.dumps({"total_heuristic_ms": tot_h, "total_best_ms": tot_best, "total_cublas_ms": tot_lib, "flush_us": base * 1e3,
                  "calls": len(rec), "shapes": len(rows)}))
