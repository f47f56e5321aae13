"""Is the GEMM main loop bound by the L2 -> SM fabric or by what one SM can take in?

One-wave scaling of the top UNet conv shape and of the plain GEMM with the same K, at BN = 160 and no split (forced), per-tile
launch: 32, 64 and 128 tiles, each inside one wave of 132 SMs.  If the aggregate fabric is the bound, the time of a wave grows
with the number of CTAs pulling at once; if one SM's ingest (or latency) is the bound, it stays flat and each k-block costs
more than the 4 * BN = 640 tensor cycles.  Per case:
  * device time per call, warm L2 (a CUDA graph of REPS back-to-back calls) and cold L2 (REPS x (256 MB flush, call) minus a
    graph of the flushes), and the same in SM cycles at the clock read during the run;
  * the phase stamps of CTA (0,0,0) (o2345_debug_gemm_trace, SM cycles): main loop per k-block (first operands landed -> last
    MMA done, over nk - 1), and the epilogue (last MMA -> epilogue done).
Also prints the card, its power limit and the SM clock under this load.

    python tools/gemm_wave.py
"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import torch
from o2345 import _lib as L
import o2345.ops_a as A

REPS = 20
BN = 160
lib = L.load()


def smi(q):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
side = torch.cuda.Stream()


def graph_ms(fn, cold, hold_s=0.0):
    """Device ms per call; with hold_s > 0 the graph keeps replaying for that long afterwards while the SM clock is read."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=side):
            for _ in range(REPS):
                if cold:
                    flush.zero_()
                fn()
    ts = []
    for _ in range(5):
        torch.cuda.synchronize()
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[2]
    if hold_s > 0:
        n = max(1, int(hold_s * 1e3 / ms))
        for _ in range(n):
            g.replay()
        clocks.append(smi("clocks.sm,clocks_throttle_reasons.active"))   # read while the queued replays run
        torch.cuda.synchronize()
    return ms / REPS


buf = torch.zeros(32, dtype=torch.int64, device="cuda")


def trace(fn):
    fn()
    torch.cuda.synchronize()
    buf.zero_()
    lib.o2345_debug_gemm_trace(C.c_void_p(buf.data_ptr()))
    fn()
    torch.cuda.synchronize()
    lib.o2345_debug_gemm_trace(None)
    return buf.tolist()


def cases():
    for B in (2, 4, 8):
        x = torch.randn(B * 32 * 32, 320, device="cuda").half()
        w = (torch.randn(320, 9 * 320, device="cuda") * 0.02).half()
        bias = torch.randn(320, device="cuda")
        yield f"conv3x3 B={B} 32x32 C=N=320", B * 1024, 45, (lambda x=x, w=w, bias=bias, B=B: A.conv3x3(x, B, 32, 32, 320, w, bias=bias))
    for M in (2048, 4096, 8192):
        a = torch.randn(M, 2880, device="cuda").half()
        b = (torch.randn(320, 2880, device="cuda") * 0.02).half()
        bias = torch.randn(320, device="cuda")
        yield f"gemm M={M} N=320 K=2880", M, 45, (lambda a=a, b=b, bias=bias: A.gemm(a, b, bias=bias))


print("card:", smi("name,power.limit,clocks.max.sm"))
lib.o2345_debug_gemm_force(1, BN, 1)
lib.o2345_debug_gemm_persist(2, 0)       # one CTA per tile: the wave is the grid
clocks = []
for name, M, nk, fn in cases():
    tiles = (M // 128) * (320 // BN)
    warm = graph_ms(fn, False, hold_s=2.0)
    base = graph_ms(lambda: None, True)
    cold = graph_ms(fn, True) - base
    t = trace(fn)
    c = clocks[-1].split()[0]
    f = int(c) if c.isdigit() else float("nan")
    loop = (t[5] - t[4]) / (nk - 1)
    epi = t[7] - t[5]
    total = t[8] - t[0]
    per_kb_warm = warm * 1e3 * f / nk
    per_kb_cold = cold * 1e3 * f / nk
    a_b = (128 + BN) * 64 * 2
    print(f"{name}: tiles={tiles} nk={nk}  warm {warm * 1e3:.1f} us ({per_kb_warm:.0f} cyc/kblock at {f} MHz)  "
          f"cold {cold * 1e3:.1f} us ({per_kb_cold:.0f} cyc/kblock)  |  CTA(0,0,0): main loop {loop:.0f} cyc/kblock "
          f"(tensor {4 * BN}; {a_b / loop:.1f} B/clk per SM, {a_b * tiles / loop:.0f} B/clk all SMs), epilogue {epi} cyc, "
          f"CTA total {total} cyc, prologue->landed0 {t[4] - t[1]} cyc", flush=True)
lib.o2345_debug_gemm_force(0, 0, 0)
lib.o2345_debug_gemm_persist(0, 0)
print("SM clock / throttle samples during the warm runs:", "; ".join(sorted(set(clocks))))
print("card after:", smi("name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"))
