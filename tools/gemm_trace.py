"""Phase timeline of the wgmma GEMM for a few UNet shapes (o2345_debug_gemm_trace).
SM-cycle stamps (clock64) of CTA (0,0,0): entry, prologue done, first / last TMA issued, first operands landed, last MMA
issued, epi0, epilogue done, exit.  epi0 is "accumulator tile ready in shared memory" in the generic mode (fp32 output,
split-K) and "epilogue start, residual landed" in the staged fp16 modes, which work from the accumulator registers.  For split-K launches also wall-clock stamps (globaltimer, ns, relative to
the entry of CTA (0,0,0)) of tile (0,0): accumulator ready, partial stores issued (split 0); finalize start / end (the
split that wrote its stamp last: all splits finalize their share after the cluster barrier).  `total` = CUDA-event time of the launch."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import ctypes as C
import torch
from o2345 import _lib as L, ops_a as A
lib = L.load()
buf = torch.zeros(32, dtype=torch.int64, device="cuda")
names = ["entry", "prologue", "tma0", "tmaN", "landed0", "mmaN", "epi0", "epi", "exit"]
ns_names = {17: "acc", 18: "stores", 21: "fin0", 22: "fin1"}
flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
CASES = [(8192, 320, 320, 0, (0, 0, 0)), (8192, 320, 320, 1, (0, 0, 0)), (2048, 640, 640, 1, (2, 128, 1)), (2048, 640, 640, 1, (2, 128, 2)),
         (2048, 640, 640, 0, (2, 128, 2)), (512, 1280, 1280, 0, (2, 64, 2)), (8192, 320, 1280, 1, (2, 160, 2)),
         (128, 1280, 11520, 1, (1, 64, 6)), (2048, 640, 5760, 0, (2, 128, 3))]
if len(sys.argv) > 1:
    CASES = [c for c in CASES if c[4][2] > 1]
for M, N, K, res, force in CASES:
    a = torch.randn(M, K, device="cuda").half(); b = torch.randn(N, K, device="cuda").half()
    bias = torch.randn(N, device="cuda"); r = torch.randn(M, N, device="cuda").half() if res else None
    lib.o2345_debug_gemm_force(*force)
    for cold in (0, 1):
        A.gemm(a, b, bias=bias, residual=r)
        if cold: flush.zero_()
        torch.cuda.synchronize()
        buf.zero_()
        lib.o2345_debug_gemm_trace(C.c_void_p(buf.data_ptr()))
        e0.record(); A.gemm(a, b, bias=bias, residual=r); e1.record()
        torch.cuda.synchronize()
        lib.o2345_debug_gemm_trace(None)
        t = buf.tolist()
        line = f"M={M} N={N} K={K} res={res} force={force} cold={cold} total={e0.elapsed_time(e1)*1e3:.1f}us: " + \
            "  ".join(f"{n}={t[i]-t[0]}" for i, n in enumerate(names))
        if t[9]:
            line += f"  gap={t[4]-t[9]}"   # persistent launch: last MMA of the previous tile -> first operands of the last
        if force[2] > 1:
            line += "  | ns: " + "  ".join(f"{n}={t[i]-t[16]}" for i, n in ns_names.items() if t[i])
        print(line)
lib.o2345_debug_gemm_force(0, 0, 0)
# persistent launch on the batch-64 K = 320 transformer GEMM (bias + residual) and the 32 x 32 ResBlock conv: `gap` is the
# last MMA of CTA (0,0,0)'s second-to-last tile -> first operands of its last tile, in SM cycles
if len(sys.argv) == 1:
    lib.o2345_debug_gemm_persist(1, 0)
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(65536, 320, device="cuda", generator=g).half(); w = (torch.randn(320, 320, device="cuda", generator=g) * 0.05).half()
    wc = (torch.randn(320, 2880, device="cuda", generator=g) * 0.02).half()
    bias = torch.randn(320, device="cuda", generator=g); r = torch.randn(65536, 320, device="cuda", generator=g).half()
    for name, fn in (("gemm 65536x320x320 res", lambda: A.gemm(a, w, bias=bias, residual=r)),
                     ("conv 64x32x32 C=N=320 res", lambda: A.conv3x3(a, 64, 32, 32, 320, wc, bias=bias, residual=r))):
        fn(); torch.cuda.synchronize()
        buf.zero_()
        lib.o2345_debug_gemm_trace(C.c_void_p(buf.data_ptr()))
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        lib.o2345_debug_gemm_trace(None)
        t = buf.tolist()
        print(f"persistent {name}: total={e0.elapsed_time(e1)*1e3:.1f}us  " + "  ".join(f"{n}={t[i]-t[0]}" for i, n in enumerate(names)) +
              (f"  gap={t[4]-t[9]}" if t[9] else ""))
    lib.o2345_debug_gemm_persist(0, 0)
