"""Volume-rendering throughput only (the "rays" block of bench.py) without the Zero123 stages."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch
import bench
from o2345 import synthetic as S
from o2345.pipeline import build_networks, synthetic_sample
dev = torch.device("cuda:0")
tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
sample = synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W)
imgs, fmaps, cond, sizeW, sizeH = tr._conditional_features(sample)
pk = bench.peaks()
from o2345 import ops
_rb = ops.render_blend
hist = {}
def spy(*a, **k):
    r = _rb(*a, **k)
    if "h" not in hist:
        nv = r[1][r[1] > 0]
        hist["h"] = torch.bincount(nv, minlength=33).tolist()
    return r
ops.render_blend = spy
for prec in [int(a) for a in os.environ.get("BLEND_PRECISIONS", "1").split(",")]:   # 1: mma.sync kernel (default), 0: fp32 kernel
    tr.sdf_renderer_lod0.blend_precision = prec
    r = bench.render_throughput(tr, sample, imgs, fmaps, cond, sizeW, sizeH, dev, pk)
    print("precision", prec, json.dumps(r))
print("nvalid histogram (first blend call, active samples):", hist.get("h"))
