"""GPU: the reconstruction kernels (csrc/featnet.cu, costvol.cu, spconv.cu and the ray kernels of render.cu) checked one
by one against float64 references written here from the reference's definitions.

The parity tests run these kernels only in composition, on a few fixed scenes.  Here every kernel sees the shapes, tails
and edges where it could go wrong: tile tails of the 2-D convolution, views written at a channel offset, the one-pixel
fringe of the cost-volume gather, points within an ulp of a half-cell boundary, odd coarsening minima, row counts around
the sparse-conv CTA tile, and hierarchical-sampling inputs where the answer is known sample by sample.

Integer, mask, index and copy outputs are compared bit for bit.  Every float comparison states its bound beside it; the
bound is derived from the operation (first-order rounding analysis with unit roundoff U = 2^-24) and evaluated on the
data, and each test prints the largest error as a fraction of its bound."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import recon_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24              # fp32 unit roundoff
U64 = 2.0 ** -53            # fp64 unit roundoff
DEV = "cuda"
f32 = np.float32


def _L():
    from o2345 import _lib
    return _lib


def _ops():
    from o2345 import ops
    return ops


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gamma(n):
    """gamma_n = n U / (1 - n U): the relative error bound of an n-term fp32 sum / dot product."""
    return n * U / (1 - n * U)


def _assert_within(name, err, tol):
    """err <= tol everywhere; prints the largest error and the worst err / bound."""
    err, tol = err.double().cpu(), tol.double().cpu()
    if err.numel() == 0:
        print(f"{name}: nothing to compare")
        return
    assert bool(torch.isfinite(err).all()), name
    ratio = float((err / tol.clamp_min(1e-300)).max())
    print(f"{name}: max err {float(err.max()):.3e} (bound {float(tol.max()):.3e}), worst err / bound {ratio:.3f}")
    assert ratio <= 1.0, (name, ratio)


def _rng(seed):
    return np.random.default_rng(seed)


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV).contiguous()


SENTINEL = -4242.0


# ==================================================================================================== FeatureNet
CONV_CFG = [(8, 3, 1), (16, 3, 1), (32, 3, 1), (16, 5, 2), (32, 5, 2), (32, 1, 1)]
# (Cin, N, bias) per input size: every Cin at every size but 256^2, N = 32 only on the small images
CONV_CASES = {
    (1, 1): [(3, 32, True), (5, 1, False), (8, 3, True), (16, 32, False), (32, 1, True)],
    (15, 16): [(3, 3, True), (5, 32, False), (8, 1, True), (16, 3, False), (32, 1, True)],
    (17, 33): [(3, 1, False), (5, 3, True), (8, 3, False), (16, 1, True), (32, 3, True)],
    (31, 47): [(3, 3, True), (5, 1, True), (8, 1, False), (16, 3, True), (32, 1, False)],
    (256, 256): [(3, 1, True), (5, 1, False)],
}


def _conv2d(x, w, b, stride, pad, stats):
    N, Cin, H, W = x.shape
    Cout, _, K, _ = w.shape
    Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
    out = torch.full((N, Cout, Ho, Wo), SENTINEL, dtype=torch.float32, device=DEV)
    _L().call("o2345_conv2d", _ptr(x), N, Cin, H, W, _ptr(w), _ptr(b), Cout, K, stride, pad, _ptr(out), _ptr(stats),
              _stream())
    return out


@pytest.mark.parametrize("hw", list(CONV_CASES), ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("cfg", CONV_CFG, ids=lambda c: f"co{c[0]}k{c[1]}s{c[2]}")
def test_conv2d_matches_fp64(cfg, hw):
    """o2345_conv2d against fp64 F.conv2d (pad = K // 2, as FeatureNet uses).

    Output: bias plus Cin K^2 fused multiply-adds in fp32, so |y - y64| <= gamma_{Cin K^2 + 1} (|b| + sum |w| |x|), the
    sum evaluated by the same fp64 convolution on |x|, |w|, |b|.  Stats: each CTA adds its 256 outputs by a 5-level
    shuffle tree and 8 warp partials in order (13 fp32 additions deep) before the fp64 atomics, so
    |S1 - sum y64| <= sum B + 14 U sum |y| and |S2 - sum y64^2| <= sum (2|y| + B) B + 15 U sum y^2.  The stats buffer is
    filled with 1e300 before the first call and reused for a second: both must be reset by the call."""
    Cout, K, S = cfg
    H, W = hw
    pad = K // 2
    rng = _rng(Cout * 1000 + K * 100 + H)
    for Cin, N, has_bias in CONV_CASES[hw]:
        x = rng.standard_normal((N, Cin, H, W)).astype(f32)
        w = (rng.standard_normal((Cout, Cin, K, K)) / np.sqrt(Cin * K * K)).astype(f32)
        b = rng.standard_normal(Cout).astype(f32) if has_bias else None
        xd, wd, bd = _cuda(x), _cuda(w), (_cuda(b) if has_bias else None)
        stats = torch.full((2 * Cout,), 1e300, dtype=torch.float64, device=DEV)
        y = _conv2d(xd, wd, bd, S, pad, stats)
        s1 = stats.clone()
        y2 = _conv2d(xd, wd, bd, S, pad, stats)
        assert torch.equal(y, y2), "conv2d is not deterministic"
        x64, w64 = torch.from_numpy(x).double(), torch.from_numpy(w).double()
        b64 = torch.from_numpy(b).double() if has_bias else None
        ref = F.conv2d(x64, w64, b64, S, pad)
        A = F.conv2d(x64.abs(), w64.abs(), b64.abs() if has_bias else None, S, pad)
        B = _gamma(Cin * K * K + 1) * A
        yc = y.double().cpu()
        tag = f"conv2d co{Cout} k{K} s{S} cin{Cin} n{N} {H}x{W} bias={has_bias}"
        assert yc.shape == ref.shape
        _assert_within(tag, (yc - ref).abs(), B)
        cnt_s = (ref.abs().sum((0, 2, 3)), (ref ** 2).sum((0, 2, 3)))
        b_s1 = B.sum((0, 2, 3)) + 14 * U * cnt_s[0]
        b_s2 = ((2 * ref.abs() + B) * B).sum((0, 2, 3)) + 15 * U * cnt_s[1]
        for st in (s1, stats):
            st = st.cpu()
            _assert_within(tag + " sum", (st[:Cout] - ref.sum((0, 2, 3))).abs(), b_s1)
            _assert_within(tag + " sumsq", (st[Cout:] - (ref ** 2).sum((0, 2, 3))).abs(), b_s2)


def _dest(layout, N, Ctot, H, W):
    shape = (N, Ctot, H, W) if layout == "nchw" else (N, H, W, Ctot)
    return torch.full(shape, SENTINEL, dtype=torch.float32, device=DEV)


def _channels(out, layout):
    """[N, C, H, W] view of a destination in either layout."""
    return out if layout == "nchw" else out.permute(0, 3, 1, 2)


def _check_sentinel(out, layout, c0, C):
    o = _channels(out, layout).cpu()
    others = torch.cat([o[:, :c0], o[:, c0 + C:]], 1)
    assert bool((others == SENTINEL).all()), "a channel outside [c0, c0 + C) was written"


@pytest.mark.parametrize("c0", [0, 3])
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_abn_apply_matches_fp64(layout, c0):
    """o2345_abn_apply against InPlaceABN in fp64: two-pass mean / biased variance, (x - mean) / sqrt(var + eps) *
    (|gamma| + eps) + beta, leaky-ReLU 0.01, written into a channel-offset NCHW or NHWC view.

    Channels: a plain one, a negative gamma, an off-centre one (mean = 50 std), a constant one (variance 0, output beta
    exactly), a tiny-variance one with |gamma| < eps, and a wide one.  Stats are exact fp64 sums of the fp32 input.
    With s = (|gamma| + eps) / sqrt(var + eps) and t = x - mean: fp32 rounds (float)mean (U |mean|), the difference
    (U |t|), the fp64 -> fp32 scale and the three products / sums (5 U |t| s and 2 U (|y| + |beta|)); the kernel's
    one-pass fp64 variance adds at most 4 U64 (E[x^2] + mean^2), i.e. s |t| dvar / (2 (var + eps)).  Leaky-ReLU is
    1-Lipschitz and rounds once more (U |y|)."""
    rng = _rng(7 + c0)
    N, Cc, H, W = 3, 6, 7, 9
    x = rng.standard_normal((N, Cc, H, W))
    x[:, 1] *= 2.0
    x[:, 2] = 5.0 + 0.1 * x[:, 2]
    x[:, 3] = 2.5
    x[:, 4] *= 1e-3
    x[:, 5] = 1.0 + 3.0 * x[:, 5]
    x = x.astype(f32)
    gamma = np.array([1.3, -0.7, 0.9, -1.1, -2e-6, 0.4], f32)
    beta = np.array([0.1, -0.2, 0.3, 0.05, -0.4, 0.0], f32)
    eps, slope = 1e-5, 0.01
    x64 = torch.from_numpy(x).double()
    stats = torch.cat([x64.sum((0, 2, 3)), (x64 ** 2).sum((0, 2, 3))])
    out = _dest(layout, N, Cc + c0 + 2, H, W)
    ops = _ops()
    ops.abn_apply(_cuda(x), stats.to(DEV), _cuda(gamma), _cuda(beta), ops.view_of(out, layout, c0), eps=eps, slope=slope)
    _check_sentinel(out, layout, c0, Cc)
    got = _channels(out, layout)[:, c0:c0 + Cc].double().cpu()
    mean = x64.mean((0, 2, 3), keepdim=True)
    var = ((x64 - mean) ** 2).mean((0, 2, 3), keepdim=True)
    g64 = torch.from_numpy(gamma).double().view(1, -1, 1, 1)
    b64 = torch.from_numpy(beta).double().view(1, -1, 1, 1)
    s = (g64.abs() + eps) / torch.sqrt(var + eps)
    t = x64 - mean
    y = t * s + b64
    ref = torch.where(y > 0, y, y * slope)
    dvar = 4 * U64 * ((x64 ** 2).mean((0, 2, 3), keepdim=True) + mean ** 2)
    bound = s * U * (mean.abs() + 6 * t.abs()) + s * t.abs() * dvar / (2 * (var + eps)) + 2 * U * (y.abs() + b64.abs()) \
        + U * ref.abs()
    _assert_within(f"abn_apply {layout} c0={c0}", (got - ref).abs(), bound)
    assert torch.equal(got[:, 3], torch.full_like(got[:, 3], float(beta[3]))), "constant channel must give beta exactly"


def _upsample(x, factor, out, layout, c0, add):
    ops = _ops()
    ops.upsample_bilinear(x, factor, ops.view_of(out, layout, c0), add=add)


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("add", [False, True])
@pytest.mark.parametrize("factor", [1, 2, 4])
def test_upsample_bilinear_matches_fp64(factor, add, layout):
    """o2345_upsample_bilinear against fp64 F.interpolate(bilinear, align_corners=True) (+ add), into a channel-offset
    view.  Factor 1 without add is a copy and must be bit-exact.

    The kernel's source coordinate fy = fl(fl((H-1)/(Ho-1)) * h) is off by at most 2 U fy; the fractional weight is
    exact given fy and 1 - ly rounds once (U).  The interpolant is bilinear in (ly, lx) with slopes below 2 M (M the
    largest |x| of the plane), and its six products / sums round by at most 6 U M, so
    |v - v64| <= M U (4 (fx + fy) + 10) + U |v| with the add."""
    rng = _rng(factor * 10 + int(add))
    c0 = 2
    for H, W in [(2, 2), (3, 3), (5, 7), (64, 64)]:
        N, Cc = 2, 3
        x = rng.standard_normal((N, Cc, H, W)).astype(f32)
        Ho, Wo = H * factor, W * factor
        a = rng.standard_normal((N, Cc, Ho, Wo)).astype(f32) if add else None
        out = _dest(layout, N, Cc + c0 + 1, Ho, Wo)
        _upsample(_cuda(x), factor, out, layout, c0, _cuda(a) if add else None)
        _check_sentinel(out, layout, c0, Cc)
        got = _channels(out, layout)[:, c0:c0 + Cc].double().cpu()
        x64 = torch.from_numpy(x).double()
        ref = x64 if factor == 1 else F.interpolate(x64, scale_factor=factor, mode="bilinear", align_corners=True)
        if add:
            ref = ref + torch.from_numpy(a).double()
        tag = f"upsample x{factor} add={add} {layout} {H}x{W}"
        if factor == 1 and not add:
            assert torch.equal(got, x64), tag + ": a copy must be bit-exact"
            print(tag + ": bit-exact copy")
            continue
        M = x64.abs().amax((2, 3), keepdim=True)
        fy = torch.arange(Ho, dtype=torch.float64).view(1, 1, -1, 1) * (H - 1) / max(Ho - 1, 1)
        fx = torch.arange(Wo, dtype=torch.float64).view(1, 1, 1, -1) * (W - 1) / max(Wo - 1, 1)
        bound = M * U * (4 * (fx + fy) + 10) + U * ref.abs()
        _assert_within(tag, (got - ref).abs(), bound)


# ==================================================================================================== cost volume
CV_D, CV_SIZE, CV_H, CV_W = 10, 8, 6, 9         # lattice side, image size (sizeH = sizeW), feature map h x w


def _cv_views(V):
    """[V,4,4] projections (K @ w2c layout; voxel size 1, origin 0, so world = lattice index):
    0: gx = 2x/7 - 1, gy = 2y/7 - 1 exactly: voxels x = 0 / 7 land exactly on gx = -1 / +1;
    1: every voxel behind the camera (iz = -1) but inside the image;
    2: a non-finite row (inf * 0 = NaN at x = 0, inf elsewhere);
    3: perspective with iz = z/4 - 1 crossing zero (iz == 0 is clamped to 1e-6) and negative for z < 4;
    4..: near-affine views spread over the image and one to two pixels beyond it (the fringe)."""
    rng = _rng(1234)
    P = np.zeros((32, 4, 4), f32)
    P[:, 3, 3] = 1
    P[0, 0] = [1, 0, 0, 0]
    P[0, 1] = [0, 1, 0, 0]
    P[0, 2] = [0, 0, 0, 1]
    P[1, 0] = [-0.9, -0.05, 0, 0.7]
    P[1, 1] = [-0.03, -0.8, 0, 0.6]
    P[1, 2] = [0, 0, 0, -1]
    P[2, 0] = [np.inf, 0, 0, 0]
    P[2, 1] = [0, 1, 0, 0]
    P[2, 2] = [0, 0, 0, 1]
    P[3, 0] = [0.8, 0, 0.875, -7.1]
    P[3, 1] = [0, 0.6, 0.875, -6.2]
    P[3, 2] = [0, 0, 0.25, -1]
    for v in range(4, 32):
        P[v, 0] = [rng.uniform(0.8, 1.1), rng.uniform(-0.08, 0.08), 0, rng.uniform(-1.5, -0.5)]
        P[v, 1] = [rng.uniform(-0.08, 0.08), rng.uniform(0.75, 1.05), 0, rng.uniform(-2.0, -0.3)]
        P[v, 2] = [0, 0, rng.uniform(0, 0.02), 1]
    return torch.from_numpy(P[:V].copy())


def _cv_reference(feats, proj, rows, C):
    """fp64 cost rows [n, 2C] and their bounds, plus the fp32 projections of the rows' voxels."""
    V = proj.shape[0]
    coords = O.lattice_coords(CV_D)
    gx, gy, iz, mask = O.project_voxels(coords, torch.zeros(3), 1.0, proj, CV_SIZE, CV_SIZE)
    r = torch.from_numpy(rows).long()
    gx, gy, iz, m = gx[:, r].double(), gy[:, r].double(), iz[:, r].double(), mask[r]
    fin = torch.isfinite(gx) & torch.isfinite(gy)
    grid = torch.stack([torch.where(fin, gx, 10.0).clamp(-10, 10), torch.where(fin, gy, 10.0).clamp(-10, 10)], -1)
    f64 = feats.double()                                                      # [V, C, h, w]
    f = F.grid_sample(f64, grid[:, None], mode="bilinear", padding_mode="zeros", align_corners=True)[:, :, 0]
    f = f.permute(2, 0, 1)                                                    # [n, V, C]
    cnt = m.sum(1).double()
    inv = 1.0 / (cnt + 1e-5)
    mean = f.sum(1) * inv[:, None]
    e2 = (f ** 2).sum(1) * inv[:, None]
    var = e2 - mean ** 2
    # per view: |f - f64| <= M U (16 + 8 (|fx| + |fy|)) (weights from fp32 fx, fy; four fused taps), M = max |feature|
    fx = ((gx + 1) / 2 * (CV_W - 1)).t()
    fy = ((gy + 1) / 2 * (CV_H - 1)).t()
    # views with x0 < -2 or x0 > w (and so on) give exactly 0 on both sides, whatever the rounding of fx
    M = f64.abs().amax((2, 3))                                                # [V, C]
    near = fin.t() & (fx >= -2) & (fx <= CV_W) & (fy >= -2) & (fy <= CV_H)
    Bv = torch.where(near[..., None], M[None] * U * (16 + 8 * (fx.abs() + fy.abs()).nan_to_num(0, 0, 0)[..., None]),
                     torch.zeros(()))
    Bm = inv[:, None] * (Bv.sum(1) + (V + 1) * U * f.abs().sum(1)) + 3 * U * mean.abs()
    Bvar = inv[:, None] * (((2 * f.abs() + Bv) * Bv).sum(1) + (V + 5) * U * (f ** 2).sum(1)) \
        + (2 * mean.abs() + Bm) * Bm + 2 * U * mean ** 2
    proj_info = {"fx": fx, "fy": fy, "iz": iz.t(), "fin": fin.t(), "gx": gx.t(), "gy": gy.t()}
    return torch.cat([var, mean], 1), torch.cat([Bvar, Bm], 1), mask, proj_info


def _bits_of(mask):
    b = np.zeros(mask.shape[0], np.uint32)
    mk = mask.numpy().astype(np.uint32)
    for v in range(mask.shape[1]):
        b |= mk[:, v] << np.uint32(v)
    return torch.from_numpy(b.view(np.int32).copy())


def _cv_gather(feats_nhwc, proj, rows, count, max_rows, bits, C, parent, pre, entry="lod"):
    V, h, w, _ = feats_nhwc.shape
    LD = 2 * C + (16 if parent is not None else 0)
    cost = torch.full((max_rows, LD), SENTINEL, dtype=torch.float32, device=DEV)
    origin = torch.zeros(3, device=DEV)
    cnt = torch.tensor([count], dtype=torch.int32, device=DEV)
    if entry == "lod":
        _L().call("o2345_costvol_gather_lod", _ptr(feats_nhwc), C, V, h, w, CV_SIZE, CV_SIZE, _ptr(proj), _ptr(origin),
                  1.0, CV_D, _ptr(rows), _ptr(cnt), max_rows, _ptr(bits), _ptr(parent), _ptr(pre), _ptr(cost), _stream())
    else:
        _L().call("o2345_costvol_gather", _ptr(feats_nhwc), V, h, w, CV_SIZE, CV_SIZE, _ptr(proj), _ptr(origin), 1.0,
                  CV_D, _ptr(rows), _ptr(cnt), max_rows, _ptr(bits), _ptr(cost), _stream())
    return cost


@pytest.mark.parametrize("V", [1, 7, 32])
@pytest.mark.parametrize("parent", [False, True])
@pytest.mark.parametrize("C", [8, 16])
def test_costvol_gather_matches_fp64(C, parent, V):
    """o2345_costvol_gather(_lod) against fp64 grid_sample(bilinear, zeros, align_corners=True) of the fp64 feature
    maps at the fp32 (gx, gy) of project_voxels, then mean and var = E[f^2] - E[f]^2 with the count from the mask bits
    (views behind the camera or outside the image add their features but are not counted, as in the reference).

    Per view the kernel's bilinear weights come from fp32 fx = fl(fl(gx + 1) / 2 * (w - 1)) (2 U |fx| off) and
    products of fp32 differences, and four fused taps: |f - f64| <= M U (16 + 8 (|fx| + |fy|)), M the largest |feature|
    of that view and channel.  Sums over V views add (V + 1) U sum |f| and the reciprocal count 3 U |mean|; the
    variance carries the fp32 cancellation (V + 5) U E[f^2] plus the mean's error (2 |mean| + Bm) Bm.

    301 rows (not a multiple of the 64 / 128 rows of a CTA) out of a 10^3 lattice, 27 spare rows that must keep
    their sentinel, parent features copied bit-exactly, and a call with count = 0 that writes nothing."""
    rng = _rng(C * 100 + V + int(parent))
    proj = _cv_views(V)
    feats = rng.standard_normal((V, C, CV_H, CV_W)).astype(f32)
    feats[:, 0] += 3.0                                                        # an off-centre channel
    feats_t = torch.from_numpy(feats)
    count, max_rows = 301, 328
    rows = np.sort(rng.choice(CV_D ** 3, size=count, replace=False)).astype(np.int32)
    rows_pad = np.concatenate([rows, np.zeros(max_rows - count, np.int32)])
    ref, bound, mask, info = _cv_reference(feats_t, proj, rows, C)
    bits = _bits_of(mask).to(DEV)
    feats_nhwc = feats_t.permute(0, 2, 3, 1).contiguous().to(DEV)
    projd = proj.to(DEV)
    rows_d = _cuda(rows_pad)
    par = pre = None
    if parent:
        par = _cuda(rng.integers(0, 50, size=CV_D ** 3).astype(np.int32))
        pre = _cuda(rng.standard_normal((50, 16)).astype(f32))
    cost = _cv_gather(feats_nhwc, projd, rows_d, count, max_rows, bits, C, par, pre)
    tag = f"costvol_gather C={C} parent={parent} V={V}"
    got = cost[:count, :2 * C].double().cpu()
    _assert_within(tag + " var", (got[:, :C] - ref[:, :C]).abs(), bound[:, :C])
    _assert_within(tag + " mean", (got[:, C:] - ref[:, C:]).abs(), bound[:, C:])
    assert bool((cost[count:] == SENTINEL).all()), "rows at or beyond count were written"
    if parent:
        want = pre[par.long()[rows_d[:count].long()]]
        assert torch.equal(cost[:count, 2 * C:], want), "parent features must be copied bit-exactly"
    if C == 16 and not parent:
        assert torch.equal(_cv_gather(feats_nhwc, projd, rows_d, count, max_rows, bits, C, None, None, "plain"), cost)
    empty = _cv_gather(feats_nhwc, projd, rows_d, 0, max_rows, bits, C, par, pre)
    assert bool((empty == SENTINEL).all()), "count = 0 must write nothing"
    # the edges this test exists for are present among the rows
    fx, fy, fin, iz = info["fx"], info["fy"], info["fin"], info["iz"]
    x0, y0 = torch.floor(fx), torch.floor(fy)
    iny = (y0 >= -1) & (y0 <= CV_H - 1)
    inx = (x0 >= -1) & (x0 <= CV_W - 1)
    cover = {"gx = -1": (info["gx"] == -1).sum(), "gx = +1": (info["gx"] == 1).sum()}
    if V >= 7:
        cover.update({"left fringe": (fin & iny & (x0 == -1)).sum(), "right fringe": (fin & iny & (x0 == CV_W - 1)).sum(),
                      "top fringe": (fin & inx & (y0 == -1)).sum(), "bottom fringe": (fin & inx & (y0 == CV_H - 1)).sum(),
                      "behind, inside the image": (fin & inx & iny & (iz < 0)).sum(), "non-finite": (~fin).sum()})
    print(tag + " coverage: " + ", ".join(f"{k} {int(v)}" for k, v in cover.items()))
    assert all(int(v) > 0 for v in cover.values()), cover


def _half_cell_values(D):
    """fp32 coordinates within 2 ulp of every half-cell boundary ((p + 1) D - 1) / 2 = k + 1/2, k = -1 .. D - 1,
    plus +-1, the floats next to them, and points clearly outside."""
    vals = []
    for k in range(-1, D):
        c = f32((2 * k + 2) / D - 1)
        vals.append(c)
        up = dn = c
        for _ in range(2):
            up, dn = np.nextafter(up, f32(2)), np.nextafter(dn, f32(-2))
            vals += [up, dn]
    for e in (f32(-1), f32(1)):
        vals += [e, np.nextafter(e, f32(-2)), np.nextafter(e, f32(2))]
    vals += [f32(-1.5), f32(1.5), f32(-1.0 - 1.0 / D), f32(1.0 + 1.0 / D)]
    return np.array(vals, f32)


def _grid_nearest(occ, pts):
    """The reference's lookup: torch CUDA grid_sample(nearest, zeros, align_corners=False) after the xyz -> zyx flip."""
    g = torch.flip(pts.to(DEV), dims=[-1]).view(1, 1, 1, -1, 3)
    return (F.grid_sample(occ, g, mode="nearest", padding_mode="zeros", align_corners=False).view(-1) > 0).to(torch.uint8)


def _centres(D, idx):
    return ((2 * idx.astype(np.float64) + 1) / D - 1).astype(f32)


@pytest.mark.parametrize("D", [24, 96])
def test_occ_nearest_bit_exact_at_half_cells(D):
    """o2345_occ_nearest (and render.cu's copy of the lookup, through ray_midpoints' active flags) against torch CUDA
    grid_sample(nearest, align_corners=False), bit for bit.  Each axis in turn takes every fp32 value within 2 ulp of a
    half-cell boundary, +-1, the floats just outside, and points clearly outside; the other two axes sit at cell
    centres.  NaN coordinates must give 0 (grid_sample itself is not the reference there: its float -> int conversion
    of NaN is implementation-defined)."""
    ops = _ops()
    rng = _rng(D)
    occ = (torch.from_numpy(rng.random((D, D, D))) < 0.5).float().view(1, 1, D, D, D).to(DEV)
    vals = _half_cell_values(D)
    pts = []
    for a in range(3):
        p = np.stack([_centres(D, rng.integers(0, D, size=len(vals))) for _ in range(3)], 1)
        p[:, a] = vals
        pts.append(p)
    pts.append((rng.uniform(-1.2, 1.2, size=(20000, 3))).astype(f32))
    pts = np.concatenate(pts)
    ptsd = _cuda(pts)
    got = ops.occ_nearest(ops.PointSource.explicit(ptsd), occ)
    want = _grid_nearest(occ, ptsd)
    bad = int((got != want).sum())
    print(f"occ_nearest D={D}: {pts.shape[0]} explicit points, {bad} disagree with grid_sample")
    assert bad == 0
    nanp = np.tile(_centres(D, np.arange(3)), (3, 1))
    for a in range(3):
        nanp[a, a] = np.nan
    assert int(ops.occ_nearest(ops.PointSource.explicit(_cuda(nanp)), occ).sum()) == 0, "NaN points must be empty"
    # ray points: o = 0 on the ray's axis (so p = z exactly there), d = +-e_a; and oblique rays
    R = 3 * len(vals)
    o = np.zeros((R, 3), f32)
    d = np.zeros((R, 3), f32)
    zz = np.zeros(R, f32)
    for a in range(3):
        sl = slice(a * len(vals), (a + 1) * len(vals))
        for b in range(3):
            if b != a:
                o[sl, b] = _centres(D, rng.integers(0, D, size=len(vals)))
        sign = np.where(np.arange(len(vals)) % 2 == 0, 1, -1).astype(f32)
        d[sl, a] = sign
        zz[sl] = vals * sign
    o2 = rng.uniform(-1, 1, size=(500, 3)).astype(f32)
    d2 = rng.standard_normal((500, 3)).astype(f32)
    d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    z2 = rng.uniform(0, 2, size=500).astype(f32)
    o, d, zz = np.concatenate([o, o2]), np.concatenate([d, d2]), np.concatenate([zz, z2])
    z = np.stack([zz, zz], 1)                              # two equal depths: every mid-point is z itself
    p_host = o + d * zz[:, None]                           # fp32: separately rounded product and sum, as the kernels
    od, dd, zd = _cuda(o), _cuda(d), _cuda(z)
    want = _grid_nearest(occ, _cuda(p_host))
    got = ops.occ_nearest(ops.PointSource.rays(od, dd, zd), occ).view(-1, 2)
    mid, dists, active = ops.ray_midpoints(od, dd, zd, 0.0, occ)
    assert torch.equal(mid.cpu(), torch.from_numpy(z)) and bool((dists == 0).all())
    bad_r = int((got[:, 0] != want).sum() + (got[:, 1] != want).sum())
    bad_m = int((active.view(-1, 2)[:, 0] != want).sum() + (active.view(-1, 2)[:, 1] != want).sum())
    print(f"occ_nearest D={D}: {2 * len(zz)} ray points, {bad_r} disagree with grid_sample; "
          f"ray_midpoints active: {bad_m} disagree")
    assert bad_r == 0 and bad_m == 0


# ==================================================================================================== sparse conv
PATTERNS = ["single", "p02", "p50", "p86", "full", "shell", "oddmin", "faces"]


def _pattern(kind, E, seed=0):
    """Active voxels [n, 3] (int64, unique) of a lattice of side E."""
    rng = _rng(seed * 131 + E)
    c = np.stack(np.meshgrid(*[np.arange(E)] * 3, indexing="ij"), -1).reshape(-1, 3)
    if kind == "single":
        keep = np.all(c == [E // 2, E // 3, E - 1 - E // 4], 1)
    elif kind in ("p02", "p50", "p86"):
        keep = rng.random(len(c)) < {"p02": 0.02, "p50": 0.5, "p86": 0.86}[kind]
        keep[rng.integers(len(c))] = True
    elif kind == "full":
        keep = np.ones(len(c), bool)
    elif kind == "shell":
        r = np.linalg.norm(c - (E - 1) / 2, axis=1)
        keep = np.abs(r - 0.38 * E) < 0.55
    elif kind == "oddmin":
        # per-axis minimum odd on x, even (and nonzero where E allows) on y and z
        lo = np.array([3, 2, 0 if E < 8 else 4])
        inside = np.all(c >= lo, 1)
        keep = inside & (rng.random(len(c)) < 0.25)
        for a in range(3):
            cand = np.nonzero(inside & (c[:, a] == lo[a]))[0]
            keep[rng.choice(cand)] = True
    elif kind == "faces":
        face = np.any((c == 0) | (c == E - 1), 1)
        keep = face & (rng.random(len(c)) < 0.5)
        for a in range(3):
            for v in (0, E - 1):
                keep[np.nonzero((c[:, a] == v) & np.all(np.delete(c, a, 1) == E // 2, 1))[0]] = True
    else:
        raise ValueError(kind)
    xyz = torch.from_numpy(c[keep]).long()
    assert xyz.shape[0] > 0
    return xyz


def _lin(xyz, E):
    return (xyz[:, 0] * E + xyz[:, 1]) * E + xyz[:, 2]


def _level(xyz, E):
    """Host level: sorted lattice rows (ascending x*E*E + y*E + z, the torch.unique order), index lattice, sorted
    coordinates."""
    lin, order = _lin(xyz, E).sort()
    index = torch.full((E ** 3,), -1, dtype=torch.int32)
    index[lin] = torch.arange(lin.numel(), dtype=torch.int32)
    return lin.to(torch.int32), index, xyz[order]


def _coarsen_gpu(xyz, E, pad=5):
    lin, index, _ = _level(xyz, E)
    n = lin.numel()
    Ec = E // 2 + 1
    rows = torch.cat([lin, torch.zeros(pad, dtype=torch.int32)]).to(DEV)
    flags = torch.full((Ec ** 3,), 7, dtype=torch.uint8, device=DEV)
    cmin = torch.empty(3, dtype=torch.int32, device=DEV)
    cnt = torch.tensor([n], dtype=torch.int32, device=DEV)
    index_d = index.to(DEV)
    _L().call("o2345_sp_coarsen", _ptr(index_d), E, _ptr(rows), _ptr(cnt), n + pad, Ec, _ptr(flags), _ptr(cmin),
              _stream())
    f = flags.cpu()
    assert bool(((f == 0) | (f == 1)).all())
    k = torch.nonzero(f).view(-1)
    return torch.stack([k // (Ec * Ec), (k // Ec) % Ec, k % Ec], 1), Ec


def _as_set(xyz):
    return set(map(tuple, xyz.tolist()))


@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("E", [5, 13, 24, 25, 49])
def test_sp_coarsen_equals_downsample_coords(E, kind):
    """o2345_sp_coarsen against torchsparse's spdownsample rule (oracle downsample_coords), exactly, as a set of cells:
    coarse cell q exists iff a fine voxel sits at 2q + {-1,0,1}^3 and 2q >= the per-axis fine minimum.  Checked on
    two successive levels (the second in absolute units of tensor stride 2)."""
    xyz = _pattern(kind, E)
    c1, E1 = _coarsen_gpu(xyz, E)
    want1 = O.downsample_coords(xyz, 1) // 2
    assert _as_set(c1) == _as_set(want1), f"level 1 of {kind} on {E}^3"
    c2, _ = _coarsen_gpu(c1, E1)
    want2 = O.downsample_coords(want1 * 2, 2) // 4
    assert _as_set(c2) == _as_set(want2), f"level 2 of {kind} on {E}^3"
    print(f"sp_coarsen {kind} E={E}: {xyz.shape[0]} -> {c1.shape[0]} -> {c2.shape[0]} cells, exact")


SP_PAIRS = [(32, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 32), (48, 16)]
SP_CASES = [("single", 5), ("p02", 49), ("p50", 13), ("p86", 13), ("full", 5), ("shell", 25), ("oddmin", 24),
            ("faces", 13)]


def _tile_rows(cout):
    return (128 // (cout // 4)) * 4


def _sp_reference(x64, K64, fine_xyz, coarse_xyz, mode):
    """torchsparse_conv3d in fp64.  mode 0: fine -> fine; 1: fine -> coarse (stride 2); 2: coarse -> fine
    (transposed, through the map of the matching down-conv).  Coarse coordinates are in coarse lattice units."""
    z = lambda n: torch.zeros(n, 1, dtype=torch.int64)
    cf = torch.cat([fine_xyz, z(fine_xyz.shape[0])], 1)
    cc = torch.cat([coarse_xyz * 2, z(coarse_xyz.shape[0])], 1)
    if mode == 0:
        return O.torchsparse_conv3d(x64, cf, 1, K64, 1, False, {}, {})[0]
    if mode == 1:
        return O.torchsparse_conv3d(x64, cf, 1, K64, 2, False, {2: cc}, {})[0]
    km = {(1, 2): O.kernel_map(fine_xyz, coarse_xyz * 2, 1)}
    return O.torchsparse_conv3d(x64, cc, 2, K64, 2, True, {1: cf, 2: cc}, km)[0]


def _sp_conv_check(tag, cin, cout, mode, fine_xyz, Ef, coarse_xyz, Ec, seed, spare=37):
    """Runs o2345_sp_conv on one (input level, output level) pair and checks outputs, stats and untouched rows.

    Output rows: 27 Cin fused multiply-adds in fp32, |y - y64| <= gamma_{27 Cin} sum |w| |x| (the sum from the same
    fp64 conv on |x|, |w|).  Stats: per CTA, 4 rows per thread then RG row groups in order (RG + 4 fp32 additions deep)
    before the fp64 atomics: |S1 - sum y64| <= sum B + (RG + 6) U sum |y|, |S2 - sum y64^2| <= sum (2|y| + B) B +
    (RG + 7) U sum y^2."""
    rng = _rng(seed)
    lf, idx_f, fine_sorted = _level(fine_xyz, Ef)
    lc, idx_c, coarse_sorted = _level(coarse_xyz, Ec)
    if mode == 0:
        in_idx, Ein, out_rows, Eout, n_in, n_out = idx_f, Ef, lf, Ef, lf.numel(), lf.numel()
    elif mode == 1:
        in_idx, Ein, out_rows, Eout, n_in, n_out = idx_f, Ef, lc, Ec, lf.numel(), lc.numel()
    else:
        in_idx, Ein, out_rows, Eout, n_in, n_out = idx_c, Ec, lf, Ef, lc.numel(), lf.numel()
    x = rng.standard_normal((n_in, cin)).astype(f32)
    x[:, 0] += 4.0                                                            # an off-centre input channel
    k = (rng.standard_normal((27, cin, cout)) / np.sqrt(27 * cin)).astype(f32)
    max_out = n_out + spare
    out = torch.full((max_out, cout), SENTINEL, dtype=torch.float32, device=DEV)
    stats = torch.full((2 * cout,), 1e300, dtype=torch.float64, device=DEV)
    rows_d = torch.cat([out_rows, torch.zeros(spare, dtype=torch.int32)]).to(DEV)
    cnt = torch.tensor([n_out], dtype=torch.int32, device=DEV)
    xd, idx_d, kd = _cuda(x), in_idx.to(DEV), _cuda(k)      # kept alive until the launch
    _L().call("o2345_sp_conv", _ptr(xd), _ptr(idx_d), Ein, _ptr(rows_d), _ptr(cnt), max_out, Eout, mode, _ptr(kd), cin,
              cout, _ptr(out), _ptr(stats), _stream())
    x64, k64 = torch.from_numpy(x).double(), torch.from_numpy(k).double()
    ref = _sp_reference(x64, k64, fine_sorted, coarse_sorted, mode)
    A = _sp_reference(x64.abs(), k64.abs(), fine_sorted, coarse_sorted, mode)
    B = _gamma(27 * cin) * A
    got = out[:n_out].double().cpu()
    assert got.shape == ref.shape
    _assert_within(tag, (got - ref).abs(), B)
    assert bool((out[n_out:] == SENTINEL).all()), tag + ": rows at or beyond count were written"
    RG = 128 // (cout // 4)
    st = stats.cpu()
    _assert_within(tag + " sum", (st[:cout] - ref.sum(0)).abs(), B.sum(0) + (RG + 6) * U * ref.abs().sum(0))
    _assert_within(tag + " sumsq", (st[cout:] - (ref ** 2).sum(0)).abs(),
                   ((2 * ref.abs() + B) * B).sum(0) + (RG + 7) * U * (ref ** 2).sum(0))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("pair", SP_PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_sp_conv_matches_fp64(pair, mode):
    """o2345_sp_conv, every supported channel pair in modes 0 (submanifold), 1 (stride-2 down) and 2 (transposed up,
    reusing the down map), against fp64 torchsparse_conv3d on eight sparsity patterns (a single voxel, 2 / 50 / 86 %
    random, a full lattice, a thin spherical shell, an odd per-axis minimum, voxels on all six faces)."""
    cin, cout = pair
    for i, (kind, E) in enumerate(SP_CASES):
        fine = _pattern(kind, E)
        coarse = O.downsample_coords(fine, 1) // 2
        _sp_conv_check(f"sp_conv {cin}->{cout} mode {mode} {kind} E={E}", cin, cout, mode, fine, E, coarse, E // 2 + 1,
                       seed=1000 * mode + 10 * i + cin + cout)


@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("pair", [(32, 16), (16, 32), (64, 64)], ids=lambda p: f"{p[0]}-{p[1]}")
def test_sp_conv_row_tile_edges(pair, mode, delta):
    """Output row counts of TR - 1, TR and TR + 1 (TR = 128 / 64 / 32 rows per CTA for Cout = 16 / 32 / 64), with 37
    spare rows that must keep their sentinel.  The output level is an arbitrary cell set of that size; the reference
    convolution is defined for any input / output sets (the transposed one through the down map between them)."""
    cin, cout = pair
    n = _tile_rows(cout) + delta
    rng = _rng(n * 3 + mode)
    E = 13
    Ec = E // 2 + 1
    all_f = torch.from_numpy(np.stack(np.meshgrid(*[np.arange(E)] * 3, indexing="ij"), -1).reshape(-1, 3)).long()
    all_c = torch.from_numpy(np.stack(np.meshgrid(*[np.arange(Ec)] * 3, indexing="ij"), -1).reshape(-1, 3)).long()
    if mode == 0:
        fine = all_f[torch.from_numpy(rng.choice(len(all_f), n, replace=False))]
        coarse = O.downsample_coords(fine, 1) // 2
    elif mode == 1:
        fine = all_f[torch.from_numpy(rng.random(len(all_f)) < 0.5)]
        coarse = all_c[torch.from_numpy(rng.choice(len(all_c), n, replace=False))]
    else:
        fine = all_f[torch.from_numpy(rng.choice(len(all_f), n, replace=False))]
        coarse = all_c[torch.from_numpy(rng.random(len(all_c)) < 0.5)]
    _sp_conv_check(f"sp_conv {cin}->{cout} mode {mode} rows={n}", cin, cout, mode, fine, E, coarse, Ec, seed=n + mode)


@pytest.mark.parametrize("skip", [False, True])
@pytest.mark.parametrize("Cc", [16, 32, 64])
def test_sp_bn_relu_matches_fp64(Cc, skip):
    """o2345_sp_bn_relu against nn.BatchNorm1d training semantics in fp64 (biased variance, eps in the sqrt), ReLU,
    optional skip add; an off-centre channel (mean = 50 std) and a negative gamma.  Stats are exact fp64 sums.  With
    s = |gamma| / sqrt(var + eps), t = x - mean: |y - y64| <= s U (|mean| + 6 |t|) + s |t| dvar / (2 (var + eps)) +
    2 U (|y| + |beta|) (+ U |out| for the skip add), dvar = 4 U64 (E[x^2] + mean^2).  300 live rows, 33 spare rows
    untouched; the in-place call (out = x) must give the same bits."""
    rng = _rng(Cc + int(skip))
    n, spare = 300, 33
    x = rng.standard_normal((n, Cc))
    x[:, 1] = 5.0 + 0.1 * x[:, 1]
    x[:, 2] *= 3.0
    x = x.astype(f32)
    gamma = rng.uniform(0.5, 1.5, Cc).astype(f32)
    gamma[::3] *= -1
    beta = (0.2 * rng.standard_normal(Cc)).astype(f32)
    sk = rng.standard_normal((n, Cc)).astype(f32) if skip else None
    x64 = torch.from_numpy(x).double()
    stats = torch.cat([x64.sum(0), (x64 ** 2).sum(0)]).to(DEV)
    xd = torch.cat([_cuda(x), torch.full((spare, Cc), SENTINEL, device=DEV)])
    out = torch.full((n + spare, Cc), SENTINEL, dtype=torch.float32, device=DEV)
    cnt = torch.tensor([n], dtype=torch.int32, device=DEV)
    skd = torch.cat([_cuda(sk), torch.zeros(spare, Cc, device=DEV)]) if skip else None
    eps = 1e-5
    gd, bd = _cuda(gamma), _cuda(beta)
    args = lambda o: ("o2345_sp_bn_relu", _ptr(xd), _ptr(cnt), n + spare, Cc, _ptr(stats), _ptr(gd), _ptr(bd), eps,
                      _ptr(skd), _ptr(o), _stream())
    _L().call(*args(out))
    assert bool((out[n:] == SENTINEL).all()), "rows at or beyond count were written"
    mean = x64.mean(0)
    var = x64.var(0, unbiased=False)
    g64, b64 = torch.from_numpy(gamma).double(), torch.from_numpy(beta).double()
    ref = O.batchnorm_rows(x64, g64, b64, eps)
    y = ref
    ref = torch.relu(ref)
    if skip:
        ref = ref + torch.from_numpy(sk).double()
    s = g64.abs() / torch.sqrt(var + eps)
    t = x64 - mean
    dvar = 4 * U64 * ((x64 ** 2).mean(0) + mean ** 2)
    bound = s * U * (mean.abs() + 6 * t.abs()) + s * t.abs() * dvar / (2 * (var + eps)) + 2 * U * (y.abs() + b64.abs()) \
        + U * ref.abs()
    _assert_within(f"sp_bn_relu C={Cc} skip={skip}", (out[:n].double().cpu() - ref).abs(), bound)
    _L().call(*args(xd))
    assert torch.equal(xd[:n], out[:n]), "in-place call differs"


COSTREG_LAMBDA = 8.0


def _costreg_bound(feats64, xyz, sd):
    """Error bound of SparseCostRegNet on these rows, propagated block by block beside the fp64 reference.

    A worst-case bound compounds sum |w| over ten convolutions and grows past any use, so the convolutions follow the
    probabilistic model of Higham & Mary (2019): rounding errors are independent and zero-mean, so an n-term fused sum
    adds a standard deviation of at most sqrt(n) U sum |w||x|, and incoming errors propagate as variances through w^2
    and, averaged over n rows, into the BatchNorm mean and variance with a 1 / sqrt(n) factor.  The rest is taken at
    its worst and added linearly: the statistics' own RG + 6 deep fp32 summation, the normalisation's roundings, one
    rounding per skip add; ReLU is 1-Lipschitz.  The bound is COSTREG_LAMBDA = 8 standard deviations."""
    coords = torch.cat([xyz.int(), torch.zeros(xyz.shape[0], 1, dtype=torch.int32)], 1)
    st = {"cm": {}, "km": {}}

    def conv(x, c, s, k, stride, tr):
        y, c2, s2, st["cm"], st["km"] = O.torchsparse_conv3d(x, c, s, k, stride, tr, st["cm"], st["km"])
        return y, c2, s2

    def block(name, x, sx, c, s, stride=1, tr=False):
        k, g, b = sd[name + ".net.0.kernel"], sd[name + ".net.1.weight"], sd[name + ".net.1.bias"]
        cin, cout = k.shape[1], k.shape[2]
        y, c2, s2 = conv(x, c, s, k, stride, tr)
        A = conv(x.abs(), c, s, k.abs(), stride, tr)[0]
        sy = torch.sqrt(conv(sx ** 2, c, s, k ** 2, stride, tr)[0] + 27 * cin * (U * A) ** 2)
        depth = 128 // (cout // 4) + 6
        mu = y.mean(0)
        yc = y - mu
        var = (yc ** 2).mean(0)
        sig = torch.sqrt(var + 1e-5)
        n = y.shape[0]
        smu = torch.sqrt((sy ** 2).mean(0) / n) + depth * U * y.abs().mean(0)
        svar = torch.sqrt(((2 * y * sy) ** 2).mean(0) / n) + 2 * mu.abs() * smu + 2 * depth * U * (y ** 2).mean(0) \
            + 4 * U64 * ((y ** 2).mean(0) + mu ** 2)
        ssig = svar / (2 * sig)
        z = yc / sig * g + b
        sz = g.abs() / sig * (sy + smu + U * (mu.abs() + 6 * yc.abs())) + yc.abs() / sig * g.abs() * ssig / sig \
            + 2 * U * (z.abs() + b.abs())
        return torch.relu(z), sz, c2, s2

    def add(a, sa, b, sb):
        return a + b, torch.sqrt(sa ** 2 + sb ** 2) + U * (a + b).abs()

    c0, s_c0, cc0, s0 = block("conv0", feats64, torch.zeros_like(feats64), coords, 1)
    x, e, c, s = block("conv1", c0, s_c0, cc0, s0, 2)
    c2, s_c2, cc2, s2 = block("conv2", x, e, c, s)
    x, e, c, s = block("conv3", c2, s_c2, cc2, s2, 2)
    c4, s_c4, cc4, s4 = block("conv4", x, e, c, s)
    x, e, c, s = block("conv5", c4, s_c4, cc4, s4, 2)
    x, e, c, s = block("conv6", x, e, c, s)
    x, e, c, s = block("conv7", x, e, c, s, 2, True)
    x, e = add(x, e, c4, s_c4)
    x, e, c, s = block("conv9", x, e, c, s, 2, True)
    x, e = add(x, e, c2, s_c2)
    x, e, c, s = block("conv11", x, e, c, s, 2, True)
    return COSTREG_LAMBDA * add(x, e, c0, s_c0)[1]


def test_costreg_net_forward_on_shell_matches_fp64():
    """One full SparseCostRegNet.forward (coarsening, ten convolutions, BatchNorm / ReLU, skips) on a thin spherical
    shell in a 25^3 lattice -- a sparsity pattern unlike the parity scenes -- against oracle cost_reg_net run in fp64,
    within the propagated bound of _costreg_bound."""
    from o2345.sparse_sdf_network import SparseCostRegNet
    from o2345.synthetic import costreg_channels
    ops = _ops()
    E, d_in, d_out = 25, 32, 16
    rng = _rng(25)
    xyz = _pattern("shell", E)
    lin, _, xyz_sorted = _level(xyz, E)
    sd = {}
    for name, cin, cout in costreg_channels(d_in, d_out):
        sd[name + ".net.0.kernel"] = torch.from_numpy((rng.standard_normal((27, cin, cout)) / np.sqrt(27 * cin)).astype(f32))
        g = rng.uniform(0.5, 1.5, cout).astype(f32)
        g[::4] *= -1
        sd[name + ".net.1.weight"] = torch.from_numpy(g)
        sd[name + ".net.1.bias"] = torch.from_numpy((0.1 * rng.standard_normal(cout)).astype(f32))
    net = SparseCostRegNet(d_in, d_out)
    net.load_state_dict(sd, strict=False)
    net = net.to(DEV)
    feats = rng.standard_normal((lin.numel(), d_in)).astype(f32)
    flags = torch.zeros(E ** 3, dtype=torch.uint8)
    flags[lin.long()] = 1
    rows, index, count = ops.compact(flags.to(DEV))
    assert int(count.item()) == lin.numel() and torch.equal(rows[:lin.numel()].cpu(), lin)
    level0 = ops.SparseLevel(E, rows, index, count, E ** 3)
    got = net(_cuda(feats), level0)[:lin.numel()].double().cpu()
    sd64 = {k: v.double() for k, v in sd.items()}
    f64 = torch.from_numpy(feats).double()
    ref = O.cost_reg_net(f64, xyz_sorted, sd64, prefix="")
    bound = _costreg_bound(f64, xyz_sorted, sd64)
    _assert_within(f"SparseCostRegNet shell E={E} ({lin.numel()} voxels)", (got - ref).abs(), bound)


# ==================================================================================================== ray kernels
RAY_D = 96                     # occupancy side of the ray tests: 96 cells along each ray


def _ray_layout(R, S, seed):
    """Rays along +x at cell-centre (y, z) columns, one column each; S depths per ray placed in the middle 60 % of
    the cells (never within 0.2 cell of a boundary, so the occupancy of every sample is unambiguous).  Returns rays_o,
    rays_d, z [R, S] and the x-cell of every sample."""
    D = RAY_D
    h = 2.0 / D
    k = np.arange(S)
    cell = k * D // S
    first = np.searchsorted(cell, cell, side="left")
    ncell = np.bincount(cell, minlength=D)[cell]
    off = (-0.3 + 0.6 * (k - first + 0.5) / ncell) * h
    x = (2 * cell + 1) / D - 1 + off                    # sample x in [-1, 1]
    z = np.tile((x + 1).astype(f32), (R, 1))          # o_x = -1: p_x = fl(z - 1) ~ x
    col = np.arange(R)
    o = np.stack([np.full(R, -1.0), _centres(D, col % D), _centres(D, (col // D) % D)], 1).astype(f32)
    d = np.tile(np.array([1, 0, 0], f32), (R, 1))
    return o, d, z, np.tile(cell, (R, 1))


PROFILES = ["one crossing", "crossing in the first section", "crossing in the last section", "all positive",
            "all negative", "several crossings", "constant"]
OCC_PATTERNS = ["occupied", "empty", "blocks"]


def _ray_scene(R, S, seed):
    """Rays, depths, SDF profiles (ray r: PROFILES[r % 7]), occupancy (OCC_PATTERNS[(r // 7) % 3] along the ray's
    column) and the per-sample occupancy the nearest lookup must find."""
    rng = _rng(seed)
    o, d, z, cell = _ray_layout(R, S, seed)
    D = RAY_D
    occ = np.zeros((D, D, D), f32)
    m = np.zeros((R, S), f32)
    sdf = np.zeros((R, S), f32)
    for r in range(R):
        pat = OCC_PATTERNS[(r // 7) % 3]
        colocc = {"occupied": np.ones(D), "empty": np.zeros(D), "blocks": ((np.arange(D) // 8) % 2 == 0)}[pat]
        occ[:, r % D, (r // D) % D] = colocc
        m[r] = colocc[cell[r]]
        zr = z[r].astype(np.float64)
        prof = PROFILES[r % 7]
        if prof == "one crossing":
            j = S // 2 - 1 if S > 2 else 0
            zc = zr[j] + rng.uniform(0.2, 0.8) * (zr[j + 1] - zr[j])
            s = zc - zr
        elif prof == "crossing in the first section":
            s = zr[0] + rng.uniform(0.2, 0.8) * (zr[1] - zr[0]) - zr
        elif prof == "crossing in the last section":
            s = zr[-2] + rng.uniform(0.2, 0.8) * (zr[-1] - zr[-2]) - zr
        elif prof == "all positive":
            s = 0.3 + 0.1 * np.sin(5 * zr + r)
        elif prof == "all negative":
            s = -0.3 - 0.1 * np.sin(5 * zr + r)
        elif prof == "several crossings":
            s = 0.05 * np.sin(2 * np.pi * 3 * zr + r)
        else:
            s = np.full(S, 0.02)
        sdf[r] = s
    return o, d, z, sdf, occ, m


def _sig_err(x, dx):
    """sigmoid(x) and its fp32 error bound given |dx| on the argument: sigma' dx + 4 U sigma (expf, add, divide), plus
    2^-126 for results below the normal range (expf(-x) overflows for x < -88.7 and the kernel returns exactly 0)."""
    p = torch.sigmoid(x)
    return p, p * (1 - p) * dx + 4 * U * p + 2.0 ** -126


def _alpha_err(xp, dxp, xn, dxn, m):
    """alpha = m (pc - nc + 1e-5) / (pc + 1e-5) and its fp32 error bound."""
    pc, dpc = _sig_err(xp, dxp)
    nc, dnc = _sig_err(xn, dxn)
    num, den = pc - nc + 1e-5, pc + 1e-5
    a = num / den
    dnum = dpc + dnc + 2 * U * ((pc - nc).abs() + 1e-5)
    dden = dpc + U * den
    da = (dnum + a.abs() * dden) / den + U * a.abs()
    return pc, dpc, a * m, da * m


def _transmittance(alpha, dalpha):
    """Exclusive T_s = prod_{j<s} (1 - alpha_j + 1e-7) and its bound T_s (sum_{j<s} dalpha_j / f_j + 3 U s): each
    factor f_j rounds twice and each product once; dT_s / dalpha_j = -T_s / f_j."""
    R, n = alpha.shape
    f = 1 - alpha + 1e-7
    T = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=alpha.dtype), f[:, :-1]], 1), 1)
    rel = torch.cumsum(torch.cat([torch.zeros(R, 1, dtype=alpha.dtype), (dalpha / f)[:, :-1]], 1), 1) \
        + 3 * U * torch.arange(n, dtype=alpha.dtype)
    return T, T * rel


def _upsample_reference(z, sdf, m, inv_s):
    """fp64 up_sample + sample_pdf weights of every section and the per-ray bound delta on the fp32 CDF.

    Section s (samples s, s+1): mid = (s0 + s1) / 2, dist = z1 - z0, dot = (s1 - s0) / (dist + 1e-5),
    d = clip(min(dot_{s-1}, dot_s), -10, 0) * m_s m_{s+1}, sigmoid arguments (mid -+ d dist / 2) inv_s,
    alpha = mask (pc - nc + 1e-5) / (pc + 1e-5), w = alpha T + 1e-5.  fp32 error of the arguments: mid U |mid|,
    dot 4 U |dot| (hence d), the product d dist / 2 2 U, the difference and the scaling one U each.  Then the CDF
    c_k = sum_{s<k} w_s / W (fp32 sum of S - 1 weights, divisions, running sum):
    delta_k = (sum_{s<k} dw_s + c_k dW) / W + (k + 1) U c_k, dW = sum dw + (S - 1) U W; delta = max_k delta_k."""
    z, s = z.double(), sdf.double()
    mm = m[:, :-1] * m[:, 1:]
    s0, s1, z0, z1 = s[:, :-1], s[:, 1:], z[:, :-1], z[:, 1:]
    mid = (s0 + s1) * 0.5
    dist = z1 - z0
    dot = (s1 - s0) / (dist + 1e-5)
    prev = torch.cat([torch.zeros_like(dot[:, :1]), dot[:, :-1]], 1)
    d = torch.minimum(prev, dot).clip(-10.0, 0.0) * mm
    dd = 4 * U * torch.maximum(prev.abs(), dot.abs()) * mm
    q = d * dist * 0.5
    dq = (dd * dist + d.abs() * U * dist) * 0.5 + 2 * U * q.abs()
    xp, xn = (mid - q) * inv_s, (mid + q) * inv_s
    dxp = inv_s * (U * mid.abs() + dq + U * (mid - q).abs()) + U * xp.abs()
    dxn = inv_s * (U * mid.abs() + dq + U * (mid + q).abs()) + U * xn.abs()
    _, _, alpha, dalpha = _alpha_err(xp, dxp, xn, dxn, mm)
    T, dT = _transmittance(alpha, dalpha)
    w = alpha * T + 1e-5
    dw = dalpha * T + alpha * dT + 2 * U * w
    W = w.sum(1, keepdim=True)
    dW = dw.sum(1, keepdim=True) + (w.shape[1]) * U * W
    cw = torch.cumsum(w, 1)
    cdf = torch.cat([torch.zeros_like(W), cw / W], 1)                        # [R, S]
    cdw = torch.cat([torch.zeros_like(W), torch.cumsum(dw, 1)], 1)
    k = torch.arange(cdf.shape[1], dtype=torch.float64)
    delta = ((cdw + cdf * dW) / W + (k + 1) * U * cdf).amax(1)
    return cdf, delta


def _check_samples(tag, z, cdf, delta, u, new_z):
    """Per-sample check of the inverse-CDF draw (see test_ray_upsample_per_sample)."""
    R, S = z.shape
    zz = z.double()
    uu = u.double().expand(R, -1).contiguous()
    ind = torch.searchsorted(cdf, uu, right=True)
    below, above = (ind - 1).clamp(min=0), ind.clamp(max=S - 1)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(zz, 1, below), torch.gather(zz, 1, above)
    den = c1 - c0
    den_eff = torch.where(den < 1e-5, torch.ones_like(den), den)
    z64 = b0 + (uu - c0) / den_eff * (b1 - b0)
    dl = delta[:, None]
    # containment: every knot within delta of u may have moved to either side of it
    lo = torch.searchsorted(cdf, uu - dl, right=False)
    hi = torch.searchsorted(cdf, uu + dl, right=True) - 1
    zlo = torch.gather(zz, 1, (torch.minimum(lo, hi) - 1).clamp(0, S - 1))
    zhi = torch.gather(zz, 1, (torch.maximum(lo, hi) + 1).clamp(0, S - 1))
    g = new_z.double()
    slack = 2 * U * g.abs()
    assert bool(((g >= zlo - slack) & (g <= zhi + slack)).all()), tag + ": a sample left its admissible bins"
    near_knot = hi >= lo                                   # some knot lies within delta of u
    amb_branch = (den - 1e-5).abs() <= 2 * dl
    tight = ~near_knot & ~amb_branch
    bound = (b1 - b0) * (3 * dl / den_eff + 4 * U) + 2 * U * z64.abs()
    print(f"{tag}: {int(tight.sum())} of {tight.numel()} samples away from knots and the 1e-5 branch; "
          f"delta up to {float(delta.max()):.2e}")
    _assert_within(tag, (g - z64).abs()[tight], bound[tight])


@pytest.mark.parametrize("R", [1, 63, 64, 65, 4097])
@pytest.mark.parametrize("n_new", [1, 16])
@pytest.mark.parametrize("S", [2, 3, 64, 80, 112, 512])
def test_ray_upsample_per_sample(S, n_new, R):
    """o2345_ray_upsample against up_sample + sample_pdf(det=True) written out in fp64, sample by sample, at
    inv_s = 64 and 512 (the renderer's 64 * 2^i schedule) and u = linspace(0.5/n, 1 - 0.5/n, n).

    delta is the derived bound on the fp32 CDF error of the ray (_upsample_reference).  For every sample:
    - it lies between the bins of the knots within delta of u (the fp64 bin when no knot is that close);
    - where no knot is within delta of u and the fp64 bin's den is not within 2 delta of 1e-5 (so the kernel takes the
      same bin and the same den branch), |z - z64| <= (b1 - b0) (3 delta / den + 4 U) + 2 U |z64|: c0 is off by
      delta and den by 2 delta, so t = (u - c0) / den is off by 3 delta / den, plus the fp32 roundings.
    Profiles: one crossing, a crossing in the first / last section, none (all positive / all negative), several, a
    constant SDF; occupancy fully set, empty, or in blocks of 8 cells along the ray."""
    ops = _ops()
    o, d, z, sdf, occ, m = _ray_scene(R, S, seed=S * 7 + R)
    od, dd, zd, sd = _cuda(o), _cuda(d), _cuda(z), _cuda(sdf)
    occd = _cuda(occ).view(1, 1, RAY_D, RAY_D, RAY_D)
    act = ops.occ_nearest(ops.PointSource.rays(od, dd, zd), occd).view(R, S).cpu()
    assert torch.equal(act, torch.from_numpy(m).to(torch.uint8)), "sample occupancy is not the constructed one"
    u = torch.linspace(0.5 / n_new, 1.0 - 0.5 / n_new, n_new)
    for inv_s in (64.0, 512.0):
        new_z = ops.ray_upsample(od, dd, zd, sd, inv_s, occd, u.to(DEV)).cpu()
        cdf, delta = _upsample_reference(torch.from_numpy(z), torch.from_numpy(sdf), torch.from_numpy(m).double(), inv_s)
        _check_samples(f"ray_upsample S={S} n={n_new} R={R} inv_s={inv_s:g}", torch.from_numpy(z), cdf, delta, u, new_z)


def _emulate_cdf(alpha, S):
    """The kernel's fp32 CDF, bit for bit, for sections whose alpha is exactly 0 or 1 (so every product alpha T is
    exact and no fused multiply-add can change a rounding)."""
    T, ws = f32(1), []
    for a in alpha:
        a = f32(a)
        ws.append(f32(a * T + f32(1e-5)))
        T = f32(T * f32(f32(f32(1) - a) + f32(1e-7)))
    wsum = f32(0)
    for w in ws:
        wsum = f32(wsum + w)
    cdf, run = [f32(0)], f32(0)
    for w in ws:
        run = f32(run + f32(w / wsum))
        cdf.append(run)
    return np.array(cdf, f32)


@pytest.mark.parametrize("S", [64, 512])
@pytest.mark.parametrize("inside", [True, False])
def test_ray_upsample_exact_knots(inside, S):
    """Profiles whose fp32 CDF is known exactly: every sample deep inside an occupied object (pc = nc = 0, alpha = 1:
    after the first section every bin has den < 1e-5), or every section masked by occupancy (alpha = 0).  u is put
    exactly on CDF knots: searchsorted(right=True) then picks the bin that starts at the knot, t = 0 and the draw is
    that knot's depth, bit for bit; u at or past the last knot gives the last depth.  One u inside the first bin is
    held to the fp32 bound of its interpolation."""
    ops = _ops()
    R = 65
    o, d, z, _ = _ray_layout(R, S, seed=S)
    D = RAY_D
    occ = np.zeros((D, D, D), f32)
    if inside:
        for r in range(R):
            occ[:, r % D, (r // D) % D] = 1
    sdf = np.full((R, S), -3.0, f32)
    cdf = _emulate_cdf([1.0 if inside else 0.0] * (S - 1), S)
    ks = [1, 2, 3, S // 2, S - 2, S - 1]
    u_knots = sorted(set(float(cdf[k]) for k in ks))
    u_first = float(f32(0.5) * cdf[1])
    u_all = [u_first] + u_knots + ([1.0] if cdf[-1] < 1 else [])
    u = torch.tensor(u_all, dtype=torch.float32)
    for inv_s in (64.0, 512.0):
        new_z = ops.ray_upsample(_cuda(o), _cuda(d), _cuda(z), _cuda(sdf), inv_s, _cuda(occ).view(1, 1, D, D, D),
                                 u.to(DEV)).cpu()
        zt = torch.from_numpy(z)
        for j, uj in enumerate(u_all[1:], 1):
            k = int(np.searchsorted(cdf, f32(uj), side="right")) - 1
            assert torch.equal(new_z[:, j], zt[:, k]), f"u = cdf[{k}] must draw z[{k}] exactly (inside={inside})"
        c1 = float(cdf[1])
        z64 = zt[:, 0].double() + u_first / c1 * (zt[:, 1].double() - zt[:, 0].double())
        bound = (zt[:, 1] - zt[:, 0]).double() * 8 * U + 2 * U * z64.abs()
        _assert_within(f"ray_upsample exact knots S={S} inside={inside} inv_s={inv_s:g} first bin",
                       (new_z[:, 0].double() - z64).abs(), bound)
    print(f"ray_upsample exact knots S={S} inside={inside}: {len(u_knots)} knot draws bit-exact")


@pytest.mark.parametrize("S,n_new", [(64, 16), (80, 1), (2, 64), (112, 16)])
def test_ray_merge_is_a_stable_sort(S, n_new):
    """o2345_ray_merge against a stable sort of cat([old, new]) keyed by depth: on ties the old sample comes first and
    every sdf follows its depth; duplicates inside one list keep their order.  Bit-exact; 130 rays (two CTAs)."""
    ops = _ops()
    rng = _rng(S + n_new)
    R = 130
    old = np.sort(rng.choice(np.arange(0, 4, 0.125, dtype=f32), size=(R, S)), 1)       # duplicates inside a list
    new = np.sort(rng.choice(np.arange(0, 4, 0.125, dtype=f32), size=(R, n_new)), 1)   # and ties with the old list
    new[R // 2:] = np.sort(rng.uniform(0, 4, size=(R - R // 2, n_new)).astype(f32), 1)
    so = rng.standard_normal((R, S)).astype(f32)
    sn = rng.standard_normal((R, n_new)).astype(f32)
    oz, osdf = ops.ray_merge(_cuda(old), _cuda(so), _cuda(new), _cuda(sn))
    zc = torch.cat([torch.from_numpy(old), torch.from_numpy(new)], 1)
    sc = torch.cat([torch.from_numpy(so), torch.from_numpy(sn)], 1)
    zs, idx = torch.sort(zc, dim=1, stable=True)
    ties = sum(int(np.isin(new[r], old[r]).sum()) for r in range(R))
    print(f"ray_merge S={S} n_new={n_new}: {ties} new depths tie with an old one; bit-exact")
    assert ties > 0
    assert torch.equal(oz.cpu(), zs)
    assert torch.equal(osdf.cpu(), torch.gather(sc, 1, idx))


@pytest.mark.parametrize("per_ray", [False, True])
@pytest.mark.parametrize("S", [1, 5, 64])
def test_ray_midpoints_exact(S, per_ray):
    """o2345_ray_midpoints(_per_ray): dists = fl(z[s+1] - z[s]) (the last one sample_dist, a scalar or one per ray),
    mid = fl(z + dists * 0.5), bit for bit against the same fp32 arithmetic on the host; active is the nearest
    occupancy of fl(o + fl(d * mid)), equal to occ_nearest and grid_sample at those points."""
    ops = _ops()
    rng = _rng(S + 100 * int(per_ray))
    R, D = 37, 24
    z = np.sort(rng.uniform(0.2, 2.5, size=(R, S)).astype(f32), 1)
    o = rng.uniform(-1, 1, size=(R, 3)).astype(f32)
    d = rng.standard_normal((R, 3)).astype(f32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    occ = (torch.from_numpy(rng.random((D, D, D))) < 0.5).float().view(1, 1, D, D, D).to(DEV)
    last = rng.uniform(0.01, 0.05, size=R).astype(f32) if per_ray else np.full(R, f32(0.0123), f32)
    mid, dists, active = ops.ray_midpoints(_cuda(o), _cuda(d), _cuda(z), _cuda(last) if per_ray else float(last[0]), occ)
    dw = np.concatenate([z[:, 1:] - z[:, :-1], last[:, None]], 1)
    mw = z + dw * f32(0.5)
    assert dw.dtype == np.float32 and mw.dtype == np.float32
    assert np.array_equal(dists.cpu().numpy().view(np.int32), dw.view(np.int32))
    assert np.array_equal(mid.cpu().numpy().view(np.int32), mw.view(np.int32))
    p = (o[:, None, :] + d[:, None, :] * mw[..., None]).reshape(-1, 3)
    pd = _cuda(p)
    assert torch.equal(active, ops.occ_nearest(ops.PointSource.explicit(pd), occ))
    assert torch.equal(active, _grid_nearest(occ, pd))
    print(f"ray_midpoints S={S} per_ray={per_ray}: mid, dists and active bit-exact ({int(active.sum())} active)")


def _composite_inputs(R, S, seed):
    """Per-ray cases: gradients towards / away from the ray / random / large enough to hit the +-10 clip, inactive
    samples, a step in the SDF that saturates both sigmoids."""
    rng = _rng(seed)
    d = rng.standard_normal((R, 3)).astype(f32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    z = np.sort(rng.uniform(0.5, 2.5, size=(R, S)), 1).astype(f32)
    dists = np.concatenate([np.diff(z, axis=1), np.full((R, 1), 0.01)], 1).astype(f32)
    mid = (z + dists * f32(0.5)).astype(f32)
    sdf = np.zeros((R, S), f32)
    grad = rng.standard_normal((R, S, 3)).astype(f32)
    for r in range(R):
        kind = r % 5
        zc = rng.uniform(z[r, 0], z[r, -1])
        sdf[r] = (zc - mid[r]) * rng.uniform(0.5, 2.0)
        if kind == 0:
            grad[r] = -d[r] * rng.uniform(0.5, 1.5)                # facing the ray (cos < 0)
        elif kind == 1:
            grad[r] = d[r] * rng.uniform(0.5, 1.5)                 # facing away (cos > 0)
        elif kind == 2:
            grad[r] *= 50.0                                         # |cos| up to ~100: the +-10 clip
        elif kind == 3:
            sdf[r] = np.where(mid[r] < zc, 5.0, -5.0)               # a jump: alpha saturates to exactly 1
            grad[r] = -d[r] * 20.0
    active = (rng.random((R, S)) < 0.8).astype(np.uint8)
    active[::7] = 1
    nvalid = rng.integers(0, 5, size=(R, S)).astype(np.int32)
    color = rng.random((R, S, 3)).astype(f32)
    return d, mid, dists, sdf, grad, color, active, nvalid


def _composite_reference(d, mid, dists, sdf, grad, color, active, nvalid, inv_s, ratio, bg):
    """fp64 NeuS alpha + compositing and the fp32 bounds.  cos = d . g (3 U sum |d_i g_i|), iter_cos
    (4 U (1.5 |cos| + 0.5)), e = clip(iter_cos) dists / 2 (U |e|), arguments (sdf -+ e) inv_s (2 U |x|), then the
    sigmoid / alpha / transmittance bounds shared with the up-sampling reference; colour and depth add the fp32 sums
    (S U sum |c| w)."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).double()
    d, mid, dists, sdf, grad, color = t(d), t(mid), t(dists), t(sdf), t(grad), t(color)
    m = t(active)
    R, S = mid.shape
    cos = (d[:, None, :] * grad).sum(-1)
    dcos = 3 * U * (d[:, None, :] * grad).abs().sum(-1)
    it = -(torch.relu(-cos * 0.5 + 0.5) * (1.0 - ratio) + torch.relu(-cos) * ratio) * m
    dit = (dcos * (0.5 * abs(1 - ratio) + abs(ratio)) + 4 * U * (1.5 * cos.abs() + 0.5)) * m
    e = it.clip(-10.0, 10.0) * dists * 0.5
    de = dit * dists * 0.5 + U * e.abs()
    xp, xn = (sdf - e) * inv_s, (sdf + e) * inv_s
    dxp = inv_s * de + 2 * U * xp.abs()
    dxn = inv_s * de + 2 * U * xn.abs()
    pc, dpc, alpha, dalpha = _alpha_err(xp, dxp, xn, dxn, m)
    alpha = alpha.clip(0.0, 1.0)
    T, dT = _transmittance(alpha, dalpha)
    w = alpha * T
    dw = dalpha * T + alpha * dT + U * w
    wsum = w.sum(1)
    dwsum = dw.sum(1) + S * U * wsum
    col = (color * w[..., None]).sum(1)
    dcol = (color.abs() * dw[..., None]).sum(1) + S * U * (color.abs() * w[..., None]).sum(1)
    if bg is not None:
        k = bg * (1 - wsum)
        col = col + k[:, None]
        dcol = dcol + abs(bg) * dwsum[:, None] + 2 * U * k.abs()[:, None] + U * col.abs()
    depth = (mid * w).sum(1, keepdim=True)
    ddepth = (mid.abs() * dw).sum(1, keepdim=True) + S * U * (mid.abs() * w).sum(1, keepdim=True)
    cmask = ((t(nvalid) >= 2).sum(1) > 8).to(torch.uint8)[:, None]
    return {"color": (col, dcol), "depth": (depth, ddepth), "weights": (w, dw), "cdf": (pc, dpc),
            "alpha": (alpha, dalpha), "weights_sum": (wsum[:, None], dwsum[:, None])}, cmask


def _composite(d, mid, dists, sdf, grad, color, active, nvalid, inv_s, ratio, bg):
    ops = _ops()
    return ops.ray_composite(_cuda(d), _cuda(mid), _cuda(dists), _cuda(sdf.reshape(-1, 1)), _cuda(grad.reshape(-1, 3)),
                             _cuda(color.reshape(-1, 3)), _cuda(active.reshape(-1)), _cuda(nvalid.reshape(-1)), inv_s,
                             ratio, bg)


@pytest.mark.parametrize("bg", [None, 1.0])
@pytest.mark.parametrize("ratio", [0.0, 0.5, 1.0])
def test_ray_composite_matches_fp64(ratio, bg):
    """o2345_ray_composite against fp64 NeuS alpha and compositing (reference render_core): every output -- colour,
    depth, weights, cdf, alpha, weights_sum within their derived bounds (_composite_reference), color_mask exactly."""
    R, S = 200, 24
    inp = _composite_inputs(R, S, seed=int(ratio * 10) + (bg is not None))
    for inv_s in (64.0, 512.0):
        out = _composite(*inp, inv_s, ratio, bg)
        ref, cmask = _composite_reference(*inp, inv_s, ratio, bg)
        for key, (want, bound) in ref.items():
            _assert_within(f"ray_composite ratio={ratio} bg={bg} inv_s={inv_s:g} {key}",
                           (out[key].double().cpu().view_as(want) - want).abs(), bound)
        assert torch.equal(out["color_mask"].cpu(), cmask)
        sat = int((ref["alpha"][0] == 1).sum())
        print(f"ray_composite ratio={ratio} bg={bg} inv_s={inv_s:g}: {sat} samples with alpha exactly 1")


@pytest.mark.parametrize("S,n_ge2,want", [(8, 8, 0), (9, 9, 1), (16, 8, 0), (16, 9, 1)])
def test_ray_composite_color_mask_threshold(S, n_ge2, want):
    """color_mask = (number of samples with nvalid >= 2) > 8, exactly at the threshold: 8 such samples give 0 and 9
    give 1 (the rest of the samples have nvalid 0 or 1)."""
    R = 5
    inp = list(_composite_inputs(R, S, seed=S + n_ge2))
    nvalid = np.tile(np.array([2] * n_ge2 + [1, 0] * S, np.int32)[:S], (R, 1))
    rolled = np.roll(nvalid[1], 3)
    nvalid[1] = np.where(rolled >= 2, rolled + 5, rolled)           # other positions, nvalid up to 7
    inp[7] = nvalid
    out = _composite(*inp, 64.0, 0.5, None)
    assert bool((out["color_mask"].cpu() == want).all()), (S, n_ge2, out["color_mask"].view(-1).tolist())
