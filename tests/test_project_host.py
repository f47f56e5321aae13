"""CPU tests of the input-view projection: the model of oracle/project_oracle.py on hand-computed cases (facing, near
plane, image bounds, depth test, background, normals, alpha), the two intrinsics rules (the depth buffer's shift, shown
with the rasterizer's oracle, and the photo's rescale), the photo loader, the command line and the ABI checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import project_oracle as PO
from oracle import raster_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
W = H = 64
INTR = (100.0, 100.0, 32.0, 32.0)
EYE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], F)     # camera at the origin looking down +z
RGB = (200, 100, 50)
BASE = F(0.25)


def photo(rgb=RGB):
    return np.tile(np.array(rgb, np.uint8), (H, W, 1))


def run(points, normals, depth_value=None, s=1, alpha=None, depth=None):
    """Weights and colours of points with normals, a uniform photo and a buffer of one depth (the plane at z = 2)."""
    p, n = np.asarray(points, F).reshape(-1, 3), np.asarray(normals, F).reshape(-1, 3)
    if depth is None:
        depth = np.full((s * H, s * W), F(2.0) if depth_value is None else F(depth_value), F)
    base = np.full((len(p), 3), BASE, F)
    return PO.project_view(p, n, base, EYE, INTR, photo(), alpha, depth)


def tilted(cos):
    """A unit normal at angle acos(cos) to the direction from (0, 0, 2) to the camera."""
    return [0.0, np.sqrt(1 - cos * cos), -cos]


def test_plane_facing_the_camera_takes_the_photo():
    out, w = run([0, 0, 2], [0, 0, -1])
    assert w[0] == 1
    np.testing.assert_allclose(out[0], np.array(RGB) / 255, rtol=0, atol=1e-7)


@pytest.mark.parametrize("cos, want", [(0.7 + 1e-4, 1.0), (0.9, 1.0), (0.5, 0.5), (0.4, 0.25), (0.3 - 1e-4, 0.0),
                                       (0.0, 0.0), (-1.0, 0.0)])
def test_facing_weight_ramps_between_the_constants(cos, want):
    _, w = run([0, 0, 2], tilted(cos))
    assert w[0] == pytest.approx(want, abs=2e-6)


def test_points_behind_the_camera_or_at_near_are_not_seen():
    _, w = run([[0, 0, -1], [0, 0, 0.1], [0, 0, 0.05], [0, 0, 0.1001]], [[0, 0, -1]] * 4,
               depth=np.zeros((H, W), F))
    assert w.tolist() == [0, 0, 0, 1]


def test_points_outside_the_image_by_half_a_pixel_are_not_seen():
    z = 2.0
    xs = np.array([-0.5, W - 0.5, 0.25, W - 1.25], np.float64)         # image x of each point (pixel i's centre at i)
    pts = [[(x - INTR[2]) * z / INTR[0], 0, z] for x in xs] + [[0, (y - INTR[3]) * z / INTR[1], z] for y in xs]
    _, w = run(pts, [[0, 0, -1]] * len(pts))
    assert w.tolist() == [0, 0, 1, 1] * 2


@pytest.mark.parametrize("s", [1, 2, 4])
def test_depth_test_allows_two_buffer_pixels_of_slope(s):
    tau = 2 * 2.0 / (s * INTR[0])                                        # TAU_PIX q.z / (s fx) / cos, cos = 1
    for d, want in ((2.0, 1), (2.0 - 0.9 * tau, 1), (2.0 - 1.1 * tau, 0), (1.5, 0), (2.5, 1)):
        _, w = run([0, 0, 2], [0, 0, -1], depth_value=d, s=s)
        assert w[0] == want, (s, d)
    # a tilted surface gets a wider band: tau / cos
    _, w = run([0, 0, 2], tilted(0.8), depth_value=2.0 - 1.1 * tau, s=s)
    assert w[0] == 1
    _, w = run([0, 0, 2], tilted(0.8), depth_value=2.0 - 1.3 * tau, s=s)
    assert w[0] == 0


def test_background_buffer_pixels_count_as_seen():
    _, w = run([0, 0, 2], [0, 0, -1], depth_value=0.0)
    assert w[0] == 1


def test_zero_and_non_finite_normals_are_not_seen():
    normals = [[0, 0, 0], [np.nan, 0, -1], [0, np.inf, -1], [0, 0, -np.inf], [0, 0, -1e-30], [0, 0, -1e-10], [0, 0, -5]]
    _, w = run([[0, 0, 2]] * len(normals), normals)
    # the length does not matter, the direction does; a length whose fp32 square underflows counts as zero
    assert w.tolist() == [0, 0, 0, 0, 0, 1, 1]


def test_non_finite_points_are_not_seen():
    _, w = run([[np.nan, 0, 2], [0, np.inf, 2], [0, 0, np.inf], [0, 0, np.nan]], [[0, 0, -1]] * 4)
    assert w.tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("a, want", [(0, 0.0), (128, F(128) / F(255)), (255, 1.0)])
def test_alpha_scales_the_weight(a, want):
    out, w = run([0, 0, 2], [0, 0, -1], alpha=np.full((H, W), a, np.uint8))
    assert w[0] == want
    if a == 0:
        assert (out[0] == BASE).all()


def test_unseen_points_keep_the_base_colour_bit_for_bit():
    p = np.array([[0, 0, -1], [0, 0, 2], [100, 0, 2]], F)
    n = np.array([[0, 0, -1]] * 3, F)
    base = np.array([[-0.0, np.nan, 0.3], [0.1, 0.2, 0.3], [np.float32(1) / 3, -0.0, 7.0]], F)
    out, w = PO.project_view(p, n, base, EYE, INTR, photo(), None, np.full((H, W), 2, F))
    assert w.tolist() == [0, 1, 0]
    for i in (0, 2):
        assert np.array_equal(out[i].view(np.uint32), base[i].view(np.uint32))


def test_bilinear_follows_the_projector():
    img = np.arange(4 * 5, dtype=np.uint8).reshape(4, 5, 1) * 10
    x = np.array([0, 4, 1.5, 3.25, 4, 0], F)
    y = np.array([0, 3, 2.5, 0.75, 1.5, 3], F)
    got = PO.bilinear(img, x, y)[:, 0]
    xf, yf = x.astype(np.float64), y.astype(np.float64)
    a = img[..., 0].astype(np.float64)
    # reference: separable linear interpolation in fp64
    want = [np.interp(xv, np.arange(5), np.array([np.interp(yv, np.arange(4), a[:, c]) for c in range(5)]))
            for xv, yv in zip(xf, yf)]
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-4)


def test_photo_colour_is_sampled_where_the_point_projects():
    img = np.zeros((H, W, 3), np.uint8)
    img[20, 40] = (255, 128, 0)
    p = np.array([[(40 - INTR[2]) * 2 / INTR[0], (20 - INTR[3]) * 2 / INTR[1], 2]], F)
    out, w = PO.project_view(p, [[0, 0, -1]], np.zeros((1, 3), F), EYE, INTR, img, None, np.full((H, W), 2, F))
    assert w[0] == 1
    np.testing.assert_allclose(out[0], [1, 128 / 255, 0], atol=1e-6)


def test_face_normals():
    v = np.array([[0, 0, 0], [2, 0, 0], [0, 3, 0], [0, 0, 0], [1, 1, 1], [2, 2, 2]], F)
    f = np.array([[0, 1, 2], [0, 2, 1], [3, 4, 5], [0, 1, 9]])
    n = PO.face_normals(v, f, [0, 1, 2, 3, -1, 4, 0])
    np.testing.assert_array_equal(n, [[0, 0, 1], [0, 0, -1], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 1]])


# ----------------------------------------------------------------------------- the two intrinsics rules
@pytest.mark.parametrize("s", [1, 2, 3, 4])
def test_photo_pixel_covers_its_s_by_s_block_of_the_depth_buffer(s):
    """The square of photo pixel (i, k) (image coordinates i +- 0.5, k +- 0.5) at depth 2, rendered into the buffer
    with depth_intrinsics, covers exactly buffer pixels s i .. s i + s - 1 (and rows alike); the projection's buffer
    pixel of any point inside the square lies in that block."""
    from o2345.mesh_texture import depth_intrinsics
    i, k, z = 17, 40, 2.0
    corners = [(i - 0.5, k - 0.5), (i + 0.5, k - 0.5), (i + 0.5, k + 0.5), (i - 0.5, k + 0.5)]
    verts = np.array([[(x - INTR[2]) * z / INTR[0], (y - INTR[3]) * z / INTR[1], z] for x, y in corners], F)
    faces = np.array([[0, 1, 2], [0, 2, 3]])
    r = RO.render(verts, faces, EYE[None], np.array([depth_intrinsics(INTR, s)], F), s * W, s * H)
    rows, cols = np.nonzero(r["tri"][0] >= 0)
    assert sorted(set(cols)) == list(range(s * i, s * i + s)) and sorted(set(rows)) == list(range(s * k, s * k + s))
    assert len(rows) == s * s
    # points inside the square find their buffer pixel in the block: floor(s (x + 0.5))
    for fx_, fy_ in ((0.0, 0.0), (-0.49, 0.3), (0.49, -0.49), (0.2, 0.49)):
        x, y = F(i + fx_), F(k + fy_)
        j, kk = int(np.floor(F(s) * (x + F(0.5)))), int(np.floor(F(s) * (y + F(0.5))))
        assert s * i <= j < s * i + s and s * k <= kk < s * k + s
        assert r["tri"][0, kk, j] >= 0


def test_depth_scale_is_capped():
    from o2345.mesh_texture import depth_scale
    assert [depth_scale(n, n) for n in (64, 256, 1024, 1300, 2048, 4096, 8192)] == [4, 4, 4, 3, 2, 1, 1]
    assert depth_scale(256, 2048) == 2


def test_rescaled_intrinsics_keep_pixel_centres():
    """Resizing 256 -> S maps the image span [-0.5, 255.5] onto [-0.5, S - 0.5]: a point's coordinate u becomes
    (u + 0.5) S / 256 - 0.5, so f' = f S / 256 and c' = (c + 0.5) S / 256 - 0.5."""
    from o2345.mesh_texture import rescale_intrinsics
    K = (280.0, 280.0, 128.0, 128.0)
    for S in (256, 512, 1000, 2048):
        fx, fy, cx, cy = rescale_intrinsics(K, (256, 256), (S, S))
        assert (fx, cx) == (280.0 * S / 256, 128.5 * S / 256 - 0.5) and (fy, cy) == (fx, cx)
        for X, Z in ((0.1, 2.0), (-0.3, 1.7), (0.0, 3.0)):
            u = K[0] * X / Z + K[2]
            assert fx * X / Z + cx == pytest.approx((u + 0.5) * S / 256 - 0.5, abs=1e-9)
    assert rescale_intrinsics(K, (256, 256), (256, 256)) == K
    # the image edges map onto each other; a half-pixel slip would move them
    fx, _, cx, _ = rescale_intrinsics(K, (256, 256), (1024, 1024))
    edge = lambda fxx, cxx, u: (u - cxx) / fxx                           # X / Z of image coordinate u
    assert edge(fx, cx, -0.5) == pytest.approx(edge(K[0], K[2], -0.5)) and \
        edge(fx, cx, 1023.5) == pytest.approx(edge(K[0], K[2], 255.5))


def test_load_photo_keeps_alpha_and_matches_load_input(tmp_path):
    from PIL import Image
    import run as run_cli
    rng = np.random.default_rng(0)
    rgba = rng.integers(0, 256, (300, 500, 4), dtype=np.uint8)
    p = str(tmp_path / "a.png")
    Image.fromarray(rgba, "RGBA").save(p)
    ph = run_cli.load_photo(p)
    assert ph["photo"].shape == (500, 500, 3) and ph["alpha"].shape == (500, 500)
    # the same composite on white: resized to 256 it is load_input's image
    comp = Image.alpha_composite(Image.new("RGBA", (500, 300), (255,) * 4), Image.fromarray(rgba, "RGBA")).convert("RGB")
    assert np.array_equal(ph["photo"], np.asarray(comp.resize((500, 500), Image.LANCZOS)))
    assert np.array_equal(run_cli.load_input(p), np.asarray(comp.resize((256, 256), Image.LANCZOS)))
    assert np.array_equal(ph["alpha"], np.asarray(Image.fromarray(rgba[..., 3]).resize((500, 500), Image.LANCZOS)))
    q = str(tmp_path / "b.png")
    Image.fromarray(rgba[:100, :120, :3], "RGB").save(q)
    ph = run_cli.load_photo(q)
    assert ph["photo"].shape == (256, 256, 3) and ph["alpha"] is None
    assert [run_cli.photo_side(*wh) for wh in ((100, 50), (300, 500), (4000, 10))] == [256, 500, 2048]


# ----------------------------------------------------------------------------- command line and the ABI
def test_run_py_project_input_argument():
    import run as run_cli
    assert run_cli.parse_args(["--img_path", "a.png", "--project_input"]).project_input
    assert not run_cli.parse_args(["--img_path", "a.png"]).project_input
    a = run_cli.parse_args(["--img_path", "a.png", "b.png", "--project_input", "--texture_size", "512", "--output_format",
                            ".glb"])
    assert a.project_input and a.texture_size == 512


def test_project_entry_points_are_declared_and_bound():
    from o2345 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "o2345.h")).read(), flags=re.S)
    for name in ("o2345_project_view", "o2345_face_normals"):
        assert re.search(rf"\bint {name}\s*\(", src), name
        assert name in _lib.EXPORTED
    assert re.search(r"#define O2345_ABI_VERSION 14\b", open(os.path.join(ROOT, "include", "o2345.h")).read())
    assert _lib.ABI_VERSION == 14
    # the constants the oracle restates are the header's
    for name, v in (("COS_LO", PO.COS_LO), ("COS_HI", PO.COS_HI), ("TAU_PIX", PO.TAU_PIX)):
        m = re.search(rf"#define O2345_PROJECT_{name} ([0-9.]+)f", src)
        assert m and F(m.group(1)) == v, name


def test_project_abi_checks_return_einval_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    ok = dict(fx=100.0, fy=100.0, cx=32.0, cy=32.0, near=0.1, W=64, H=64, s=4)

    def pv(n=10, fx=ok["fx"], fy=ok["fy"], cx=ok["cx"], near=ok["near"], W=ok["W"], H=ok["H"], s=ok["s"], photo=fake):
        return lib.o2345_project_view(fake, fake, fake, n, fake, fx, fy, cx, 32.0, near, photo, None, W, H, fake, s, fake,
                                      fake, None)
    cases = [
        lambda: pv(n=0), lambda: pv(photo=None), lambda: pv(fx=0.0), lambda: pv(fy=-1.0), lambda: pv(fx=float("inf")),
        lambda: pv(cx=float("nan")), lambda: pv(near=0.0), lambda: pv(W=0), lambda: pv(s=0), lambda: pv(W=8192, s=4),
        lambda: lib.o2345_face_normals(fake, 3, fake, 1, fake, 0, fake, None),
        lambda: lib.o2345_face_normals(fake, 0, fake, 1, fake, 10, fake, None),
        lambda: lib.o2345_face_normals(None, 3, fake, 1, fake, 10, fake, None),
    ]
    for i, call in enumerate(cases):
        assert call() == -1, (i, _lib.last_error())
        assert len(_lib.last_error()) > 0
