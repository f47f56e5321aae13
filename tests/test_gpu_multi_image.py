"""GPU: several images -> several meshes (pipeline.images_to_meshes, zero123.generate_views_multi, run.py with several
paths), everything through the C ABI.  Seeded synthetic weights, 4 / 2 DDIM steps and R = 64 keep it short."""
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

STEPS = dict(ddim_steps=4, stage2_steps=2)        # S = 3 is not a valid uniform schedule (timestep 1000)
R = 64


@pytest.fixture(scope="module")
def nets():
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks
    from o2345.zero123 import build_zero123
    dev = torch.device("cuda:0")
    z = build_zero123(dev, seed=0, clip=True).half()
    tr = build_networks(dev, vol_dim=96, states=S.all_states(0), perturb=0.0)
    return z, tr, dev


def _images(n, seed=7):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        im = np.full((256, 256, 3), 255, np.uint8)
        im[48:208, 56:200] = rng.integers(0, 255, (160, 144, 3), dtype=np.uint8)     # an "object" on white
        out.append(im)
    return out


def _u8(v):
    return v.cpu().numpy() if torch.is_tensor(v) else v


def _same_mesh(a, b):
    for k in ("vertices", "triangles", "colors"):
        x, y = np.asarray(_u8(a[k])), np.asarray(_u8(b[k]))
        assert x.shape == y.shape and x.dtype == y.dtype and np.array_equal(x, y), k


def test_one_image_is_the_single_image_run(nets):
    from o2345.pipeline import image_to_mesh, images_to_meshes
    from o2345.zero123 import generate_views, generate_views_multi
    z, tr, dev = nets
    x = _images(1)[0]
    s = 23
    torch.cuda.manual_seed(s)
    v1 = generate_views(z, x, 60, device=dev, keep_on_device=True, **STEPS)
    vm = generate_views_multi(z, [x], [60], seed=s, device=dev, keep_on_device=True, **STEPS)
    assert len(vm) == 1 and vm[0][2] == v1[2]
    for a, b in ((v1[0], vm[0][0]), (v1[1], vm[0][1])):
        assert list(a) == list(b)
        for k in a:
            assert torch.equal(a[k], b[k]), k
    torch.cuda.manual_seed(s)
    want = image_to_mesh(z, tr, x, polar_angle=60, resolution=R, **STEPS)
    got = list(images_to_meshes(z, tr, [x], [60], seed=s, resolution=R, **STEPS))
    assert [i for i, _ in got] == [0] and len(want["vertices"]) > 100
    _same_mesh(want, got[0][1])


def test_packed_against_one_at_a_time(nets, tmp_path):
    from o2345.pipeline import images_to_meshes, sample_from_views
    from o2345.zero123 import generate_views_multi
    z, tr, dev = nets
    xs = _images(3)
    polars = [60, 70, 65]
    dirs = {k: [str(tmp_path / f"k{k}" / f"im{i}") for i in range(3)] for k in (1, 3)}
    meshes = {k: list(images_to_meshes(z, tr, xs, polars, seed=4, resolution=R, exp_dirs=dirs[k], max_pack=k, **STEPS))
              for k in (1, 3)}
    assert [i for i, _ in meshes[3]] == [i for i, _ in meshes[1]] == [0, 1, 2]
    from PIL import Image
    worst, means = 0, []
    for i in range(3):
        a, b = dirs[1][i], dirs[3][i]
        assert json.load(open(os.path.join(a, "pose.json"))) == json.load(open(os.path.join(b, "pose.json")))
        for sub in ("stage1_8", "stage2_8"):
            names = sorted(os.listdir(os.path.join(a, sub)))
            assert names == sorted(os.listdir(os.path.join(b, sub))) and len(names) == (8 if sub == "stage1_8" else 32)
            for f in names:
                d = np.abs(np.asarray(Image.open(os.path.join(a, sub, f)), np.int32) - np.asarray(Image.open(os.path.join(b, sub, f)), np.int32))
                worst, means = max(worst, int(d.max())), means + [float(d.mean())]
        assert os.path.exists(os.path.join(b, "mesh.ply"))
    print("packed (K = 3) vs one at a time: max |diff| %d grey levels, mean %.4f" % (worst, float(np.mean(means))))
    assert worst <= 2 and float(np.mean(means)) <= 0.2, (worst, float(np.mean(means)))
    # path B sees each image's own views: every packed mesh is the reconstruction of that image's packed views (host
    # copies, as with exp_dirs: the device hand-off divides by 255 on the GPU, which may round differently in the last bit)
    views = generate_views_multi(z, xs, polars, seed=4, device=dev, keep_on_device=False, **STEPS)
    tr.base_exp_dir = None
    for i, (s1, s2, pose) in enumerate(views):
        _same_mesh(tr(sample_from_views(s1, s2, pose, dev), mode="export_mesh", resolution=R), meshes[3][i][1])
    assert len(meshes[3][0][1]["vertices"]) != len(meshes[3][1][1]["vertices"]) or \
        not np.array_equal(meshes[3][0][1]["vertices"], meshes[3][1][1]["vertices"])


def test_mixed_elevations_in_one_pack(nets):
    from o2345 import synthetic as S
    from o2345.zero123 import generate_views_multi
    z, tr, dev = nets
    xs = _images(2, seed=9)
    views = generate_views_multi(z, xs, [60, 80], seed=0, device=dev, **STEPS)
    assert sorted(views[0][0]) == [0, 1, 2, 3, 4, 5, 6, 7]
    assert sorted(views[1][0]) == [0, 1, 2, 3, 8, 9, 10, 11]
    assert sorted(views[0][1]) == sorted(f"{i}_{j}" for i in range(8) for j in range(4))
    assert sorted(views[1][1]) == sorted(f"{i}_{j}" for i in [0, 1, 2, 3, 8, 9, 10, 11] for j in range(4))
    assert views[0][2] == S.pose_json(60.0) and views[1][2] == S.pose_json(80.0) and views[0][2] != views[1][2]
    assert all(v.dtype == np.uint8 and v.shape == (256, 256, 3) for t in views for v in list(t[0].values()) + list(t[1].values()))


def test_run_py_with_two_images(tmp_path, monkeypatch):
    from PIL import Image
    import run as run_cli
    monkeypatch.chdir(tmp_path)
    paths = []
    for name, im in zip(("a", "b"), _images(2, seed=5)):
        paths.append(str(tmp_path / f"{name}.png"))
        Image.fromarray(im).save(paths[-1])
    out = run_cli.main(["--img_path", *paths, "--mesh_resolution", "64", "--polar_angle", "60", "80"])
    assert len(out) == 2
    for name, polar, ply in zip(("a", "b"), (60.0, 80.0), out):
        d = tmp_path / "exp" / name
        assert os.path.samefile(ply, d / "mesh.ply")
        assert len(os.listdir(d / "stage1_8")) == 8 and len(os.listdir(d / "stage2_8")) == 32
        from o2345 import synthetic as S
        assert json.load(open(d / "pose.json")) == json.loads(json.dumps(S.pose_json(polar)))
        data = (d / "mesh.ply").read_bytes()
        assert data.startswith(b"ply") and int(data.split(b"element vertex ")[1].split(b"\n")[0]) > 100
