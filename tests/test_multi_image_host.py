"""CPU: the host side of the multi-image path -- run.py's arguments, the split of images into packs and ranks, and the
noise contract (image i is seeded with seed + i whatever the pack size and the number of ranks), the last through a
world-size-2 gloo run of pipeline.images_to_meshes with the sampler and the reconstruction replaced by stand-ins that
report the noise each image received."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

import run as run_cli  # noqa: E402
from o2345 import pipeline, sharding, zero123  # noqa: E402

N1, N2 = 3, 2          # sampler iterations of the stand-in stages


def test_one_path_parses_as_before():
    a = run_cli.parse_args(["--img_path", "x/thing.png"])
    assert a.img_path == ["x/thing.png"] and a.polar_angle == [60.0] and a.seed is None
    dirs, polars = run_cli.plan_inputs(a.img_path, a.polar_angle)
    assert dirs == [os.path.join("exp", "thing")] and polars == [60.0]


def test_several_paths_and_polar_angles():
    a = run_cli.parse_args(["--img_path", "a/one.png", "b/two.jpg", "three.png", "--polar_angle", "80", "--seed", "5"])
    assert a.seed == 5
    dirs, polars = run_cli.plan_inputs(a.img_path, a.polar_angle)
    assert dirs == [os.path.join("exp", n) for n in ("one", "two", "three")] and polars == [80.0] * 3
    a = run_cli.parse_args(["--img_path", "one.png", "two.png", "--polar_angle", "60", "85"])
    assert run_cli.plan_inputs(a.img_path, a.polar_angle)[1] == [60.0, 85.0]
    with pytest.raises(SystemExit, match="one value or one per image"):
        run_cli.plan_inputs(["one.png", "two.png", "three.png"], [60.0, 70.0])


def test_duplicate_basenames_are_refused_before_any_gpu_work(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit, match="basename 'thing'"):
        run_cli.main(["--img_path", "a/thing.png", "b/thing.jpg"])
    assert not (tmp_path / "exp").exists()


def test_packs_and_ranks():
    assert pipeline.pack_slices(7, 3) == [(0, 3), (3, 6), (6, 7)]
    assert pipeline.pack_slices(2, 8) == [(0, 2)]
    assert pipeline.pack_slices(3, 1) == [(0, 1), (1, 2), (2, 3)]
    with pytest.raises(ValueError):
        pipeline.pack_slices(3, 0)
    assert pipeline.MAX_PACK >= 1
    for n, world in ((8, 1), (8, 3), (5, 2), (2, 4)):
        shares = [sharding.assign_scenes(n, world, r) for r in range(world)]
        assert sorted(i for s in shares for i in s) == list(range(n))


def test_stage1_ids_follow_the_elevation():
    assert zero123._stage1_ids(60.0) == [0, 1, 2, 3, 4, 5, 6, 7]
    assert zero123._stage1_ids(75.0) == [0, 1, 2, 3, 4, 5, 6, 7]
    assert zero123._stage1_ids(80.0) == [0, 1, 2, 3, 8, 9, 10, 11]


def _fingerprint(draws):
    return [float(x_T.double().sum()) + sum(float(t.double().sum()) * (k + 2) for k, t in enumerate(noise))
            for _, (x_T, noise) in sorted(draws.items())]


class _Trainer(torch.nn.Module):
    """Stand-in for GenericTrainer: returns as the 'mesh' what the stand-in sample carries."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.base_exp_dir = None

    def forward(self, sample, mode, resolution):
        assert mode == "export_mesh"
        return sample


def _run(n, seed, max_pack, world, rank, polars):
    """images_to_meshes over this rank's share with the sampler replaced by the noise each image gets under the contract."""
    calls = []

    def fake_generate_views_multi(model, inputs_u8, polar_angles, ddim_steps, stage2_steps, scale, seed=0, indices=None,
                                  exp_dirs=None, device="cuda", keep_on_device=False):
        calls.append(list(indices))
        return [(zero123.image_noise(seed, i, p, N1, N2, "cpu"), None, {"polar": p}) for i, p in zip(indices, polar_angles)]

    real = (zero123.generate_views_multi, pipeline.sample_from_views)
    zero123.generate_views_multi = fake_generate_views_multi
    pipeline.sample_from_views = lambda s1, s2, pose, dev: (_fingerprint(s1), pose["polar"])
    try:
        mine = sharding.assign_scenes(n, world, rank)
        out = list(pipeline.images_to_meshes(None, _Trainer(), [np.zeros((2, 2, 3), np.uint8)] * len(mine),
                                             [polars[i] for i in mine], seed=seed, max_pack=max_pack, indices=mine))
    finally:
        zero123.generate_views_multi, pipeline.sample_from_views = real
    return out, calls


def _worker(rank, world, port, out):
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out[rank] = _run(5, 11, 2, world, rank, [60.0, 80.0, 60.0, 60.0, 90.0])
    dist.destroy_process_group()


def test_image_seed_does_not_depend_on_pack_or_world_size():
    polars = [60.0, 80.0, 60.0, 60.0, 90.0]
    one, calls = _run(5, 11, 1, 1, 0, polars)
    assert [i for i, _ in one] == list(range(5)) and calls == [[0], [1], [2], [3], [4]]
    packed, calls = _run(5, 11, 3, 1, 0, polars)
    assert calls == [[0, 1, 2], [3, 4]] and packed == one
    # image i's noise is that of a generator seeded with 11 + i, drawn in generate_views' order for its own elevation
    for i, (fp, polar) in one:
        assert polar == polars[i]
        assert fp == _fingerprint(zero123.image_noise(11 + i, 0, polars[i], N1, N2, "cpu"))
    assert len({tuple(fp) for _, (fp, _) in one}) == 5

    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, 29531, out), nprocs=world, join=True)
    (r0, c0), (r1, c1) = out[0], out[1]
    assert c0 == [[0, 2], [4]] and c1 == [[1, 3]]
    assert sorted(r0 + r1) == one
