"""CPU: the camera layer of the any-camera renderer (synthetic.normalise_cameras / orbit_cameras) against the reference
dataset's own cameras (tests/golden/views_mini.npz, oracle/pin_views_against_reference.py), the turntable command line,
and the argument checks of the ABI-6 entry points."""
import os
import sys

import numpy as np
import pytest

from o2345 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gv():
    return np.load(os.path.join(ROOT, "tests", "golden", "views_mini.npz"))


def test_stage1_cameras_match_the_reference_dataset(gv):
    meta = S.pose_json(60.0)
    cams = S.scene_cameras(meta)
    poses = np.array(list(meta["c2ws"].values()))
    c2w, K, nf = S.normalise_cameras(cams, poses[:8], meta["intrinsics"])
    assert c2w.shape == (8, 4, 4) and K.shape == (8, 3, 3) and nf.shape == (8, 2)
    np.testing.assert_allclose(np.linalg.inv(c2w.astype(np.float64)), gv["target_candidate_w2cs"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(c2w[0], gv["query_c2w"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(nf[0], gv["query_near_far"], rtol=0, atol=1e-5)
    # view 0 exactly as the sample dict holds it
    assert np.array_equal(c2w[0], cams["query_c2w"]) and np.array_equal(nf[0], cams["query_near_far"])
    assert np.array_equal(K[0], cams["query_intrinsic"])


def test_source_views_reproduce_the_scene_bit_for_bit():
    meta = S.pose_json(80.0)
    cams = S.scene_cameras(meta, n_src=6, img_wh=(64, 64))
    poses = np.array(list(meta["c2ws"].values()))
    c2w, _, nf = S.normalise_cameras(cams, poses[8:14], meta["intrinsics"])
    assert np.array_equal(c2w, cams["c2ws"]) and np.array_equal(nf, cams["near_fars"][1:])


def test_orbit_starts_at_the_input_view():
    for elev in (60.0, 100.0):
        meta = S.pose_json(elev)
        view0 = np.array(next(iter(meta["c2ws"].values())))
        orbit = S.orbit_cameras(meta, 36)
        assert orbit.shape == (36, 4, 4)
        np.testing.assert_allclose(orbit[0], view0, rtol=0, atol=1e-6)
        c = orbit[:, :3, 3].astype(np.float64)
        r = np.linalg.norm(c, axis=1)
        np.testing.assert_allclose(r, np.linalg.norm(view0[:3, 3]), rtol=1e-6)
        np.testing.assert_allclose(c[:, 2] / r, view0[2, 3] / r[0], atol=1e-6)       # constant elevation
        az = np.unwrap(np.arctan2(c[:, 0], -c[:, 1]))
        np.testing.assert_allclose(np.diff(az), 2 * np.pi / 36, atol=1e-5)           # evenly spaced azimuths
        # every camera looks at the origin (Blender: the camera looks along -z)
        fwd = -orbit[:, :3, 2]
        np.testing.assert_allclose(np.einsum("ij,ij->i", fwd, -c / r[:, None]), 1.0, atol=1e-5)


def test_turntable_arguments():
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import exp_runner_generic_blender_val as runner
    args = runner.parse_args(["--specific_dataset_name", "exp/x", "--mode", "turntable"])
    assert args.mode == "turntable" and args.n_frames == 36 and args.specific_dataset_name == "exp/x"
    assert runner.parse_args(["--mode", "turntable", "--n_frames", "12"]).n_frames == 12
    assert runner.parse_args([]).mode == "export_mesh"
    for bad in (["--mode", "train"], ["--mode", "turntable", "--n_frames", "0"]):
        with pytest.raises(SystemExit):
            runner.parse_args(bad)


def test_abi6_argument_checks_without_touching_the_gpu():
    import ctypes as C
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    views = _lib.Views(V=4, H=8, W=8, maps=0x1000, proj=0x1000, centers=0x1000)
    # dir_mode 2 takes the direction from each sample's ray: explicit points have none
    assert lib.o2345_render_blend(C.byref(_lib.Points(mode=_lib.PTS_EXPLICIT, pts=0x1000)), 4, None, fake, fake, 8,
                                  C.byref(views), 2, None, None, fake, _lib.BLEND_TC_FP16, fake, None, None) == -1
    assert "ray" in _lib.last_error()
    for prec in (_lib.BLEND_FP32, _lib.BLEND_TC_FP16):
        assert lib.o2345_render_blend(C.byref(_lib.Points(mode=_lib.PTS_EXPLICIT, pts=0x1000)), 4, None, fake, fake, 8,
                                      C.byref(views), 2, fake, None, fake, prec, fake, None, None) == -1
    # unknown dir_mode
    assert lib.o2345_render_blend(C.byref(_lib.Points(mode=_lib.PTS_RAYS)), 4, None, fake, fake, 8, C.byref(views), 3, fake,
                                  fake, fake, _lib.BLEND_TC_FP16, fake, None, None) == -1
    # the per-ray last section is required
    assert lib.o2345_ray_midpoints_per_ray(fake, fake, 4, fake, 8, None, fake, 8, fake, fake, fake, None) == -1
    assert len(_lib.last_error()) > 0
