"""GPU: VAE decode / encode on the wgmma path against the reference goldens (fp16 storage: see test_gpu_unet.py)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def vae():
    from o2345 import synthetic as S
    from o2345.autoencoder import AutoencoderKL
    net = AutoencoderKL()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in S.vae_state().items()})
    return net.cuda().requires_grad_(False)


def test_decode_and_encode_match_reference(vae):
    from oracle.pin_vae_against_reference import vae_inputs
    gold = np.load(os.path.join(ROOT, "tests", "golden", "vae_mini.npz"))
    z, x = vae_inputs()
    img = vae.decode(torch.from_numpy(z).cuda())
    assert img.shape == (1, 3, 256, 256)
    err = (img.cpu()[:, :, ::4, ::4] - torch.from_numpy(gold["dec"])).abs()
    print("decode: max", float(err.max()), "mean", float(err.mean()))
    assert float(err.max()) < 1.8e-2 and float(err.mean()) < 3e-3       # 3x the measured 5.8e-3 max (images in [-1, 1])
    post = vae.encode(torch.from_numpy(x).cuda())
    m = torch.cat([post.mean, post.logvar], 1)
    err = (m.cpu() - torch.from_numpy(gold["moments"])).abs()
    print("encode: max", float(err.max()), "mean", float(err.mean()))
    assert post.mode().shape == (1, 4, 32, 32)
    assert float(err.max()) < 1.8e-2 and float(err.mean()) < 3e-3


def test_vae_oracle_agrees_on_another_input(vae):
    from o2345 import synthetic as S
    from oracle import vae_oracle as VO
    sd = {k: torch.from_numpy(v) for k, v in S.vae_state().items()}
    g = torch.Generator().manual_seed(9)
    z = torch.randn(2, 4, 32, 32, generator=g)
    want = VO.decode(sd, z)
    got = vae.decode(z.cuda()).cpu()
    assert float((got - want).abs().max()) < 0.06
