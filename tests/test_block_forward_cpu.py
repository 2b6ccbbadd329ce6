"""The differentiable path (autograd_blocks.py) runs each block's own inference forward: a training forward gives the
inference result bit for bit, and the two share one packed-weight build per module.  Kernels emulated on CPU
(tests/cpu_emulation.py)."""
import pytest
import torch

import cpu_emulation
import engine_checks as EC
import make_golden as MG
from diffusion_e2e_ft_b200 import autograd_blocks as ab
from diffusion_e2e_ft_b200 import ops
from test_vae_attention_cpu import _attention_d512_emulated


@pytest.fixture
def emulated(monkeypatch):
    cpu_emulation.install(monkeypatch)
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)


def test_fused_vae_attention_after_a_differentiable_forward(emulated, monkeypatch):
    """A differentiable forward fills the packed-weight cache that the fused inference path then reads."""
    from diffusion_e2e_ft_b200.vae import VAEAttention
    monkeypatch.setattr(ops, "attention_d512", _attention_d512_emulated([]))
    torch.manual_seed(0)
    att = VAEAttention(512, 32).eval().requires_grad_(False)
    with torch.no_grad():
        for p in att.parameters():
            p.normal_(0, 0.05)
    x = torch.randn(2, 5, 7, 512)
    ab.vae_attention(att, x.clone().requires_grad_(True))
    with torch.no_grad():
        unfused = att.run(x)
        att.memory_efficient = True
        fused = att.run(x)
    rel = ((fused - unfused).norm() / unfused.norm()).item()
    assert rel <= 2e-3, rel


@pytest.mark.parametrize("ckpt", [False, True])
@pytest.mark.parametrize("hw", [(16, 16), (15, 20)])
@pytest.mark.parametrize("kind", ["marigold", "geowizard"])
def test_unet_training_forward_equals_inference_forward(emulated, kind, hw, ckpt):
    """(15, 20) is not a multiple of 2^3: the up path resizes to the skip sizes (Upsample2D's second branch)."""
    ref, _ = MG.build_tiny(kind)
    unet, _ = EC.engine_from_oracle(ref, None, "cpu")
    unet.single_step_specialisations = False
    if ckpt:
        unet.enable_gradient_checkpointing()
    x = MG.inputs(1, 2, 8, *hw)
    if kind == "geowizard":            # class-embedding projection, joint self-attention over the image pair
        c, kw = MG.inputs(2, 2, 1, 96, scale=0.5), dict(class_labels=MG.inputs(3, 2, 10, scale=0.5))
    else:
        c, kw = MG.inputs(2, 2, 77, 128, scale=0.5), {}
    with torch.no_grad():
        want = unet(x, 999, c, **kw).sample
    unet.requires_grad_(True)
    got = unet(x, 999, c, **kw).sample
    assert got.requires_grad and torch.equal(got.detach(), want)


def test_decoder_training_forward_equals_inference_forward(emulated):
    unet_ref, vae_ref = MG.build_tiny()
    _, vae = EC.engine_from_oracle(unet_ref, vae_ref, "cpu")
    z = MG.inputs(4, 2, 4, 8, 8, scale=0.5)
    with torch.no_grad():
        want = vae.decoder(z)
    got = vae.decoder(z.clone().requires_grad_(True))
    assert got.requires_grad and torch.equal(got.detach(), want)
