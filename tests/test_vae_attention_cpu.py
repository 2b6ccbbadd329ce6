"""CPU tests of the memory-efficient VAE attention: argument checks of the d=512 C entry point, the dispatch rule, the
diffusers `enable_/disable_xformers_memory_efficient_attention` surface, the per-image size limit, and the host wiring
of the fused path with the kernel emulated in this file."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ C ABI
def _d512(L, q=16, k=16, v=16, out=16, q_ls=1536, o_ls=512, B=1, Lq=64, Lk=64):
    return L.b200_attention_d512(q, q_ls * Lq, q_ls, k, 1536 * Lk, 1536, v, 1536 * Lk, 1536, out, o_ls * Lq, o_ls,
                                 B, Lq, Lk, 0.044, None)


def test_attention_d512_rejects_bad_arguments_without_launching():
    from diffusion_e2e_ft_b200 import lib
    L = lib.load()
    for kw in (dict(q=None), dict(k=None), dict(v=None), dict(out=None)):
        assert _d512(L, **kw) < 0 and b"null pointer" in L.b200_last_error_string()
    assert _d512(L, q_ls=1540) < 0 and b"multiples of 8" in L.b200_last_error_string()
    assert _d512(L, o_ls=504) < 0 and b">= 512" in L.b200_last_error_string()
    assert _d512(L, out=24) < 0 and b"16-byte aligned" in L.b200_last_error_string()
    for kw in (dict(Lq=0), dict(Lk=0), dict(B=0), dict(Lq=-3)):
        assert _d512(L, **kw) < 0 and b"bad shape" in L.b200_last_error_string()


# ------------------------------------------------------------------------------------------------ dispatch
def test_dispatch_rule():
    from diffusion_e2e_ft_b200.vae import use_fused_attention
    assert not use_fused_attention(8, 9216, 512)             # 768^2 bs 8: the headline keeps the unfused path
    assert not use_fused_attention(15, 16384, 512)           # 1024^2 bs 15
    assert not use_fused_attention(1, 32400, 512)            # 1920x1080
    assert not use_fused_attention(8, 32400, 512)            # batch offsets are 64-bit: B does not enter
    assert not use_fused_attention(1, 65528, 512)            # L * Lp = 4293918784 < 2^32 - 1
    assert use_fused_attention(1, 65536, 512)                # L * Lp = 2^32: b200_linear cannot index the scores
    assert use_fused_attention(1, 129600, 512)               # 3840x2160
    assert use_fused_attention(1, 190512, 512)               # 4032x3024
    assert use_fused_attention(8, 9216, 512, memory_efficient=True)
    assert use_fused_attention(1, 1, 512, memory_efficient=True)
    assert not use_fused_attention(1, 129600, 256)           # no flash kernel for other widths
    assert not use_fused_attention(8, 9216, 128, memory_efficient=True)


# ------------------------------------------------------------------------------------------------ diffusers API
def _tiny_vae():
    from diffusion_e2e_ft_b200 import B200AutoencoderKL
    return B200AutoencoderKL(block_out_channels=(32, 512), layers_per_block=1)


def _attns(vae):
    from diffusion_e2e_ft_b200.vae import VAEAttention
    return [m for m in vae.modules() if isinstance(m, VAEAttention)]


def test_vae_enable_disable_memory_efficient_attention():
    vae = _tiny_vae()
    attns = _attns(vae)
    assert len(attns) == 2 and not any(a.memory_efficient for a in attns)      # encoder + decoder, off by default
    vae.enable_xformers_memory_efficient_attention()
    assert all(a.memory_efficient for a in attns) and vae.memory_efficient_attention
    vae.disable_xformers_memory_efficient_attention()
    assert not any(a.memory_efficient for a in attns) and not vae.memory_efficient_attention
    vae.enable_xformers_memory_efficient_attention(attention_op=object())     # an xformers op is accepted, ignored
    assert all(a.memory_efficient for a in attns)


class _Spy:
    def __init__(self):
        self.calls = []

    def enable_xformers_memory_efficient_attention(self, attention_op=None):
        self.calls.append(("enable", attention_op))

    def disable_xformers_memory_efficient_attention(self):
        self.calls.append(("disable",))


@pytest.mark.parametrize("kind", ["marigold", "geowizard"])
def test_pipelines_forward_memory_efficient_attention(kind):
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline, MarigoldPipeline
    from diffusion_e2e_ft_b200.unet import B200UNet2DConditionModel
    vae, spy = _tiny_vae(), _Spy()
    sched = DDIMScheduler()
    if kind == "marigold":
        pipe = MarigoldPipeline(spy, vae, sched)
    else:
        pipe = DepthNormalEstimationPipeline(spy, vae, sched, image_encoder=None)
    assert hasattr(pipe, "enable_xformers_memory_efficient_attention")
    pipe.enable_xformers_memory_efficient_attention()
    assert spy.calls == [("enable", None)] and all(a.memory_efficient for a in _attns(vae))
    pipe.disable_xformers_memory_efficient_attention()
    assert spy.calls[-1] == ("disable",) and not any(a.memory_efficient for a in _attns(vae))
    # a registered module without the method (scheduler, missing encoder) is skipped; the UNet's stays a no-op
    assert B200UNet2DConditionModel.enable_xformers_memory_efficient_attention(None) is None


def test_pipeline_rejects_images_over_the_per_image_limit():
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    from diffusion_e2e_ft_b200.pipelines import _check_image_size
    _check_image_size(3024, 4032)                               # 12 MP: 3.1e9 < 2^32 elements
    _check_image_size(4096, 4095)
    with pytest.raises(ValueError, match="processing_res"):
        _check_image_size(4096, 4096)                           # 256 * H * W = 2^32
    pipe = MarigoldPipeline(_Spy(), _tiny_vae(), DDIMScheduler())
    with pytest.raises(ValueError, match="per-image limit of 16.8 MP"):            # raised before anything touches a device
        pipe(torch.zeros((3, 4000, 6000), dtype=torch.uint8), processing_res=0)
    with pytest.raises(ValueError):
        pipe(torch.zeros((3, 4000, 6000), dtype=torch.uint8), processing_res=6000)


# ------------------------------------------------------------------------------------------------ host wiring
def _attention_d512_emulated(calls):
    def attention_d512(q, k, v, scale, out=None):
        assert q.dtype == k.dtype == v.dtype == torch.float16
        assert q.shape[-1] == k.shape[-1] == v.shape[-1] == 512 and q.stride(-1) == 1
        for t in (q, k, v):                                     # what the C entry point checks
            assert t.stride(1) % 8 == 0 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0
        calls.append((q, k, v, scale))
        s = q.float() @ k.float().transpose(1, 2) * scale
        return (torch.softmax(s, dim=-1) @ v.float()).half()
    return attention_d512


@pytest.mark.parametrize("hw", [(8, 8), (5, 7)])
def test_fused_path_host_wiring(monkeypatch, hw):
    import cpu_emulation
    from diffusion_e2e_ft_b200 import ops
    from diffusion_e2e_ft_b200.vae import VAEAttention
    cpu_emulation.install(monkeypatch)
    calls = []
    monkeypatch.setattr(ops, "attention_d512", _attention_d512_emulated(calls))
    torch.manual_seed(0)
    att = VAEAttention(512, 32).eval()
    with torch.no_grad():
        for p in att.parameters():
            p.normal_(0, 0.05)
    x = torch.randn(2, *hw, 512)
    with torch.no_grad():
        default = att.run(x)
        assert not calls                                         # the default path does not touch the kernel
        att.memory_efficient = True
        fused = att.run(x)
    assert len(calls) == 1
    q, k, v, scale = calls[0]
    L = hw[0] * hw[1]
    assert q.shape == k.shape == v.shape == (2, L, 512) and scale == pytest.approx(512 ** -0.5)
    # q, k, v are views of ONE [B, L, 1536] QKV projection
    assert q.stride() == k.stride() == v.stride() == (L * 1536, 1536, 1)
    assert k.data_ptr() - q.data_ptr() == 512 * 2 and v.data_ptr() - q.data_ptr() == 1024 * 2
    assert fused.shape == default.shape and fused.dtype == default.dtype
    rel = ((fused - default).norm() / default.norm()).item()
    assert rel <= 2e-3, rel
    # the attention output matters: a fused run with a different V changes the result
    with torch.no_grad():
        att.to_v.weight.mul_(2.0)
        assert ((att.run(x) - fused).norm() / fused.norm()).item() > 1e-3
