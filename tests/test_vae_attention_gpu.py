"""-m gpu: the d=512 flash attention of the VAE mid-block (`ops.attention_d512`) and the memory-efficient VAE path it
serves: kernel against a chunked fp32 reference and against the unfused path, the full-size VAE against the fp32
oracle, native-resolution pipelines up to 12 MP, and the per-image size limit."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import engine_checks as EC  # noqa: E402

pytestmark = pytest.mark.gpu

GB = 1024 ** 3


def _need_free(nbytes, what):
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB free; the device has {free / GB:.1f} of {total / GB:.1f} GB free")


def _qkv(B, L, seed):
    """One fused [B, L, 1536] projection buffer; q, k, v are strided views of it (as the module passes them)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = (torch.randn(B, L, 1536, device="cuda", generator=g) * 1.5).half()
    return buf, buf[..., :512], buf[..., 512:1024], buf[..., 1024:]


def _reference(q, k, v, scale, rows=None, chunk=1024):
    """fp32 softmax(q k^T scale) v, computed over query chunks (never a full L x L matrix)."""
    B, L = q.shape[:2]
    rows = torch.arange(L, device=q.device) if rows is None else rows
    out = torch.empty(B, rows.numel(), 512, device=q.device)
    kf, vf = k.float(), v.float()
    for i in range(0, rows.numel(), chunk):
        r = rows[i:i + chunk]
        s = torch.einsum("bqd,bkd->bqk", q[:, r].float(), kf) * scale
        out[:, i:i + chunk] = torch.softmax(s, dim=-1) @ vf
    return out


def _unfused(q, k, v, scale):
    """The unfused VAEAttention path on the same operands: S = QK^T fp32, row softmax -> fp16 P, O = P V."""
    from diffusion_e2e_ft_b200 import ops
    B, L = q.shape[:2]
    Lp = (L + 7) // 8 * 8
    vt_buf = torch.zeros((B, 512, Lp), dtype=torch.float16, device=q.device)
    vt_buf[:, :, :L] = v.transpose(1, 2)
    s_buf = torch.empty((B, L, Lp), dtype=torch.float32, device=q.device)
    ops.linear(q, k, out=s_buf[:, :, :L])
    p_buf = ops.softmax_rows(s_buf, scale, cols=L)
    del s_buf
    return ops.linear(p_buf[:, :, :L], vt_buf[:, :, :L])


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("L", [1, 37, 64, 9216, 9217, 32400])
def test_attention_d512_matches_fp32_reference_and_unfused_path(B, L):
    from diffusion_e2e_ft_b200 import ops
    if L == 32400:
        _need_free(B * L * L * 6 + 4 * GB, "the unfused comparison at L=32400")
    _, q, k, v = _qkv(B, L, seed=L + B)
    scale = 512 ** -0.5
    got = ops.attention_d512(q, k, v, scale)
    assert got.shape == (B, L, 512) and got.dtype == torch.float16
    want = _reference(q, k, v, scale)
    r_ref = EC.rel_l2(got, want)
    r_unf = EC.rel_l2(got, _unfused(q, k, v, scale))
    print(f"B={B} L={L}: rel-L2 vs fp32 {r_ref:.2e}, vs unfused {r_unf:.2e}")
    assert torch.isfinite(got).all()
    assert r_ref <= 2e-3 and r_unf <= 1e-3, (r_ref, r_unf)


def test_attention_d512_separate_outputs_and_padded_strides():
    """Contiguous q / k / v of different lengths (Lq != Lk) and an output with a padded row stride."""
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(2, 100, 512, device="cuda", generator=g).half()
    k = torch.randn(2, 333, 512, device="cuda", generator=g).half()
    v = torch.randn(2, 333, 512, device="cuda", generator=g).half()
    out_buf = torch.full((2, 100, 520), 7.0, dtype=torch.float16, device="cuda")
    ops.attention_d512(q, k, v, 0.05, out=out_buf[..., :512])
    assert EC.rel_l2(out_buf[..., :512], _reference(q, k, v, 0.05)) <= 2e-3
    assert (out_buf[..., 512:] == 7.0).all()                   # nothing written past the 512 columns


def test_attention_d512_large_L_has_no_quadratic_buffer():
    """One VAE attention call at 4K UHD (L = 129600): matches the chunked reference on a sample of query rows, and
    its peak allocation is its output (no L x L scores)."""
    from diffusion_e2e_ft_b200 import ops
    L = 129600
    _need_free(4 * GB, "the L=129600 attention call")
    buf, q, k, v = _qkv(1, L, seed=11)
    scale = 512 ** -0.5
    out = torch.empty((1, L, 512), dtype=torch.float16, device="cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ops.attention_d512(q, k, v, scale, out=out)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    print(f"L={L}: peak allocation during the call {extra} B beyond inputs ({buf.numel() * 2} B) and output "
          f"({out.numel() * 2} B)")
    assert extra <= 256 * 1024 ** 2
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = torch.cat([torch.arange(0, 512, device="cuda"), torch.arange(L - 512, L, device="cuda"),
                      torch.randint(0, L, (1024,), device="cuda", generator=g)])
    want = _reference(q, k, v, scale, rows=rows, chunk=512)
    r = EC.rel_l2(out[:, rows], want)
    print(f"L={L}: rel-L2 vs fp32 on {rows.numel()} rows {r:.2e}")
    assert r <= 2e-3


def _full_vae():
    from oracle.unet import seeded_init
    from oracle.vae import AutoencoderKLRef, VAEConfig
    from diffusion_e2e_ft_b200 import B200AutoencoderKL
    vref = seeded_init(AutoencoderKLRef(VAEConfig()), seed=99).eval()
    vae = B200AutoencoderKL(block_out_channels=vref.config.block_out_channels)
    vae.load_state_dict(vref.state_dict(), strict=True)
    return vref.cuda(), vae.cuda().eval().requires_grad_(False)


@torch.no_grad()
def test_full_vae_768_memory_efficient_matches_oracle_and_default_is_unchanged():
    from oracle import pipeline as OP
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    vref, vae = _full_vae()
    g = torch.Generator().manual_seed(7)
    rgb = (torch.rand(1, 3, 768, 768, generator=g) * 2 - 1).cuda()
    z = (torch.randn(1, 4, 96, 96, generator=g) * 0.5).cuda()
    enc0 = vae.encode_scaled_mean(rgb)
    dec0 = vae.decoder(vae.post_quant_conv(z))
    vae.enable_xformers_memory_efficient_attention()
    enc1 = vae.encode_scaled_mean(rgb)
    dec1 = vae.decoder(vae.post_quant_conv(z))
    vae.disable_xformers_memory_efficient_attention()
    enc2 = vae.encode_scaled_mean(rgb)
    dec2 = vae.decoder(vae.post_quant_conv(z))
    assert torch.equal(enc0, enc2) and torch.equal(dec0, dec2)       # disabled: bit-identical to the default path
    want_enc = OP.encode_rgb(vref, rgb)
    want_dec = vref.decoder(vref.post_quant_conv(z))
    r = dict(enc=EC.rel_l2(enc1, want_enc), dec=EC.rel_l2(dec1, want_dec),
             enc_default=EC.rel_l2(enc0, want_enc), dec_default=EC.rel_l2(dec0, want_dec),
             enc_vs_default=EC.rel_l2(enc1, enc0), dec_vs_default=EC.rel_l2(dec1, dec0))
    print(r)
    assert r["enc"] <= 3e-3 and r["dec"] <= 3e-3, r


def _full_pipeline():
    from oracle.unet import UNet2DConditionRef, UNetConfig, seeded_init
    from oracle.vae import AutoencoderKLRef, VAEConfig
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    uref = seeded_init(UNet2DConditionRef(UNetConfig()), seed=4321).eval()
    vref = seeded_init(AutoencoderKLRef(VAEConfig()), seed=99).eval()
    unet, vae = EC.engine_from_oracle(uref, vref, "cuda")
    ete = (torch.randn(1, 2, 1024, generator=torch.Generator().manual_seed(7)) * 0.5).cuda()
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=ete)
    pipe.use_cuda_graph = False                 # a captured graph would keep a second copy of every activation
    return pipe


def _image(h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g)


def _depth(pipe, img):
    return pipe(img, denoising_steps=1, ensemble_size=1, processing_res=0, noise="zeros",
                show_progress_bar=False).depth_np


@torch.no_grad()
def test_pipeline_1080p_native_resolution_both_paths_agree():
    _need_free(30 * GB, "the 1920x1080 pipeline")
    pipe = _full_pipeline()
    img = _image(1080, 1920)
    d_default = _depth(pipe, img)
    pipe.enable_xformers_memory_efficient_attention()
    d_fused = _depth(pipe, img)
    pipe.disable_xformers_memory_efficient_attention()
    r = float(np.linalg.norm(d_fused - d_default) / np.linalg.norm(d_default))
    print(f"1080p depth, memory-efficient vs default: rel-L2 {r:.2e}")
    assert d_fused.shape == (1080, 1920) and r <= 2e-3


@torch.no_grad()
def test_pipeline_4k_native_resolution():
    _need_free(40 * GB, "the 3840x2160 pipeline")
    pipe = _full_pipeline()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    d = _depth(pipe, _image(2160, 3840, seed=1))
    print(f"4K UHD depth: peak allocation {torch.cuda.max_memory_allocated() / GB:.1f} GB")
    assert d.shape == (2160, 3840) and np.isfinite(d).all() and d.min() >= 0.0 and d.max() <= 1.0


def test_pipeline_rejects_images_over_the_per_image_limit_before_launching():
    pipe = _full_pipeline()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="processing_res"):
        _depth(pipe, torch.zeros((3, 4000, 6000), dtype=torch.uint8))        # 24 MP
    assert torch.cuda.memory_allocated() == before


@torch.no_grad()
def test_pipeline_12mp_native_resolution():
    """4032 x 3024: the decoder's 256-channel full-resolution tensors hold 3.1e9 elements (over 2^31)."""
    _need_free(60 * GB, "the 4032x3024 pipeline")
    pipe = _full_pipeline()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    d = _depth(pipe, _image(3024, 4032, seed=2))
    print(f"12 MP depth: peak allocation {torch.cuda.max_memory_allocated() / GB:.1f} GB")
    assert d.shape == (3024, 4032) and np.isfinite(d).all() and d.min() >= 0.0 and d.max() <= 1.0
