"""GPU tests of GeoWizard's SD-1-shaped UNet: the flash kernel, rowdot and the attention backward at head widths 40,
80 and 160 against fp64 torch, and the tiny / full-size SD-1 UNet (1x1-conv projections, joint attention) against the
fp32 oracle and its autograd.  Tolerances are those of the head-width-64 checks (tests/kernel_checks.py,
tests/bwd_checks.py, tests/test_multistep_gpu.py)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = torch.float16
LENGTHS = [1, 77, 127, 128, 129, 2304]


def _rand(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(F16).to(DEV)


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _split(t, heads):
    return t.double().unflatten(-1, (heads, -1)).transpose(1, 2)


def _joint(t):
    t0, t1 = t.chunk(2, 0)
    return torch.cat([torch.cat([t0, t1], 2)] * 2, 0)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("D", [40, 80, 160])
@pytest.mark.parametrize("Lq", LENGTHS)
@pytest.mark.parametrize("Lk", LENGTHS)
@pytest.mark.parametrize("kv_segments", [1, 2])
def test_flash_forward_and_lse_vs_fp64(D, Lq, Lk, kv_segments):
    """Q / K / V as head slices of fused [B, L, 3C] projection buffers (row stride 3C), 8 heads as in SD-1."""
    from diffusion_e2e_ft_b200 import ops
    B, heads = 2, 8
    C = heads * D
    qkv = _rand(B, Lq, 3 * C, seed=D + Lq)
    kvb = qkv if Lk == Lq else _rand(B, Lk, 3 * C, seed=D + Lk + 1)
    q, k, v = qkv[..., :C], kvb[..., C:2 * C], kvb[..., 2 * C:]
    scale = D ** -0.5 * 2.0                                       # logit std ~2: a softmax that is not uniform
    out, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)
    torch.cuda.synchronize()
    qd, kd, vd = _split(q, heads), _split(k, heads), _split(v, heads)
    if kv_segments == 2:
        kd, vd = _joint(kd), _joint(vd)
    s = qd @ kd.transpose(-1, -2) * scale
    ref = (torch.softmax(s, -1) @ vd).transpose(1, 2).reshape(B, Lq, C)
    lse_ref = torch.logsumexp(s, -1) * 1.4426950408889634
    e_out = _rel_l2(out, ref)
    e_lse = ((lse.double() - lse_ref).abs().max() / lse_ref.abs().max().clamp_min(1.0)).item()
    assert e_out <= 2e-3 and e_lse <= 1e-5, (e_out, e_lse)


@pytest.mark.parametrize("D", [40, 64, 80, 160])
def test_rowdot_vs_fp64(D):
    from diffusion_e2e_ft_b200 import ops
    B, L, heads = 2, 300, 8
    C = heads * D
    a = _rand(B, L, 3 * C, seed=1)[..., C:2 * C]                  # strided view, as a slice of d(qkv)
    c = _rand(B, L, C, seed=2)
    got = ops.rowdot_heads_d(a, c, heads, D)
    ref = (_split(a, heads) * _split(c, heads)).sum(-1)
    assert _rel_l2(got, ref) <= 1e-5
    if D == 64:
        assert torch.equal(got, ops.rowdot_heads(a, c, heads))


@pytest.mark.parametrize("D", [40, 80, 160])
@pytest.mark.parametrize("T,Tk,fused", [(192, 192, True), (300, 300, True), (256, 77, False), (4, 77, False),
                                        (129, 1, False)])
def test_attention_bwd_vs_fp64_autograd(D, T, Tk, fused):
    from diffusion_e2e_ft_b200 import backward as bw
    B, heads = 2, 8
    C = heads * D
    scale = D ** -0.5
    if fused:
        qkv = _rand(B, T, 3 * C, seed=D + T)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:
        q = _rand(B, T, C, seed=D + T)
        kv = _rand(B, Tk, 2 * C, seed=D + Tk + 1)
        k, v = kv[..., :C], kv[..., C:]
    do = _rand(B, T, C, seed=D + 7)
    dq, dk, dv = bw.attention_bwd(q, k, v, do, heads, scale)
    torch.cuda.synchronize()
    qr, kr, vr = (_split(t, heads).detach().requires_grad_(True) for t in (q, k, v))
    o = torch.softmax(qr @ kr.transpose(-1, -2) * scale, dim=-1) @ vr
    (o * _split(do, heads)).sum().backward()
    back = lambda t: t.transpose(1, 2).flatten(2)
    if Tk == 1:                                                    # softmax over one key: exactly zero dQ / dK
        assert not dq.any() and not dk.any()
        assert _rel_l2(dv, back(vr.grad)) <= 3e-3
        return
    errs = [_rel_l2(a, back(b.grad)) for a, b in ((dq, qr), (dk, kr), (dv, vr))]
    assert max(errs) <= 3e-3, errs


# ------------------------------------------------------------------------------------------------ tiny graph
@pytest.fixture
def sd1(monkeypatch):
    import sd1_checks as S
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    S.sd1_tiny(monkeypatch)


@pytest.mark.parametrize("hw", [(16, 16), (15, 20)])
def test_tiny_sd1_geowizard_unet_backward_joint_attention(sd1, hw):
    import engine_checks as EC
    r = EC.run_unet_backward_tiny(device=DEV, hw=hw, kind="geowizard")
    print("tiny_sd1_backward", hw, r)
    assert not r["missing"], r["missing"]
    assert r["forward"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


@pytest.mark.parametrize("hw", [(16, 16), (15, 20)])
def test_tiny_sd1_general_and_constant_context_paths(sd1, hw):
    import engine_checks as EC
    r = EC.run_single_step_specialisations(device=DEV, hw=hw)
    print("tiny_sd1_paths", hw, r)
    assert r["general_vs_oracle"] <= 3e-3 and r["spec_vs_oracle"] <= 3e-3 and r["spec_vs_general"] <= 2e-3, r
    assert r["per_image_ctx_vs_oracle"] <= 3e-3 and r["repeat_call"] == 0.0, r


def test_tiny_sd1_gradient_checkpointing_matches_plain_backward(sd1):
    import engine_checks as EC
    r = EC.run_checkpointing_tiny(device=DEV)
    print("tiny_sd1_checkpointing", r)
    assert r["global_rel_diff"] <= 3e-3 and r["worst_rel_diff"] <= 1e-2, r
    assert r["ckpt_vs_oracle_global"] <= 1e-2, r


def test_tiny_sd1_e2e_ft_loss_geowizard_gradients(sd1):
    import engine_checks as EC
    r = EC.run_training_step_geowizard_tiny(device=DEV)
    print("tiny_sd1_e2e_ft_geowizard", r)
    assert not r["missing"], r["missing"]
    assert r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 6e-2 and r["grad_worst"] <= 0.2, r


def test_tiny_sd1_diffusion_loss_geowizard_gradients(sd1):
    import diffusion_training_checks as DTC
    r = DTC.run_diffusion_step_tiny(device=DEV)
    print("tiny_sd1_diffusion_geowizard", r)
    assert not r["missing"], r["missing"]
    assert r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


# ------------------------------------------------------------------------------------------------ full size
@pytest.mark.parametrize("steps,noise", [(1, "zeros"), (10, "gaussian")])
@torch.no_grad()
def test_full_size_sd1_geowizard_pipeline_vs_oracle(steps, noise):
    """768x768, SD-1 widths (320 / 640 / 1280 / 1280, 8 heads, context 768, conv projections), bs 1; the fp32 oracle
    runs with torch ops on this GPU."""
    import engine_checks as E
    import multistep_oracle as MO
    import sd1_checks as S
    from oracle.unet import seeded_init
    from oracle.vae import AutoencoderKLRef, VAEConfig
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = S.sd1_config(in_channels=8, class_embed_type="projection", projection_class_embeddings_input_dim=10,
                     joint_attention=True)
    uref = seeded_init(S.unet_ref(cfg), seed=4321).eval()
    vref = seeded_init(AutoencoderKLRef(VAEConfig()), seed=99).eval()
    unet, vae = S.engine_from_oracle_sd1(uref, vref, DEV)
    uref, vref = uref.to(DEV), vref.to(DEV)
    g = torch.Generator().manual_seed(7)
    rgb = (torch.rand(1, 3, 768, 768, generator=g) * 2 - 1).to(DEV)
    emb = (torch.randn(1, 1, 768, generator=g) * 0.5).to(DEV)
    pipe = DepthNormalEstimationPipeline(unet, vae, DDIMScheduler())
    torch.manual_seed(23)
    np.random.seed(23)
    d, n = pipe.single_infer(rgb, steps, "indoor", noise=noise, img_embed=emb)
    torch.manual_seed(23)
    init = torch.randn((1, 4, 96, 96), device=DEV) if noise == "gaussian" else None
    wd, wn = MO.geowizard_infer(uref, vref, MO.DDIMRef(), rgb, emb, "indoor", steps, init_latent=init)
    res = dict(depth_rel_l2=E.rel_l2(d, wd), normal_mean_angle_deg=E.mean_angle_deg(n, wn), **E.absrel_protocol(d, wd))
    print("full_size_sd1_geowizard", steps, noise, res)
    gd = 3e-3 if steps == 1 else 5e-3
    assert res["depth_rel_l2"] <= gd and res["normal_mean_angle_deg"] <= 0.5 and res["absrel_delta"] <= 1e-3, res
