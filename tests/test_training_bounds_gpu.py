"""The loss, post-op, backward-sum and optimizer kernels against fp64 references, element by element, under the
bounds derived in tests/training_bounds.py.  Each case asserts max(|got - ref| / bound) <= 1 and prints that ratio;
masks, counts, the latent mask, skipped steps and the state block's integer fields are compared exactly.  The shapes
follow the fixed-order cluster reductions (cluster_reduce.cuh): one CTA per 4096 pixels of an image up to 8, one per
4096 elements of a batch-wide sum up to 16, and the shares' edges."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import training_bounds as TB  # noqa: E402
from test_training_bounds_cpu import (BETAS, EPS, GROUP_LRS, GROUP_WDS, adamw_inputs, angular_inputs,  # noqa: E402
                                      decode_post_inputs, group_table, latent_inputs, per_element, ssi_inputs)

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, F32 = torch.float16, torch.float32


def _check(what, got, ref, bound):
    r = TB.bound_ratio(got.cpu(), ref, bound)
    print(f"{what}: max err / bound {r:.3g}")
    assert r <= 1.0, f"{what}: max err / bound {r:.3g}"
    return r


def _go(v):
    return torch.tensor(v, dtype=F32, device=DEV)


# ------------------------------------------------------------------------------------------------ SSI
_HWS = [1, 511, 4095, 4096, 4097, 8 * 4096 + 1, 480 * 640, 352 * 1216, 768 * 768]
SSI_CASES = [(B, HW, "random") for HW in _HWS for B in (1, 2, 5)] + [(1, 2048 * 2048, "random")]
SSI_CASES += [(1, 16 * 4096 - 1, "random"), (1, 16 * 4096 + 1, "random")]
SSI_CASES += [(B, HW, r) for HW in (4097, 8 * 4096 + 1, 480 * 640) for B in (2, 5)
              for r in ("small_s", "exact", "exact_mixed", "const", "one_pixel", "last_pixel", "last_share",
                        "one_empty", "all_empty")]


@pytest.mark.parametrize("B,HW,regime", SSI_CASES)
def test_ssi_loss_and_backward_within_bound(B, HW, regime):
    from diffusion_e2e_ft_b200 import ops
    p, y, m = ssi_inputs(B, HW, regime, seed=B + HW)
    pd, yd, md = (t.reshape(B, 1, 1, HW).to(DEV) for t in (p, y, m))
    loss = ops.ssi_loss(pd, yd, md)
    ref, bound = TB.ssi_loss_ref_bound(p, y, m)
    tag = f"ssi B={B} HW={HW} {regime}"
    if regime == "all_empty":
        assert torch.isnan(loss).item()
    else:
        _check(tag + " loss", loss, ref, bound)
    for go in (1.0, 1024.0, 2.0 ** 20):
        g = ops.ssi_loss_bwd(pd, yd, md, _go(go)).reshape(B, HW)
        ref, bound = TB.ssi_bwd_ref_bound(p, y, m, go)
        assert (g.cpu()[~m] == 0).all()
        if regime in ("exact", "all_empty", "const", "one_pixel", "last_pixel"):
            assert (g == 0).all(), f"{tag}: the gradient must be exactly 0"
        _check(f"{tag} grad go={go}", g, ref, bound)


# ------------------------------------------------------------------------------------------------ angular
ANG_CASES = [(B, HW, "random") for B, HW in ((1, 1), (2, 511), (5, 4097), (1, 16 * 4096 - 1), (1, 16 * 4096 + 1),
                                             (4, 16 * 4096 + 1), (5, 480 * 640), (1, 2048 * 2048))]
ANG_CASES += [(2, 4097, "near_one"), (1, 16 * 4096 + 1, "near_one"), (2, 4097, "identical")]


@pytest.mark.parametrize("B,HW,regime", ANG_CASES)
def test_angular_loss_and_backward_within_bound(B, HW, regime):
    from diffusion_e2e_ft_b200 import ops
    p, y, m = angular_inputs(B, HW, regime, seed=B + HW)
    pd, yd = (t.reshape(B, 3, 1, HW).to(DEV) for t in (p, y))
    md = m.reshape(B, 1, 1, HW).to(DEV)
    tag = f"angular B={B} HW={HW} {regime}"
    ref, bound = TB.angular_loss_ref_bound(p, y, m)
    _check(tag + " loss", ops.angular_loss(pd, yd, md), ref, bound)
    for go in (1.0, 2.0 ** 20):
        g = ops.angular_loss_bwd(pd, yd, md, _go(go)).reshape(B, 3, HW)
        ref, bound = TB.angular_bwd_ref_bound(p, y, m, go)
        if regime == "identical":                     # d = 1: torch's gradient is -inf / NaN, the kernel's is 0
            assert (g == 0).all()
        _check(f"{tag} grad go={go}", g, ref, bound)


# ------------------------------------------------------------------------------------------------ decode_post
@pytest.mark.parametrize("normals", [False, True])
@pytest.mark.parametrize("NB,H,W,regime", [(2, 9, 13, "edges"), (3, 480, 640, "random"), (1, 352, 1216, "edges")])
def test_decode_post_and_backward_within_bound(normals, NB, H, W, regime):
    from diffusion_e2e_ft_b200 import ops
    x = decode_post_inputs(NB, H, W, regime, seed=H)
    dout = torch.randn(NB, 3 if normals else 1, H, W, generator=torch.Generator().manual_seed(W))
    tag = f"decode_post {'normals' if normals else 'depth'} {NB}x{H}x{W} {regime}"
    out = ops.decode_post(x.to(DEV), normals=normals, training=True)
    _check(tag, out, *TB.decode_post_ref_bound(x, normals))
    dx = ops.decode_post_bwd(x.to(DEV), dout.to(DEV), normals=normals)
    _check(tag + " bwd", dx, *TB.decode_post_bwd_ref_bound(x, dout, normals))


# ------------------------------------------------------------------------------------------------ latent MSE
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("B,C,H,W,regime", [(1, 4, 70, 93, "random"), (2, 4, 96, 128, "block_edges"),
                                            (2, 4, 64, 64, "empty"), (2, 4, 355, 1219, "random"),
                                            (5, 4, 768, 768, "random")])
def test_masked_latent_mse_within_bound(dtype, B, C, H, W, regime):
    from diffusion_e2e_ft_b200 import ops
    pred, tgt, vm = latent_inputs(B, C, H, W, dtype, regime, seed=H + W)
    loss, lm, ws = ops.masked_latent_mse(pred.to(DEV), tgt.to(DEV), vm[:, None].to(DEV))
    ref, bound, lm_ref = TB.masked_latent_mse_ref_bound(pred, tgt, vm)
    assert torch.equal(lm.cpu().bool(), lm_ref)
    assert ws[1].item() == 2 * C * int(lm_ref.sum())
    tag = f"latent mse {B}x{C}x{H}x{W} {regime} {dtype}"
    if regime == "empty":
        assert loss.item() == 0.0
    _check(tag, loss, ref, bound)
    g = ops.masked_latent_mse_bwd(pred.to(DEV), tgt.to(DEV), lm, ws, _go(1024.0))
    assert g.dtype == dtype
    _check(tag + " bwd", g, *TB.masked_latent_mse_bwd_ref_bound(pred, tgt, lm_ref, 1024.0))


# ------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("silu", [True, False])
def test_act_bwd_every_f16_within_bound(silu):
    """Every finite fp16 x, with random dy."""
    from diffusion_e2e_ft_b200 import ops
    from test_training_bounds_cpu import all_finite_f16
    x = all_finite_f16()
    dy = torch.randn(x.shape, generator=torch.Generator().manual_seed(1)).half()
    act = ops.ACT_SILU if silu else ops.ACT_GELU
    got = ops.act_bwd(x.to(DEV), dy.to(DEV), act)
    _check(f"act_bwd {'silu' if silu else 'gelu'} every fp16", got, *TB.act_bwd_ref_bound(x, dy, silu))


@pytest.mark.parametrize("inner", [1, 320, 1280])
def test_geglu_bwd_every_f16_within_bound(inner):
    """Every finite fp16 gate value, strided [rows, 2 inner] value / gate halves and gradient halves."""
    from diffusion_e2e_ft_b200 import ops
    from test_training_bounds_cpu import all_finite_f16
    gv = all_finite_f16()
    rows = -(-gv.numel() // inner)
    gen = torch.Generator().manual_seed(inner)
    g = torch.cat([gv, torch.randn(rows * inner - gv.numel(), generator=gen).half()]).reshape(rows, inner)
    h = (torch.randn(rows, inner, generator=gen) * 4).half()
    dy = ((torch.rand(rows, inner, generator=gen) * 2 - 1) * 0.99).half()   # |dy gelu(g)| stays below fp16's max
    d = ops.geglu_bwd(torch.cat([h, g], 1).to(DEV).contiguous(), dy.to(DEV))
    rb = TB.geglu_bwd_ref_bound(h, g, dy)
    _check(f"geglu_bwd inner={inner} dh", d[:, :inner], *rb["dh"])
    _check(f"geglu_bwd inner={inner} dg", d[:, inner:], *rb["dg"])


# ------------------------------------------------------------------------------------------------ sums
@pytest.mark.parametrize("rows,C,ld,dtype", [(7, 4, 4, F32), (511, 40, 43, F16), (513, 72, 72, F32),
                                             (4097, 1280, 1290, F16), (40000, 40, 48, F32), (2 * 4096 + 1, 72, 80, F16)])
def test_col_sum_within_bound(rows, C, ld, dtype):
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, ld, generator=g).to(dtype)[:, :C]
    out0 = torch.randn(C, generator=g)
    got = ops.col_sum(x.to(DEV), out0.to(DEV).clone())
    R = TB.cluster_ctas(rows, 512)
    _check(f"col_sum rows={rows} C={C} ld={ld} {dtype} R={R}", got, *TB.col_sum_ref_bound(x, out0))


@pytest.mark.parametrize("hw,ohw", [((6, 6), (12, 12)), ((12, 12), (23, 23)), ((23, 23), (45, 45)),
                                    ((7, 7), (15, 15)), ((1, 1), (3, 3)), ((12, 23), (23, 45))])
@pytest.mark.parametrize("with_add", [False, True])
def test_upsample_nearest_bwd_within_bound(hw, ohw, with_add):
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(ohw[0])
    dy = torch.randn(2, ohw[0], ohw[1], 8, generator=g)
    add = torch.randn(2, hw[0], hw[1], 8, generator=g) if with_add else None
    got = ops.upsample_nearest_bwd(dy.to(DEV), hw, None if add is None else add.to(DEV))
    _check(f"upsample_nearest_bwd {hw}->{ohw} add={with_add}", got, *TB.upsample_nearest_bwd_ref_bound(dy, hw, add))


# ------------------------------------------------------------------------------------------------ optimizer
@pytest.mark.parametrize("n", [1, 3, 5, 4 * 16384 - 1, 4 * 16384 + 1, 4 * 16384 * 3 + 1, 4 * 16384 * 16 - 1,
                               4 * 16384 * 16 + 1, 4 * 16384 * 17 + 3, 10 ** 8 + 3])
def test_sumsq_within_bound(n):
    from diffusion_e2e_ft_b200 import ops
    x = torch.randn(n, generator=torch.Generator().manual_seed(n))
    got = ops.grad_norm_sq(x.to(DEV))
    _check(f"sumsq n={n}", got[0], *TB.sumsq_ref_bound(x))


def _state(S, step_before, skipped=0.0):
    return torch.tensor([S, 0.0, float(step_before), skipped, 0.0, 0.0, 0.0, 0.0], dtype=F32, device=DEV)


def _check_adamw(tag, bufs, rb):
    for name, got in zip(("param", "exp_avg", "exp_avg_sq"), bufs):
        _check(f"{tag} {name}", got, *rb[name])


ADAMW_CASES = [(step, clipped, 4099) for step in (1, 2, 3, 10, 1000, 30000) for clipped in (False, True)]
ADAMW_CASES += [(2, True, n) for n in (4097, 4098, 4099 + 262144)] + [(10, False, 132 * 8 * 1024 * 4 + 7)]


@pytest.mark.parametrize("step,clipped,n", ADAMW_CASES)
def test_adamw_state_groups_within_bound(step, clipped, n):
    """16 groups and up to 1024 runs, run starts just below / above float4 and 256-thread boundaries; the state block
    sets the step count; its integer fields are exact, clip / bc1 / bc2 within their bounds."""
    from diffusion_e2e_ft_b200 import ops
    p, g, m, v = adamw_inputs(n, step + n)
    S, W = 1024.0, 1.0
    g = g * S
    starts, groups = group_table(n, 16, min(1024, n // 4))
    lrs, wds = [TB.f32(x) for x in GROUP_LRS], [TB.f32(x) for x in GROUP_WDS]
    lr_e, wd_e = per_element(lrs, starts, groups, n), per_element(wds, starts, groups, n)
    dev = [t.to(DEV).contiguous() for t in (p, g, m, v)]
    nsq_t = ops.grad_norm_sq(dev[1])
    nsq = nsq_t.item()
    max_norm = 0.05 if clipped else 0.0
    clip = TB.clip_ref(nsq, max_norm, scale=S, inv_world=W)
    assert (clip < 1 / S) == clipped
    rs, rg = ops.adamw_run_table(starts, groups, n, 16, DEV)
    state = _state(S, step - 1)
    ops.adamw_step_state_groups(*dev, state, nsq_t, rs, rg, lrs, wds, betas=BETAS, eps=EPS, max_grad_norm=max_norm,
                                inv_world=W, dynamic_scale=False)
    st = state.cpu()
    assert st[2].item() == step and st[3].item() == 0 and st[4].item() == 0 and st[0].item() == S
    assert abs(st[5].item() - clip) <= TB.E_C * clip, (st[5].item(), clip)
    for k in (0, 1):
        ref, b = TB.bias_correction_ref_bound(BETAS[k], step)
        err = abs(st[6 + k].item() - ref)
        print(f"bc{k + 1} step {step}: err / bound {err / b:.3g}")
        assert err <= b, f"state[{6 + k}] = 1 - beta{k + 1}^{step}: off by {err:.3g} > {b:.3g}"
    rb = TB.adamw_ref_bound(p, g, m, v, step, lr_e.double(), wd_e.double(), BETAS, EPS, clip)
    _check_adamw(f"adamw groups step={step} clip={clipped} n={n}", dev[0:1] + dev[2:4], rb)


def test_adamw_state_skips_nonfinite_step_bitwise():
    from diffusion_e2e_ft_b200 import ops
    n = 4099
    p, g, m, v = adamw_inputs(n, 1)
    dev = [t.to(DEV).contiguous() for t in (p, g, m, v)]
    before = [t.clone() for t in dev]
    state = _state(1024.0, 5, skipped=2.0)
    ops.adamw_step_state(*dev, state, torch.tensor([float("inf")], dtype=torch.float64, device=DEV),
                         dynamic_scale=True)
    st = state.cpu()
    assert st.tolist()[:5] == [512.0, 0.0, 5.0, 3.0, 1.0]
    assert all(torch.equal(a, b) for a, b in zip(dev, before))


@pytest.mark.parametrize("step,unscale,max_norm", [(1, 1.0, 0.0), (2, 1 / 1024, 0.0), (3, 1 / 4096, 0.05),
                                                   (1000, 1 / 65536, 1.0)])
def test_adamw_step_scaled_within_bound(step, unscale, max_norm):
    """The legacy entry point: step count and 1 / loss scale passed from the host."""
    from diffusion_e2e_ft_b200 import ops
    n = 4 * 1031 + 3
    p, g, m, v = adamw_inputs(n, step)
    g = g / unscale
    dev = [t.to(DEV).contiguous() for t in (p, g, m, v)]
    nsq_t = ops.grad_norm_sq(dev[1])
    ops.adamw_step(*dev, step, lr=3e-5, betas=BETAS, eps=EPS, weight_decay=1e-2, grad_norm_sq_t=nsq_t,
                   max_grad_norm=max_norm, grad_unscale=unscale)
    clip = TB.clip_ref(nsq_t.item(), max_norm, scale=1.0 / TB.f32(unscale))
    rb = TB.adamw_ref_bound(p, g, m, v, step, 3e-5, 1e-2, BETAS, EPS, clip)
    _check_adamw(f"adamw scaled step={step} unscale={unscale} max_norm={max_norm}", dev[0:1] + dev[2:4], rb)


@pytest.mark.parametrize("n", [1, 6, 4099, 132 * 8 * 256 * 4 + 5])
def test_ema_update_bitwise(n):
    """b200_ema_update against torch's fp32 ema.sub_(omd * (ema - p)), bit for bit."""
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(n)
    ema, p = torch.randn(n, generator=g).to(DEV), torch.randn(n, generator=g).to(DEV)
    omd = 1 - 0.9999 ** 0.75
    ref = ema.clone()
    ref.sub_(torch.tensor(TB.f32(omd), dtype=F32, device=DEV) * (ref - p))
    ops.ema_update(ema, p, omd)
    assert torch.equal(ema, ref)
