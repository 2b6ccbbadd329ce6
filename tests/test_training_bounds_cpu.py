"""The per-element bounds of tests/training_bounds.py, checked without a GPU:
* not too tight: a CPU emulation of each kernel's documented arithmetic (fp32 where the kernel is fp32, fp64 sums in
  the kernel's cluster shares) stays within its bound at the shapes of the GPU cases;
* not too loose: each planted mutant (one pixel or one CTA share dropped from a moment sum, sign(0) taken as +1, the
  inclusive clamp test made exclusive, a neighbouring group's learning rate, the n % 4 tail skipped, the previous
  step's bc2, the fp32 bias correction) exceeds its bound;
* the edge behaviours the kernels copy from torch hold for torch's fp64 autograd."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import training_bounds as TB  # noqa: E402

F16, F32, F64 = torch.float16, torch.float32, torch.float64


def _ratio(what, got, ref, bound):
    r = TB.bound_ratio(got, ref, bound)
    print(f"{what}: max err / bound {r:.3g}")
    return r


# ------------------------------------------------------------------------------------------------ SSI emulation
def emulate_ssi_moments(p, y, m, mutant=None):
    """ssi_moments_kernel: per image, R CTAs of contiguous shares, fp64 sums of fp32 values.  p, y fp32 [B, HW]."""
    B, HW = p.shape
    R = TB.cluster_ctas(HW, 8 * TB.LOSS_THREADS)
    ws = []
    for b in range(B):
        acc = [0.0] * 5
        for r in range(R):
            lo, hi = TB.cluster_share(HW, R, r)
            if mutant == "drop_share" and r == R - 1 and R > 1:
                continue
            sel = m[b, lo:hi].clone()
            if mutant == "drop_pixel" and r == R - 1:
                nz = sel.nonzero()
                if len(nz):
                    sel[nz[-1, 0]] = False
            pv, yv = p[b, lo:hi][sel].double(), y[b, lo:hi][sel].double()
            for k, t in enumerate((pv * pv, pv, torch.ones_like(pv), pv * yv, yv)):
                acc[k] += t.sum().item()
        ws.append(acc)
    return ws


def _fit(a):
    a00, a01, a11, b0, b1 = a
    det = a00 * a11 - a01 * a01
    s = t = 0.0
    if det > 0:
        s = (a11 * b0 - a01 * b1) / det
        t = (-a01 * b0 + a00 * b1) / det
    return s, t, det


def _residual32(s, t, p, y):
    sf, tf = torch.tensor(s, dtype=F32), torch.tensor(t, dtype=F32)
    return (sf * p + tf) - y


def emulate_ssi_loss(p, y, m, mutant=None):
    ws = emulate_ssi_moments(p, y, m, mutant)
    tot, cnt = 0.0, 0.0
    for b, a in enumerate(ws):
        s, t, _ = _fit(a)
        r = _residual32(s, t, p[b], y[b])[m[b]]
        tot += r.abs().double().sum().item()
        cnt += float(m[b].sum())
    return torch.tensor(tot / cnt if cnt else float("nan"), dtype=F32)


def emulate_ssi_bwd(p, y, m, grad_out, mutant=None):
    """ssi_bwd_*: moments, sign sums of the fp32 residual, and the fp64 gradient formula stored as fp32."""
    B, HW = p.shape
    ws = emulate_ssi_moments(p, y, m, mutant)
    N = sum(a[2] for a in ws)
    out = torch.zeros(B, HW, dtype=F32)
    for b, a in enumerate(ws):
        s, t, det = _fit(a)
        r = _residual32(s, t, p[b], y[b])
        sg = torch.sign(r).double()
        if mutant == "sign0":
            sg = torch.where(r == 0, torch.ones_like(sg), sg)
        sg = sg * m[b].double()
        if N == 0:
            continue
        G0, G1 = sg.sum().item() / N, (sg * p[b].double()).sum().item() / N
        pv, yv = p[b].double(), y[b].double()
        g = sg * s / N
        if det > 0:
            a00, a01, a11, b0, b1 = a
            ddet = 2.0 * pv * a11 - 2.0 * a01
            dns = a11 * yv - b1
            dnt = -b0 - a01 * yv + 2.0 * pv * b1
            g = g + (G1 * (dns - s * ddet) + G0 * (dnt - t * ddet)) / det
        out[b] = torch.where(m[b], grad_out * g, torch.zeros_like(g)).float()
    return out


def ssi_inputs(B, HW, regime, seed=0):
    """pred, target fp32 [B, HW], mask bool [B, HW] for one regime (the GPU cases use the same generator)."""
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(B, HW, generator=g) * 2 + 0.5
    noise = torch.randn(B, HW, generator=g)
    m = torch.rand(B, HW, generator=g) < 0.8
    if regime == "exact":                                   # dyadic p, y = 2p + 1: r = 0 exactly
        p = torch.randint(0, 256, (B, HW), generator=g).float() / 64
        y = 2 * p + 1
    elif regime == "exact_mixed":                           # y = 2p + 1 +- 1/8 on pixel pairs of equal p: the fit is
        p = torch.randint(0, 256, (B, HW), generator=g).float() / 64    # still exactly (2, 1), and r = 0 off the pairs
        y = 2 * p + 1
        npair = HW // 4
        p[:, 1:2 * npair:2] = p[:, 0:2 * npair:2]
        y = 2 * p + 1
        y[:, 0:2 * npair:2] += 0.125
        y[:, 1:2 * npair:2] -= 0.125
        m = torch.ones(B, HW, dtype=torch.bool)
    elif regime == "small_s":                               # s ~ 1e-3 (DESIGN.md 8.6)
        y = 1e-3 * p + 1 + 1e-4 * noise
    elif regime == "const":                                 # constant dyadic prediction: det = 0
        p = torch.full((B, HW), 0.75)
        y = 0.5 + noise
    else:
        y = 0.7 * p - 0.3 + 0.2 * noise
    if regime == "one_pixel":
        m = torch.zeros(B, HW, dtype=torch.bool)
        m[:, HW // 2] = True
    elif regime == "last_pixel":
        m = torch.zeros(B, HW, dtype=torch.bool)
        m[:, HW - 1] = True
    elif regime == "last_share":
        R = TB.cluster_ctas(HW, 8 * TB.LOSS_THREADS)
        lo, _ = TB.cluster_share(HW, R, R - 1)
        m[:, :lo] = False
    elif regime == "one_empty":
        m[B // 2] = False
    elif regime == "all_empty":
        m[:] = False
    if regime in ("exact", "const"):
        m[:, 0] = True
    return p.float(), y.float(), m


SSI_SHAPES = [(1, 1), (2, 511), (5, 4095), (1, 4096), (2, 4097), (1, 8 * 4096 + 1), (2, 480 * 640)]
SSI_REGIMES = ["random", "small_s", "exact", "exact_mixed", "const", "one_pixel", "last_pixel", "last_share", "one_empty"]


@pytest.mark.parametrize("B,HW", SSI_SHAPES)
@pytest.mark.parametrize("regime", SSI_REGIMES)
def test_ssi_emulation_within_bound(B, HW, regime):
    if regime == "one_empty" and B == 1:
        pytest.skip("needs two images")
    p, y, m = ssi_inputs(B, HW, regime, seed=B * HW)
    ref, bound = TB.ssi_loss_ref_bound(p, y, m)
    assert _ratio("ssi fwd", emulate_ssi_loss(p, y, m), ref, bound) <= 1
    for go in (1.0, 1024.0, 2.0 ** 20):
        ref, bound = TB.ssi_bwd_ref_bound(p, y, m, go)
        assert _ratio(f"ssi bwd go={go}", emulate_ssi_bwd(p, y, m, go), ref, bound) <= 1


def test_ssi_exact_target_has_zero_gradient():
    """y = 2p + 1 with dyadic p: s = 2, t = 1 and r = 0 exactly; torch's abs backward gives 0 there, and so must the
    kernel's sign(0) = 0."""
    p, y, m = ssi_inputs(2, 4097, "exact")
    fits = TB._ssi_fit_bounds(p.double(), y.double(), m)
    assert all(f["s"] == 2 and f["t"] == 1 and f["e_sf"] == 0 and f["e_tf"] == 0 for f in fits)
    ref, bound = TB.ssi_bwd_ref_bound(p, y, m, 1024.0)
    assert (ref == 0).all() and (emulate_ssi_bwd(p, y, m, 1024.0) == 0).all()


def test_ssi_det_zero_cases_have_zero_fit():
    for regime in ("one_pixel", "const"):
        p, y, m = ssi_inputs(2, 4097, regime)
        fits = TB._ssi_fit_bounds(p.double(), y.double(), m)
        assert all(f["det"] == 0 and f["s"] == 0 and f["t"] == 0 and f["e_det"] == 0 for f in fits)


def test_ssi_all_empty_is_nan_and_zero_gradient():
    p, y, m = ssi_inputs(2, 511, "all_empty")
    ref, _ = TB.ssi_loss_ref_bound(p, y, m)
    assert math.isnan(ref.item()) and math.isnan(emulate_ssi_loss(p, y, m).item())
    ref, bound = TB.ssi_bwd_ref_bound(p, y, m, 1.0)
    assert (ref == 0).all() and (bound == 0).all() and (emulate_ssi_bwd(p, y, m, 1.0) == 0).all()


@pytest.mark.parametrize("B,HW", [(1, 4097), (2, 8 * 4096 + 1), (2, 480 * 640)])
@pytest.mark.parametrize("mutant", ["drop_share", "drop_pixel"])
def test_ssi_dropped_moment_exceeds_bound(B, HW, mutant):
    p, y, m = ssi_inputs(B, HW, "random", seed=3)
    ref, bound = TB.ssi_bwd_ref_bound(p, y, m, 1.0)
    assert _ratio(f"ssi bwd {mutant}", emulate_ssi_bwd(p, y, m, 1.0, mutant), ref, bound) > 1


def test_ssi_sign_of_zero_as_one_exceeds_bound():
    """With every residual 0, sign(0) = +1 still gives a zero gradient (sum r = 0 for any p at the fit), so the mutant
    is shown on a fit that is exact with both zero and nonzero residuals."""
    p, y, m = ssi_inputs(2, 4097, "exact_mixed")
    fits = TB._ssi_fit_bounds(p.double(), y.double(), m)
    assert all(f["s"] == 2 and f["t"] == 1 and f["e_sf"] == 0 for f in fits)
    ref, bound = TB.ssi_bwd_ref_bound(p, y, m, 1.0)
    assert _ratio("ssi bwd sign(0)=1", emulate_ssi_bwd(p, y, m, 1.0, "sign0"), ref, bound) > 1


# ------------------------------------------------------------------------------------------------ angular
def emulate_angular_d(p, y):
    return (p[:, 0] * y[:, 0] + p[:, 1] * y[:, 1]) + p[:, 2] * y[:, 2]


def emulate_angular_loss(p, y, m):
    d = emulate_angular_d(p, y).clamp(-1, 1)
    a = torch.acos(d).double()[m]
    return torch.tensor(a.sum().item() / m.sum().item(), dtype=F32)


def emulate_angular_bwd(p, y, m, grad_out):
    d = emulate_angular_d(p, y)
    k = torch.tensor(grad_out / m.sum().item(), dtype=F32)
    live = (d > -1) & (d < 1) & m
    w = torch.where(live, 1 - d * d, torch.ones_like(d))
    g = torch.where(live, -k * torch.rsqrt(w), torch.zeros_like(d))
    return g[:, None] * y


def angular_inputs(B, HW, regime, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.nn.functional.normalize(torch.randn(B, 3, HW, generator=g), dim=1)
    y = torch.nn.functional.normalize(p + 0.3 * torch.randn(B, 3, HW, generator=g), dim=1)
    m = torch.rand(B, HW, generator=g) < 0.8
    if regime == "near_one":                         # d = +-(1 - k 2^-24), k = 1..64, exact fp32 dots
        k = torch.arange(HW) % 64 + 1
        sgn = torch.where(torch.arange(HW) % 128 < 64, 1.0, -1.0)
        d = (sgn * (1 - k.double() * 2.0 ** -24)).float()
        p = torch.zeros(B, 3, HW)
        y = torch.zeros(B, 3, HW)
        ax = torch.arange(HW) % 3
        p[:, ax, torch.arange(HW)] = d
        y[:, ax, torch.arange(HW)] = 1.0
    elif regime == "identical":                      # identical axis-aligned unit vectors: d = 1 exactly
        p = torch.zeros(B, 3, HW)
        p[:, 1] = 1.0
        y = p.clone()
    return p.float(), y.float(), m


@pytest.mark.parametrize("B,HW", [(1, 1), (2, 511), (5, 4097), (2, 16 * 4096 + 1)])
@pytest.mark.parametrize("regime", ["random", "near_one", "identical"])
def test_angular_emulation_within_bound(B, HW, regime):
    p, y, m = angular_inputs(B, HW, regime, seed=HW)
    ref, bound = TB.angular_loss_ref_bound(p, y, m)
    assert _ratio("angular fwd", emulate_angular_loss(p, y, m), ref, bound) <= 1
    for go in (1.0, 2.0 ** 20):
        ref, bound = TB.angular_bwd_ref_bound(p, y, m, go)
        assert _ratio("angular bwd", emulate_angular_bwd(p, y, m, go), ref, bound) <= 1


def test_angular_at_d_one_torch_gives_nonfinite_and_bound_pins_zero():
    """torch's inclusive clamp passes the gradient at d = 1 and acos' is -inf there; the kernel returns 0, which the
    bound pins exactly (bound 0 at those pixels)."""
    p, y, m = angular_inputs(1, 64, "identical")
    pg = p.double().requires_grad_(True)
    torch.acos(torch.clamp((pg * y.double()).sum(1), -1, 1))[m].mean().backward()
    assert not torch.isfinite(pg.grad[:, 1][m]).any()
    ref, bound = TB.angular_bwd_ref_bound(p, y, m, 1.0)
    assert (ref == 0).all() and (bound <= 2 ** -140).all()


def test_angular_near_one_bound_carries_the_cancellation():
    """At d = 1 - 2^-24 the fp32 1 - d d alone is off by about U32 d^2 / (1 - d^2) = 1/2 relative: the bound has to
    admit that, and an emulation that computes 1 - d^2 in fp64 must still be inside it."""
    p, y, m = angular_inputs(1, 128, "near_one")
    ref, bound = TB.angular_bwd_ref_bound(p, y, m, 1.0)
    rel = (bound / ref.abs().clamp(min=1e-30))[:, 0, 0]
    assert rel.item() > 0.1


# ------------------------------------------------------------------------------------------------ decode_post
def emulate_decode_post(x, normals):
    a, b, c = x[:, 0], x[:, 1], x[:, 2]
    if not normals:
        return (((a + b) + c) / 3).clamp(-1, 1)[:, None]
    nrm = torch.sqrt((a * a + b * b) + c * c)
    inv = 1 / (nrm + torch.tensor(1e-5, dtype=F32))
    return (x * inv[:, None]).clamp(-1, 1)


def emulate_decode_post_bwd(x, dout, normals, mutant=None):
    a, b, c = x[:, 0], x[:, 1], x[:, 2]
    if not normals:
        m = ((a + b) + c) / 3
        keep = (m > -1) & (m < 1) if mutant == "exclusive" else (m >= -1) & (m <= 1)
        g = torch.where(keep, dout[:, 0] / 3, torch.zeros_like(m))
        return torch.stack([g, g, g], 1)
    nrm = torch.sqrt((a * a + b * b) + c * c)
    inv = 1 / (nrm + torch.tensor(1e-5, dtype=F32))
    u = x * inv[:, None]
    g = torch.where((u >= -1) & (u <= 1), dout, torch.zeros_like(dout))
    dot = (g[:, 0] * a + g[:, 1] * b) + g[:, 2] * c
    k = torch.where(nrm > 0, dot * inv * inv / torch.where(nrm > 0, nrm, torch.ones_like(nrm)), torch.zeros_like(nrm))
    return g * inv[:, None] - x * k[:, None]


def decode_post_inputs(NB, H, W, regime, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(NB, 3, H, W, generator=g) * 0.7
    n = H * W
    if regime == "edges":                           # channel means exactly +-1 and one ulp beyond, x = 0, huge |x|
        flat = x.reshape(NB, 3, -1)
        one_up = float(np.nextafter(np.float32(1), np.float32(2)))
        vals = [(1.0, 1.0, 1.0), (-1.0, -1.0, -1.0), (0.5, 1.25, 1.25), (one_up,) * 3, (-one_up,) * 3,
                (0.0, 0.0, 0.0), (1e4, 0.0, 0.0), (0.0, -3e5, 0.0), (2e4, 2e4, 2e4)]
        for i, v in enumerate(vals):
            flat[:, :, i % n] = torch.tensor(v)
    return x.contiguous()


@pytest.mark.parametrize("normals", [False, True])
@pytest.mark.parametrize("regime", ["random", "edges"])
def test_decode_post_emulation_within_bound(normals, regime):
    x = decode_post_inputs(2, 9, 13, regime, seed=int(normals))
    g = torch.Generator().manual_seed(5)
    dout = torch.randn(2, 3 if normals else 1, 9, 13, generator=g)
    ref, bound = TB.decode_post_ref_bound(x, normals)
    assert _ratio("decode_post", emulate_decode_post(x, normals), ref, bound) <= 1
    ref, bound = TB.decode_post_bwd_ref_bound(x, dout, normals)
    assert _ratio("decode_post_bwd", emulate_decode_post_bwd(x, dout, normals), ref, bound) <= 1


def test_decode_post_bwd_exclusive_clamp_exceeds_bound():
    x = decode_post_inputs(2, 9, 13, "edges")
    dout = torch.ones(2, 1, 9, 13)
    ref, bound = TB.decode_post_bwd_ref_bound(x, dout, False)
    assert _ratio("decode_post_bwd exclusive", emulate_decode_post_bwd(x, dout, False, "exclusive"), ref, bound) > 1


def test_decode_post_bwd_at_zero_is_dout_over_eps():
    """x = 0: torch's norm backward adds nothing, so the reference is dout * 1e5."""
    x = torch.zeros(1, 3, 1, 2)
    dout = torch.tensor([1.0, -2.0, 3.0]).view(1, 3, 1, 1).expand(1, 3, 1, 2).contiguous()
    ref, _ = TB.decode_post_bwd_ref_bound(x, dout, True)
    assert torch.allclose(ref, dout.double() * 1e5, rtol=1e-12)


# ------------------------------------------------------------------------------------------------ latent MSE
def emulate_masked_latent_mse(pred, tgt, val_mask):
    lm = TB.latent_mask_ref(val_mask)
    mm = torch.cat([lm, lm])[:, None].expand_as(pred)
    d = pred.float().double() - tgt.double()
    cnt = int(mm.sum())
    return torch.tensor((d * d)[mm].sum().item() / cnt if cnt else 0.0, dtype=F32), lm


def emulate_masked_latent_mse_bwd(pred, tgt, lm, go):
    mm = torch.cat([lm, lm])[:, None].expand_as(pred)
    cnt = int(mm.sum())
    s = torch.tensor(2.0 * go / cnt if cnt else 0.0, dtype=F32)
    g = torch.where(mm, s * (pred.float() - tgt), torch.zeros_like(tgt))
    return g.to(pred.dtype)


def latent_inputs(B, C, H, W, dtype, regime, seed=0):
    g = torch.Generator().manual_seed(seed)
    pred = torch.randn(2 * B, C, H // 8, W // 8, generator=g).to(dtype)
    tgt = torch.randn(2 * B, C, H // 8, W // 8, generator=g)
    vm = torch.rand(B, H, W, generator=g) < 0.999
    if regime == "block_edges":                      # holes on the 8x8 block edges
        vm = torch.ones(B, H, W, dtype=torch.bool)
        vm[:, 7::16, :] = False
        vm[:, :, 8::24] = False
    elif regime == "empty":
        vm[:] = False
    return pred, tgt, vm


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("B,C,H,W,regime", [(1, 4, 70, 93, "random"), (2, 4, 96, 128, "block_edges"),
                                            (2, 4, 64, 64, "empty")])
def test_masked_latent_mse_emulation_within_bound(dtype, B, C, H, W, regime):
    pred, tgt, vm = latent_inputs(B, C, H, W, dtype, regime)
    ref, bound, lm = TB.masked_latent_mse_ref_bound(pred, tgt, vm)
    got, lm_e = emulate_masked_latent_mse(pred, tgt, vm)
    assert torch.equal(lm, lm_e)
    assert _ratio("latent mse", got, ref, bound) <= 1
    if regime == "empty":
        assert ref.item() == 0 and got.item() == 0
    ref, bound = TB.masked_latent_mse_bwd_ref_bound(pred, tgt, lm, 1024.0)
    assert _ratio("latent mse bwd", emulate_masked_latent_mse_bwd(pred, tgt, lm, 1024.0), ref, bound) <= 1


# ------------------------------------------------------------------------------------------------ sumsq
def emulate_sumsq(x, mutant=None):
    n = x.numel()
    n4 = n // 4
    R = TB.cluster_ctas(n4, 1024 * 16, TB.MAX_SINGLE_SLOT)
    sq = x.double() ** 2
    tot = 0.0
    for r in range(R):
        if mutant == "drop_share" and r == R - 1 and R > 1:
            continue
        lo, hi = TB.cluster_share(n4, R, r)
        part = sq[4 * lo:4 * hi].sum().item()
        if r == R - 1 and mutant != "skip_tail":
            part += sq[4 * n4:].sum().item()
        if mutant == "drop_pixel" and r == 0 and hi > lo:
            part -= sq[4 * lo].item()
        tot += part
    return torch.tensor(tot, dtype=F64)


SUMSQ_NS = [1, 3, 5, 4 * 16384 - 1, 4 * 16384 + 1, 4 * 16384 * 3 + 1, 4 * 16384 * 16 + 3, 4 * 16384 * 17 + 2]


@pytest.mark.parametrize("n", SUMSQ_NS)
def test_sumsq_emulation_within_bound(n):
    x = torch.randn(n, generator=torch.Generator().manual_seed(n))
    ref, bound = TB.sumsq_ref_bound(x)
    assert _ratio(f"sumsq n={n}", emulate_sumsq(x), ref, bound) <= 1


@pytest.mark.parametrize("n,mutant", [(5, "skip_tail"), (4 * 16384 * 17 + 3, "skip_tail"),
                                      (4 * 16384 * 3 + 1, "drop_share"), (4 * 16384 * 17 + 2, "drop_pixel")])
def test_sumsq_mutants_exceed_bound(n, mutant):
    x = torch.randn(n, generator=torch.Generator().manual_seed(n))
    ref, bound = TB.sumsq_ref_bound(x)
    assert _ratio(f"sumsq {mutant}", emulate_sumsq(x, mutant), ref, bound) > 1


# ------------------------------------------------------------------------------------------------ AdamW
def emulate_bc(beta, step, mutant=None):
    if mutant == "powf":
        return float(np.float32(1) - np.power(np.float32(beta), np.float32(step)))
    return TB.f32(1.0 - TB.f32(beta) ** step)


def emulate_adamw(p, g, m, v, step, lr_e, wd_e, betas, eps, clip, mutant=None):
    """adamw_state_kernel's upd in fp32: lr_e / wd_e per element (fp32 tensors)."""
    b1, b2, eps = (torch.tensor(TB.f32(b), dtype=F32) for b in (betas[0], betas[1], eps))
    bc1 = emulate_bc(betas[0], step, mutant)
    bc2 = emulate_bc(betas[1], step - 1 if mutant == "prev_bc2" else step, mutant)
    rbc2 = torch.rsqrt(torch.tensor(bc2, dtype=F32))
    c = torch.tensor(clip, dtype=F32)
    decay = 1 - lr_e * wd_e
    step_size = lr_e / torch.tensor(bc1, dtype=F32)
    gi = g * c
    m1 = b1 * m + (1 - b1) * gi
    v1 = b2 * v + ((1 - b2) * gi) * gi
    p1 = p * decay - step_size * (m1 / (torch.sqrt(v1) * rbc2 + eps))
    if mutant == "skip_tail":
        n4 = p.numel() // 4 * 4
        p1[n4:], m1[n4:], v1[n4:] = p[n4:], m[n4:], v[n4:]
    return p1, m1, v1, (bc1, bc2)


def adamw_inputs(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    gr = torch.randn(n, generator=g) * 1e-2
    m = torch.randn(n, generator=g) * 1e-3
    v = torch.rand(n, generator=g) * 1e-4
    return p, gr, m, v


def group_table(n, n_groups, n_runs, seed=0):
    """Run starts (multiples of 4, some just below / above float4 and 256-thread block boundaries) and groups."""
    g = torch.Generator().manual_seed(seed)
    cand = sorted({s for s in (4, 252, 256, 260, 1020, 1024, 1028) if s < n}
                  | {int(s) * 4 for s in torch.randint(1, max(2, n // 4), (n_runs * 2,), generator=g)})
    starts = [0] + [s for s in cand if 0 < s < n][:n_runs - 1]
    groups = [i % n_groups for i in range(len(starts))]
    return starts, groups


def per_element(values, starts, groups, n):
    out = torch.empty(n, dtype=F32)
    for r, s in enumerate(starts):
        e = starts[r + 1] if r + 1 < len(starts) else n
        out[s:e] = values[groups[r]]
    return out


GROUP_LRS = [3e-5 * (1 + k) for k in range(16)]
GROUP_WDS = [1e-2 * (1 + (k % 3)) for k in range(16)]
BETAS, EPS = (0.9, 0.999), 1e-8


@pytest.mark.parametrize("step", [1, 2, 3, 10, 1000, 30000])
@pytest.mark.parametrize("clipped", [False, True])
def test_adamw_emulation_within_bound(step, clipped):
    n = 4099
    p, g, m, v = adamw_inputs(n, step)
    starts, groups = group_table(n, 16, 40)
    lr_e, wd_e = (per_element([TB.f32(x) for x in vals], starts, groups, n) for vals in (GROUP_LRS, GROUP_WDS))
    nsq = float((g.double() ** 2).sum())
    clip = TB.clip_ref(nsq, 0.05 if clipped else 0.0)
    assert (clip < 1) == clipped
    p1, m1, v1, (bc1, bc2) = emulate_adamw(p, g, m, v, step, lr_e, wd_e, BETAS, EPS, TB.f32(clip))
    rb = TB.adamw_ref_bound(p, g, m, v, step, lr_e.double(), wd_e.double(), BETAS, EPS, clip)
    for name, got in (("param", p1), ("exp_avg", m1), ("exp_avg_sq", v1)):
        assert _ratio(f"adamw {name} step {step}", got, *rb[name]) <= 1
    for k, bc in ((0, bc1), (1, bc2)):
        ref, b = TB.bias_correction_ref_bound(BETAS[k], step)
        assert abs(bc - ref) <= b


@pytest.mark.parametrize("mutant,step", [("neighbour_lr", 10), ("prev_bc2", 2), ("prev_bc2", 10),
                                         ("prev_bc2", 1000), ("skip_tail", 3), ("powf", 2)])
def test_adamw_mutants_exceed_bound(mutant, step):
    n = 4099
    p, g, m, v = adamw_inputs(n, 7)
    starts, groups = group_table(n, 16, 40)
    lrs = [TB.f32(x) for x in GROUP_LRS]
    lr_e = per_element(lrs, starts, groups, n)
    wd_e = per_element([TB.f32(x) for x in GROUP_WDS], starts, groups, n)
    lr_k = lr_e.clone()
    if mutant == "neighbour_lr":                     # the first element of run 5 takes run 4's group
        lr_k[starts[5]] = lrs[groups[4]]
    nsq = float((g.double() ** 2).sum())
    clip = TB.clip_ref(nsq, 0.0)
    p1, m1, v1, (bc1, bc2) = emulate_adamw(p, g, m, v, step, lr_k, wd_e, BETAS, EPS, TB.f32(clip), mutant)
    rb = TB.adamw_ref_bound(p, g, m, v, step, lr_e.double(), wd_e.double(), BETAS, EPS, clip)
    r = _ratio(f"adamw {mutant} param", p1, *rb["param"])
    if mutant == "skip_tail":
        r = max(r, _ratio("adamw skip_tail exp_avg", m1, *rb["exp_avg"]))
    if mutant == "powf":
        ref, b = TB.bias_correction_ref_bound(BETAS[1], step)
        r = max(r, abs(bc2 - ref) / b)
        print(f"fp32 bc2 at step {step}: {abs(bc2 - ref) / ref:.3g} relative, {abs(bc2 - ref) / b:.3g} x bound")
    assert r > 1


# ------------------------------------------------------------------------------------------------ sums
@pytest.mark.parametrize("rows,C,dtype", [(7, 40, F32), (511, 72, F16), (4097, 4, F32), (20000, 1280, F16)])
def test_col_sum_emulation_within_bound(rows, C, dtype):
    g = torch.Generator().manual_seed(rows)
    x = torch.randn(rows, C + 3, generator=g).to(dtype)[:, :C]
    out0 = torch.randn(C, generator=g)
    R = TB.cluster_ctas(rows, 512)
    Y = 32 if R > 1 else 8
    xf = x.float()
    tot = torch.zeros(C)
    for r in range(R):
        lo, hi = TB.cluster_share(rows, R, r)
        part = torch.zeros(C)
        for j in range(Y):
            acc = torch.zeros(C)
            for i in range(lo + j, hi, Y):
                acc = acc + xf[i]
            part = part + acc
        tot = tot + part
    ref, bound = TB.col_sum_ref_bound(x, out0)
    assert _ratio("col_sum", out0 + tot, ref, bound) <= 1


@pytest.mark.parametrize("hw,ohw", [((6, 6), (12, 12)), ((12, 12), (23, 23)), ((23, 23), (45, 45)),
                                    ((7, 7), (15, 15)), ((1, 1), (3, 3))])
def test_upsample_nearest_bwd_reference_is_the_integer_map(hw, ohw):
    """torch's nearest map at these sizes is floor(o * in / out), the map the kernels use."""
    (H, W), (OH, OW) = hw, ohw
    dy = torch.randn(1, OH, OW, 4, generator=torch.Generator().manual_seed(H))
    ref, bound = TB.upsample_nearest_bwd_ref_bound(dy, (H, W))
    got = torch.zeros(1, H, W, 4)
    for oh in range(OH):
        for ow in range(OW):
            got[0, oh * H // OH, ow * W // OW] += dy[0, oh, ow]
    assert _ratio("upsample_nearest_bwd", got, ref, bound) <= 1


# ------------------------------------------------------------------------------------------------ activations
def all_finite_f16():
    bits = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16)
    x = bits.view(F16)
    return x[torch.isfinite(x)]


def emulate_silu_grad(z):
    s = 1 / (1 + torch.exp(-z))
    return s * (1 + z * (1 - s))


def emulate_gelu_grad(x):
    cdf = 0.5 * (1 + torch.erf(x * TB.INV_SQRT2_F32))
    pdf = TB.INV_SQRT2PI_F32 * torch.exp(-0.5 * x * x)
    return cdf + x * pdf


@pytest.mark.parametrize("silu", [True, False])
def test_act_bwd_emulation_within_bound_every_f16(silu):
    x = all_finite_f16()
    dy = torch.randn(x.shape, generator=torch.Generator().manual_seed(1)).half()
    xf = x.float()
    got = (dy.float() * (emulate_silu_grad(xf) if silu else emulate_gelu_grad(xf))).half()
    assert _ratio(f"act_bwd {'silu' if silu else 'gelu'}", got, *TB.act_bwd_ref_bound(x, dy, silu)) <= 1


def test_geglu_bwd_emulation_within_bound_every_f16():
    g = all_finite_f16()
    gen = torch.Generator().manual_seed(2)
    h = (torch.randn(g.shape, generator=gen) * 4).half()
    dy = ((torch.rand(g.shape, generator=gen) * 2 - 1) * 0.99).half()      # |dy gelu(g)| stays below fp16's max
    gf = g.float()
    gelu = 0.5 * gf * (1 + torch.erf(gf * TB.INV_SQRT2_F32))
    rb = TB.geglu_bwd_ref_bound(h, g, dy)
    assert _ratio("geglu dh", (dy.float() * gelu).half(), *rb["dh"]) <= 1
    assert _ratio("geglu dg", (dy.float() * h.float() * emulate_gelu_grad(gf)).half(), *rb["dg"]) <= 1


def test_act_bwd_wrong_activation_exceeds_bound():
    x = all_finite_f16()
    dy = torch.ones_like(x)
    got = (dy.float() * emulate_gelu_grad(x.float())).half()
    assert _ratio("act_bwd gelu as silu", got, *TB.act_bwd_ref_bound(x, dy, True)) > 1
