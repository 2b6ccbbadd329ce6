"""Bitwise-reproducible training (DESIGN.md §8 item 7, §9 "Reduction order"): every reduction on the training path
(GroupNorm / LayerNorm backward sums, bias gradients, the losses, the gradient norm, the GroupNorm statistics of
recomputed inputs) gives the same bits on every run, so a micro-step repeats exactly, checkpointing leaves the
gradients unchanged and a resumed run continues an uninterrupted one bit for bit."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from diffusion_e2e_ft_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _three(fn):
    """fn() three times; every output must be bitwise equal to the first run's.  Returns the first run's."""
    runs = []
    for _ in range(3):
        out = fn()
        runs.append([t.detach().clone() for t in (out if isinstance(out, (tuple, list)) else (out,))])
    torch.cuda.synchronize()
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    return runs[0]


def _rel(got, want):
    """max |got - want| over the largest |want| (fp64 reference)."""
    got, want = got.double().cpu(), want.double().cpu()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---------------------------------------------------------------------------------------------- per kernel
@pytest.mark.parametrize("NB,H,W,C,x_f32,G", [(2, 96, 96, 320, False, 32), (2, 768, 768, 128, True, 32),
                                              (1, 24, 40, 40, False, 8)])
def test_group_norm_bwd_sums_repeat(NB, H, W, C, x_f32, G):
    g = _gen(1)
    x = torch.randn(NB, H, W, C, device=DEV, generator=g) * 2 + 0.5
    x = x if x_f32 else x.half()
    dy = (torch.randn(NB, H, W, C, device=DEV, generator=g)).half()
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.1
    mr = ops.group_norm_mean_rstd(x, 1e-6, G)
    L = ops._lib.load()

    def run():
        S = torch.zeros(NB, C, 2, device=DEV)
        ops._ck(L.b200_group_norm_bwd_sums(ops._p(x), int(x_f32), C, 0, C, ops._p(dy), NB, H * W, G, ops._p(mr),
                                           ops._p(gamma), ops._p(beta), 1, ops._p(S), ops._stream()), "bwd_sums")
        return S
    S = _three(run)[0]
    xd, dyd = x.double().view(NB, H * W, G, C // G), dy.double().view(NB, H * W, G, C // G)
    mean, rstd = mr[..., 0].double()[:, None, :, None], mr[..., 1].double()[:, None, :, None]
    xh = (xd - mean) * rstd
    z = xh * gamma.double().view(G, C // G) + beta.double().view(G, C // G)
    dz = dyd * torch.sigmoid(z) * (1 + z * (1 - torch.sigmoid(z)))
    want = torch.stack([dz.sum(1).reshape(NB, C), (dz * xh).sum(1).reshape(NB, C)], -1)
    assert _rel(S, want) <= 1e-4


@pytest.mark.parametrize("NB,H,W,C,x_f32", [(2, 96, 96, 320, False), (1, 768, 768, 128, True), (2, 12, 12, 960, False)])
def test_group_norm_stats_repeat(NB, H, W, C, x_f32):
    g = _gen(2)
    x = torch.randn(NB, H, W, C, device=DEV, generator=g) * 3 + 1.0
    x = x if x_f32 else x.half()
    L = ops._lib.load()

    def run():
        sums = torch.zeros(NB, 32, 2, dtype=torch.float64, device=DEV)
        ops._ck(L.b200_group_norm_stats(ops._p(x), C, None, 0, int(x_f32), NB, H * W, 32, ops._p(sums),
                                        ops._stream()), "stats")
        return sums
    sums = _three(run)[0]
    xd = x.double().view(NB, H * W, 32, C // 32)
    want = torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1)
    assert _rel(sums, want) <= 1e-6                 # per-thread sums are fp32 (shifted), merged in fp64


@pytest.mark.parametrize("rows,C,f32", [(2 * 9216, 320, False), (2 * 9216, 1280, True), (16, 1280 * 9 * 8, True)])
def test_col_sum_repeat(rows, C, f32):
    x = torch.randn(rows, C, device=DEV, generator=_gen(3))
    x = x if f32 else x.half()
    out = _three(lambda: ops.col_sum(x))[0]
    assert _rel(out, x.double().sum(0)) <= 1e-5


@pytest.mark.parametrize("rows,C", [(2 * 9216, 320), (2 * 9216, 1280)])
def test_layer_norm_bwd_repeat(rows, C):
    g = _gen(4)
    x = torch.randn(rows, C, device=DEV, generator=g) * 2 + 0.3
    dy = torch.randn(rows, C, device=DEV, generator=g).half()
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    dx, dgamma, dbeta = _three(lambda: ops.layer_norm_bwd(x, dy, gamma, 1e-5))
    xd = x.double()
    xh = (xd - xd.mean(1, keepdim=True)) * torch.rsqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    assert _rel(dgamma, (dy.double() * xh).sum(0)) <= 1e-4
    assert _rel(dbeta, dy.double().sum(0)) <= 1e-4


def _loss_inputs(B=2, H=768, W=768, ch=1):
    g = _gen(5)
    pred = torch.randn(B, ch, H, W, device=DEV, generator=g)
    if ch == 3:
        pred = torch.nn.functional.normalize(pred, dim=1)
        tgt = torch.nn.functional.normalize(pred + 0.3 * torch.randn(pred.shape, device=DEV, generator=g), dim=1)
    else:
        tgt = 2.0 * pred + 1.0 + 0.5 * torch.randn(pred.shape, device=DEV, generator=g)
    mask = torch.rand(B, 1, H, W, device=DEV, generator=g) > 0.2
    return pred, tgt, mask


def test_ssi_loss_repeat():
    pred, tgt, mask = _loss_inputs()
    go = torch.tensor(1.5, device=DEV)
    loss, grad = _three(lambda: (ops.ssi_loss(pred, tgt, mask), ops.ssi_loss_bwd(pred, tgt, mask, go)))
    p, t, m = pred.double(), tgt.double(), mask.double()
    a00, a01, a11 = (m * p * p).sum((1, 2, 3)), (m * p).sum((1, 2, 3)), m.sum((1, 2, 3))
    b0, b1 = (m * p * t).sum((1, 2, 3)), (m * t).sum((1, 2, 3))
    det = a00 * a11 - a01 * a01
    s, sh = (a11 * b0 - a01 * b1) / det, (-a01 * b0 + a00 * b1) / det
    want = ((s.view(-1, 1, 1, 1) * p + sh.view(-1, 1, 1, 1) - t).abs() * m).sum() / m.sum()
    assert _rel(loss, want) <= 1e-5
    assert torch.isfinite(grad).all() and grad.abs().max() > 0


def test_angular_loss_repeat():
    pred, tgt, mask = _loss_inputs(ch=3)
    go = torch.tensor(0.7, device=DEV)
    loss, grad = _three(lambda: (ops.angular_loss(pred, tgt, mask), ops.angular_loss_bwd(pred, tgt, mask, go)))
    d = (pred.double() * tgt.double()).sum(1, keepdim=True).clamp(-1, 1)
    want = torch.acos(d)[mask].mean()
    assert _rel(loss, want) <= 1e-5
    assert torch.isfinite(grad).all() and grad.abs().max() > 0


def test_masked_latent_mse_repeat():
    g = _gen(6)
    B, C, H, W = 2, 4, 768, 768
    pred = torch.randn(2 * B, C, H // 8, W // 8, device=DEV, generator=g)
    tgt = torch.randn(pred.shape, device=DEV, generator=g)
    vm = torch.rand(B, 1, H, W, device=DEV, generator=g) > 0.001
    go = torch.tensor(1.0, device=DEV)

    def run():
        loss, lm, ws = ops.masked_latent_mse(pred, tgt, vm)
        return loss, lm, ws, ops.masked_latent_mse_bwd(pred, tgt, lm, ws, go)
    loss, lm, ws, _ = _three(run)
    keep = lm.bool().repeat(2, 1, 1)[:, None].expand_as(pred)
    assert 0 < keep.sum() < keep.numel()
    assert _rel(loss, (pred.double() - tgt.double())[keep].pow(2).mean()) <= 1e-6


def test_sumsq_repeat():
    x = torch.randn((1 << 27) + 3, device=DEV, generator=_gen(7))      # n % 4 = 3: the scalar tail too
    nsq = _three(lambda: ops.grad_norm_sq(x))[0]
    assert _rel(nsq, x.double().pow(2).sum()) <= 1e-12


# ---------------------------------------------------------------------------------------------- micro-steps
def _e2e_grads(kind, unet_ckpt=False, vae_ckpt=False):
    """One tiny E2E micro-step (Marigold depth, or GeoWizard depth + normals), every UNet gradient back."""
    import engine_checks as EC
    import make_golden as MG
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss, e2e_ft_loss_geowizard
    unet_ref, vae_ref = MG.build_tiny(kind)
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
    unet.requires_grad_(True)
    if unet_ckpt:
        unet.enable_gradient_checkpointing()
    if vae_ckpt:
        vae.enable_gradient_checkpointing()
    g = torch.Generator().manual_seed(23)
    rgb = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(DEV)
    mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.2).to(DEV)
    depth = (torch.rand(2, 1, 64, 64, generator=g) * 9.9 + 0.1).to(DEV)
    if kind == "geowizard":
        normals = torch.nn.functional.normalize(torch.randn(2, 3, 64, 64, generator=g), dim=1).to(DEV)
        emb = (torch.randn(2, 1, 96, generator=g) * 0.5).to(DEV)
        loss = e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb, depth, normals, mask, emb)[0]
    else:
        ctx = (torch.randn(1, 77, 128, generator=g) * 0.5).to(DEV)
        loss = e2e_ft_loss(unet, vae, DDIMScheduler(), rgb, depth, mask, ctx, "depth")[0]
    (loss * LOSS_SCALE).backward()
    torch.cuda.synchronize()
    return {n: p.grad.clone() for n, p in unet.named_parameters() if p.grad is not None}


def _assert_equal_grads(a, b, what):
    assert a.keys() == b.keys() and len(a) > 0
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, (what, diff[:5], len(diff))


@pytest.mark.parametrize("kind", ["marigold", "geowizard"])
def test_micro_step_repeats(kind):
    _assert_equal_grads(_e2e_grads(kind), _e2e_grads(kind), f"{kind} micro-step rerun")


@pytest.mark.parametrize("kind", ["marigold", "geowizard"])
def test_checkpointing_leaves_unet_gradients_unchanged(kind):
    plain = _e2e_grads(kind)
    _assert_equal_grads(plain, _e2e_grads(kind, unet_ckpt=True), f"{kind} UNet checkpointing")
    _assert_equal_grads(plain, _e2e_grads(kind, vae_ckpt=True), f"{kind} decoder checkpointing")
    _assert_equal_grads(plain, _e2e_grads(kind, unet_ckpt=True, vae_ckpt=True), f"{kind} both")


@pytest.mark.parametrize("config", ["tiny", "768"])
def test_decoder_dx_checkpointing_is_bitwise(config):
    import test_vae_checkpointing_gpu as TV
    if config == "768":
        vae, shape = TV._full_vae(), (2, 4, 96, 96)
    else:
        vae, shape = TV._tiny_vae(), (2, 4, 12, 10)
    up = 2 ** (len(vae.decoder.up_blocks) - 1)
    g = torch.Generator(device="cpu").manual_seed(9)
    z = (torch.randn(*shape, generator=g) * 0.5).to(DEV)
    dy = torch.randn(shape[0], 3, shape[2] * up, shape[3] * up, generator=g).to(DEV)
    plain, plain2, ck = (TV._decoder_dx(vae, z, dy, c)["dx"] for c in (False, False, True))
    assert torch.isfinite(ck).all() and ck.abs().max() > 0
    assert torch.equal(plain, plain2) and torch.equal(plain, ck)


# ---------------------------------------------------------------------------------------------- resume
def test_full_loop_resume_is_exact(tmp_path):
    """The tiny GeoWizard loop (clipping, grouped AdamW, EMA, IterExponential): 4 steps straight equal 2 steps,
    save_state, a fresh trainer's load_state and 2 more, bit for bit."""
    import test_training_state_gpu as TS
    from diffusion_e2e_ft_b200 import DDIMScheduler, training
    import engine_checks as EC
    import make_golden as MG

    def loop(tr, unet, vae, g, steps):
        for _ in range(steps):
            rgb, emb, mask, gt_d, gt_n = TS._geowizard_batch(g)
            loss, _, _ = training.e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb.to(DEV), gt_d.to(DEV),
                                                        gt_n.to(DEV), mask.to(DEV), emb.to(DEV), "indoor")
            tr.micro_step(loss)

    def build():
        unet_ref, vae_ref = MG.build_tiny("geowizard")
        unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
        unet.requires_grad_(True)
        tr = training.FlatTrainer(unet, lr=1e-4, max_grad_norm=1.0, use_ema=True,
                                  param_groups=training.geowizard_param_groups(10),
                                  lr_schedule=training.IterExponential(20, 0.01, 2))
        return tr, unet, vae

    tr, unet, vae = build()
    loop(tr, unet, vae, torch.Generator().manual_seed(41), 4)
    want = TS._bufs(tr)
    tr, unet, vae = build()
    g = torch.Generator().manual_seed(41)
    loop(tr, unet, vae, g, 2)
    tr.save_state(str(tmp_path))
    tr2, unet2, vae2 = build()
    tr2.load_state(str(tmp_path))
    loop(tr2, unet2, vae2, g, 2)
    torch.cuda.synchronize()
    assert tr2.step_count == 4
    for name, a, b in zip(("param", "exp_avg", "exp_avg_sq", "state", "ema"), want, TS._bufs(tr2)):
        assert torch.equal(a, b), name


def test_clipped_optimizer_resume_is_exact(tmp_path):
    import test_training_state_gpu as TS
    from diffusion_e2e_ft_b200 import training
    tr = TS._opt_trainer(1.0)
    for k in range(4):
        TS._write_grads(tr, k)
    want = TS._bufs(tr)
    tr = TS._opt_trainer(1.0)
    for k in range(2):
        TS._write_grads(tr, k)
    tr.save_state(str(tmp_path / "checkpoint-2"))
    tr2 = TS._opt_trainer(1.0)
    assert tr2.load_state(training.latest_checkpoint(str(tmp_path))) == 2
    for k in range(2, 4):
        TS._write_grads(tr2, k)
    torch.cuda.synchronize()
    for name, a, b in zip(("param", "exp_avg", "exp_avg_sq", "state", "ema"), want, TS._bufs(tr2)):
        assert torch.equal(a, b), name


# ---------------------------------------------------------------------------------------------- torch's switch
def test_step_under_use_deterministic_algorithms():
    """A FlatTrainer micro-step and step complete with torch.use_deterministic_algorithms(True) (no op on the path
    raises), and give the same parameters as without it."""
    import test_training_state_gpu as TS
    from diffusion_e2e_ft_b200 import DDIMScheduler, training
    import engine_checks as EC
    import make_golden as MG

    def one_step():
        unet_ref, vae_ref = MG.build_tiny("geowizard")
        unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
        unet.requires_grad_(True)
        tr = training.FlatTrainer(unet, lr=1e-4, max_grad_norm=1.0, use_ema=True,
                                  param_groups=training.geowizard_param_groups(10))
        rgb, emb, mask, gt_d, gt_n = TS._geowizard_batch(torch.Generator().manual_seed(41))
        loss, _, _ = training.e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb.to(DEV), gt_d.to(DEV),
                                                    gt_n.to(DEV), mask.to(DEV), emb.to(DEV), "indoor")
        tr.micro_step(loss)
        torch.cuda.synchronize()
        assert tr.applied_steps() == 1
        return TS._bufs(tr)

    plain = one_step()
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        det = one_step()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    for a, b in zip(plain, det):
        assert torch.equal(a, b)
