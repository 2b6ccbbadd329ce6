"""Diffusion-objective training, noisy-start E2E fine-tuning and the EMA of the UNet weights on the CPU: the restated
reference math against max_pool2d / fp64, argument errors raised before any launch, and the host wiring on emulated
kernels (tests/cpu_emulation.py plus the contracts of the ABI-10 kernels below) against the oracle's autograd."""
import json
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cpu_emulation
import diffusion_training_checks as DC
import diffusion_training_oracle as DO
from diffusion_e2e_ft_b200 import DDIMScheduler, lib, ops, training


# ---- plain-torch contracts of the ABI-10 kernels (include/b200_e2eft.h)
def diffusion_inputs(rgb_latents, x0, noise, timesteps, alphas_cumprod, prediction_type, timesteps_host=None):
    B = rgb_latents.shape[0]
    n = torch.zeros_like(x0) if noise is None else noise
    unet_in = torch.cat((rgb_latents.repeat(2, 1, 1, 1), DO.add_noise(alphas_cumprod, x0, n, timesteps)), 1)
    target = n.clone() if prediction_type == "epsilon" else DO.get_velocity(alphas_cumprod, x0, n, timesteps)
    assert unet_in.shape[0] == 2 * B
    return unet_in, target


def masked_latent_mse(pred, target, val_mask):
    B, C, H, W, h, w = ops.latent_mask_shape(val_mask, pred)
    lm = (~torch.max_pool2d((~val_mask.bool()).float(), 8, 8).bool())[:, 0].to(torch.uint8)
    full = lm.bool()[:, None].repeat(2, C, 1, 1)
    d = (pred.double() - target.double())[full]
    cnt = float(full.sum())
    ws = torch.tensor([d.pow(2).sum().item(), cnt], dtype=torch.float64)
    loss = torch.tensor((ws[0] / ws[1]).item() if cnt > 0 else 0.0, dtype=torch.float32)
    return loss, lm, ws


def masked_latent_mse_bwd(pred, target, latent_mask, workspace, grad_out):
    C = pred.shape[1]
    full = latent_mask.bool()[:, None].repeat(2, C, 1, 1)
    cnt = float(workspace[1])
    s = 2.0 * float(grad_out) / cnt if cnt > 0 else 0.0
    return torch.where(full, (pred.float() - target) * s, torch.zeros_like(target)).to(pred.dtype)


def ema_update(ema, param, one_minus_decay):
    ema.sub_(float(one_minus_decay) * (ema - param))


@pytest.fixture
def emulated(monkeypatch):
    cpu_emulation.install(monkeypatch)
    for name, fn in dict(diffusion_inputs=diffusion_inputs, masked_latent_mse=masked_latent_mse,
                         masked_latent_mse_bwd=masked_latent_mse_bwd, ema_update=ema_update).items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)


@pytest.fixture
def no_launch(monkeypatch):
    """CPU tensors pass the device check, and any attempt to reach the library fails the test."""
    monkeypatch.setattr(ops, "_need_cuda", lambda *a: None)

    def load(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(lib, "load", load)


# ---- the restated reference math
@pytest.mark.parametrize("hw", [(64, 64), (120, 160), (127, 161)])
def test_latent_mask_rule_matches_max_pool(hw):
    """A latent pixel is valid iff its whole 8x8 block is; floor cropping (15x20 latent for 120x160, also for 127x161)."""
    g = torch.Generator().manual_seed(1)
    H, W = hw
    m = torch.rand(2, 1, H, W, generator=g) > 0.003
    lm = DO.latent_mask(m)
    h, w = H // 8, W // 8
    assert lm.shape == (4, 4, h, w)
    blocks = m[:, 0, :8 * h, :8 * w].reshape(2, h, 8, w, 8).all(4).all(2)
    assert torch.equal(lm[:2, 0], blocks) and torch.equal(lm[2:, 3], blocks)
    assert 0 < int(blocks.sum()) < blocks.numel()
    assert torch.equal(masked_latent_mse(torch.zeros(4, 4, h, w), torch.zeros(4, 4, h, w), m)[1].bool(), blocks)


def test_add_noise_and_velocity_match_fp64():
    ac = DDIMScheduler().alphas_cumprod
    g = torch.Generator().manual_seed(2)
    x0, eps = torch.randn(4, 4, 15, 20, generator=g), torch.randn(4, 4, 15, 20, generator=g)
    t = torch.tensor([0, 999, 421, 7])
    a = ac.double()[t][:, None, None, None]
    xt = a.sqrt() * x0.double() + (1 - a).sqrt() * eps.double()
    v = a.sqrt() * eps.double() - (1 - a).sqrt() * x0.double()
    assert (DO.add_noise(ac, x0, eps, t).double() - xt).abs().max() <= 2e-6
    assert (DO.get_velocity(ac, x0, eps, t).double() - v).abs().max() <= 2e-6
    # the kernel contract is the same expression: bit for bit on the CPU
    ui, tgt = diffusion_inputs(x0[:2], x0, eps, t, ac, "v_prediction")
    assert torch.equal(ui[:, 4:], DO.add_noise(ac, x0, eps, t)) and torch.equal(ui[:, :4], x0[:2].repeat(2, 1, 1, 1))
    assert torch.equal(tgt, DO.get_velocity(ac, x0, eps, t))


def test_masked_mse_contract_matches_reference_and_fp64():
    g = torch.Generator().manual_seed(3)
    m = torch.rand(2, 1, 120, 160, generator=g) > 0.003
    pred = torch.randn(4, 4, 15, 20, generator=g, requires_grad=True)
    tgt = torch.randn(4, 4, 15, 20, generator=g)
    lm = DO.latent_mask(m)
    ref = DO.masked_mse(pred, tgt, lm)
    ref.backward()
    loss, lm8, ws = masked_latent_mse(pred.detach(), tgt, m)
    d = (pred.detach().double() - tgt.double())[lm]
    assert abs(loss.item() - (d.pow(2).sum() / d.numel()).item()) <= 1e-6 * loss.item()
    assert abs(loss.item() - ref.item()) <= 1e-6 * ref.item()
    gr = masked_latent_mse_bwd(pred.detach(), tgt, lm8, ws, torch.tensor(1.0))
    assert torch.allclose(gr, pred.grad, rtol=1e-5, atol=1e-9)
    empty = torch.zeros_like(m)
    l0, lm0, ws0 = masked_latent_mse(pred.detach(), tgt, empty)
    assert l0.item() == 0.0 and not torch.isnan(l0)
    assert masked_latent_mse_bwd(pred.detach(), tgt, lm0, ws0, torch.tensor(1.0)).abs().max() == 0


def test_shape_mismatch_is_a_value_error():
    with pytest.raises(ValueError, match="does not match"):
        ops.latent_mask_shape(torch.ones(2, 1, 120, 160, dtype=torch.bool), torch.empty(4, 4, 16, 20))
    with pytest.raises(ValueError, match="does not match"):
        ops.latent_mask_shape(torch.ones(2, 1, 64, 64, dtype=torch.bool), torch.empty(2, 4, 8, 8))
    with pytest.raises(ValueError, match="does not match"):       # a mask 8 rows taller than the image
        ops.latent_mask_shape(torch.ones(2, 1, 135, 161, dtype=torch.bool), torch.empty(4, 4, 15, 20))
    with pytest.raises(IndexError):                                 # the reference's boolean indexing fails too
        DO.masked_mse(torch.zeros(4, 4, 15, 20), torch.zeros(4, 4, 15, 20),
                      DO.latent_mask(torch.ones(2, 1, 135, 161, dtype=torch.bool)))


@pytest.mark.parametrize("hw", [(64, 64), (60, 68), (127, 161), (120, 160), (9, 17)])
def test_latent_size_matches_the_vae_encoder_and_the_pooled_mask(hw):
    """The size check before launch predicts the VAE encoder's latent (floor(H/2) per level, as its (0,1,0,1)-padded
    stride-2 convs give), which is the size of max_pool2d(mask, 8, 8) for every image size."""
    import make_golden as MG
    from oracle import pipeline as OP
    _, vae_ref = MG.build_tiny()
    H, W = hw
    with torch.no_grad():
        lat = OP.encode_rgb(vae_ref, torch.zeros(1, 3, H, W))
    assert training._latent_hw(vae_ref, H, W) == tuple(lat.shape[2:]) == (H // 8, W // 8)


# ---- argument errors before any launch
def test_binding_argument_errors_before_launch(no_launch):
    ac = DDIMScheduler().alphas_cumprod
    x0, rgb = torch.zeros(4, 4, 8, 8), torch.zeros(2, 4, 8, 8)
    t = torch.tensor([1, 2, 1, 2])
    with pytest.raises(ValueError, match="prediction type"):
        ops.diffusion_inputs(rgb, x0, None, t, ac, "sample")
    with pytest.raises(ValueError, match="outside"):
        ops.diffusion_inputs(rgb, x0, None, torch.tensor([1, 1000, 1, 1000]), ac, "epsilon")
    with pytest.raises(ValueError, match="outside"):
        ops.diffusion_inputs(rgb, x0, None, torch.tensor([-1, 3, -1, 3]), ac, "epsilon")
    with pytest.raises(ValueError, match="2B"):
        ops.diffusion_inputs(rgb, x0, None, torch.tensor([1, 2]), ac, "epsilon")
    with pytest.raises(ValueError, match="does not match"):
        ops.masked_latent_mse(torch.zeros(4, 4, 8, 8), torch.zeros(4, 4, 8, 8), torch.ones(2, 1, 72, 64, dtype=torch.bool))


def test_training_entry_argument_errors_before_launch(no_launch):
    import make_golden as MG
    import engine_checks as EC
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(gunet_ref, vae_ref, "cpu")
    rgb, depth, normals, mask, emb = DC.diffusion_batch(2, (64, 64))
    args = (unet, vae, DDIMScheduler(), rgb, depth, normals, mask, emb)
    with pytest.raises(ValueError, match="noise type"):
        training.diffusion_loss_geowizard(*args, noise_type="uniform", timesteps=[1, 2])
    with pytest.raises(ValueError, match="prediction type"):
        training.diffusion_loss_geowizard(*args[:2], DDIMScheduler(prediction_type="sample"), *args[3:], timesteps=[1, 2])
    with pytest.raises(ValueError, match=r"\[0, 1000\)"):
        training.diffusion_loss_geowizard(*args, timesteps=[1, 1000])
    with pytest.raises(ValueError, match="does not match"):
        training.diffusion_loss_geowizard(*args[:6], torch.ones(2, 1, 56, 64, dtype=torch.bool), emb, timesteps=[1, 2])
    with pytest.raises(ValueError, match="noise type"):
        training.e2e_ft_loss(unet, vae, DDIMScheduler(), rgb, depth[:, :1], mask, emb, "depth", noise_type="uniform")
    with pytest.raises(ValueError, match="noise type"):
        training.e2e_ft_loss_geowizard(*args[:4], depth[:, :1], normals, mask, emb, noise_type="uniform")


# ---- host wiring on emulated kernels against the oracle's autograd
@pytest.mark.parametrize("prediction_type", ["v_prediction", "epsilon"])
@pytest.mark.parametrize("noise_type", ["gaussian", "pyramid", "zeros"])
def test_diffusion_step_wiring(emulated, prediction_type, noise_type):
    r = DC.run_diffusion_step_tiny("cpu", prediction_type, noise_type)
    assert not r["missing"], r["missing"]
    assert r["target_rel"] <= 3e-3, r                           # the geometry latents come from the fp16-operand encoder
    assert r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


@pytest.mark.parametrize("hw", [(60, 68), (127, 161)])
def test_diffusion_step_wiring_ragged_size(emulated, hw):
    """Image sizes that are not multiples of 8: the latent (7x8, 15x20) is the 8x8-pooled mask's size."""
    r = DC.run_diffusion_step_tiny("cpu", "v_prediction", "gaussian", hw=hw)
    assert not r["missing"] and r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


def test_diffusion_step_draws_timesteps_on_the_host(emulated, monkeypatch):
    """timesteps=None: randint with the CPU generator, shared by both halves, handed to the kernel with its host copy."""
    import make_golden as MG
    import engine_checks as EC
    seen = {}

    def spy(rgb_latents, x0, noise, timesteps, alphas_cumprod, prediction_type, timesteps_host=None):
        seen.update(t=timesteps.clone(), host=timesteps_host)
        return diffusion_inputs(rgb_latents, x0, noise, timesteps, alphas_cumprod, prediction_type)
    monkeypatch.setattr(ops, "diffusion_inputs", spy)
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(gunet_ref, vae_ref, "cpu")
    rgb, depth, normals, mask, emb = DC.diffusion_batch(2, (64, 64))
    training.diffusion_loss_geowizard(unet, vae, DDIMScheduler(), rgb, depth, normals, mask, emb,
                                      generator=torch.Generator().manual_seed(3))
    want = torch.randint(0, 1000, (2,), generator=torch.Generator().manual_seed(3)).repeat(2)
    assert torch.equal(seen["t"], want) and torch.equal(seen["host"], want) and seen["host"].device.type == "cpu"


def test_diffusion_step_empty_mask_gives_zero_loss_and_gradient(emulated):
    r = DC.run_diffusion_step_tiny("cpu", empty=True)
    assert r["loss_engine"] == 0.0 and r["loss_oracle"] == 0.0 and r["grad_abs_max"] == 0.0, r


@pytest.mark.parametrize("noise_type", ["gaussian", "pyramid"])
def test_noisy_start_e2e_wiring(emulated, noise_type):
    r = DC.run_noisy_e2e_step_tiny("cpu", noise_type)
    assert not r["missing"] and r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 3e-2 and r["grad_worst"] <= 9e-2, r
    r = DC.run_noisy_e2e_geowizard_tiny("cpu", noise_type)
    assert not r["missing"] and r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 6e-2 and r["grad_worst"] <= 0.2, r


# ---- the EMA of the weights
def _trainer(use_ema=True):
    import make_golden as MG
    import engine_checks as EC
    gunet_ref, _ = MG.build_tiny("geowizard")
    unet, _ = EC.engine_from_oracle(gunet_ref, None, "cpu")
    unet.requires_grad_(True)
    return unet, training.FlatTrainer(unet, lr=1e-3, use_ema=use_ema)


def _step_with(tr, grads):
    tr.flat_grad.copy_(grads * tr.loss_scale())
    tr._micro, tr._synced = 0, True
    tr.step()


def test_ema_decay_schedule_matches_emamodel():
    ref = DO.EMARef([])
    for k in range(1, 40):
        assert training.ema_decay(k) == ref.get_decay(k)
    assert training.ema_decay(1) == 0.0 and training.ema_decay(2) == 2 / 11
    assert training.ema_decay(10 ** 7) == 0.9999


def test_ema_buffer_follows_emamodel_including_skipped_steps(emulated):
    unet, tr = _trainer()
    assert torch.equal(tr.ema, tr.flat_param)
    g = torch.Generator().manual_seed(9)
    ref = DO.EMARef([tr.flat_param.numpy()])
    for k in range(5):
        grads = torch.randn(tr.flat_param.shape, generator=g) * 1e-2
        if k == 2:
            grads.zero_()                                       # all masks empty: AdamW skips, the EMA still steps
        _step_with(tr, grads)
        ref.step([tr.flat_param.numpy()])
        assert np.array_equal(tr.ema.numpy(), ref.shadow[0]), k
    assert tr.skipped_steps() == 1 and tr.applied_steps() == 4 and tr.ema_steps == 5
    assert not torch.equal(tr.ema, tr.flat_param)


def test_ema_store_copy_to_restore_round_trip(emulated, tmp_path):
    from diffusion_e2e_ft_b200 import modules
    unet, tr = _trainer()
    for k in range(3):
        _step_with(tr, torch.full(tr.flat_param.shape, 1e-2 * (k + 1)))
    live = tr.flat_param.clone()
    epoch = modules._WEIGHTS_EPOCH[0]
    tr.store()
    tr.copy_to()
    assert torch.equal(tr.flat_param, tr.ema) and modules._WEIGHTS_EPOCH[0] > epoch
    name, off, shape = tr._layout[5]
    assert torch.equal(dict(unet.named_parameters())[name].detach().reshape(-1), tr.ema[off:off + math.prod(shape)])
    tr.restore()
    assert torch.equal(tr.flat_param, live)
    with pytest.raises(RuntimeError):
        tr.restore()
    # saving the EMA in the middle of a caller's store() / restore() leaves both the live weights and the store alone
    tr.store()
    tr.copy_to()
    tr.save_ema(str(tmp_path / "unet_ema"))
    tr.restore()
    assert torch.equal(tr.flat_param, live)
    with pytest.raises(RuntimeError):
        _trainer(use_ema=False)[1].copy_to()


def test_ema_save_load_continues_schedule(emulated, tmp_path):
    unet, tr = _trainer()
    g = torch.Generator().manual_seed(4)
    seq = [torch.randn(tr.flat_param.shape, generator=g) * 1e-2 for _ in range(5)]
    for s in seq[:3]:
        _step_with(tr, s)
    tr.save_ema(str(tmp_path / "unet_ema"))
    cfg = json.load(open(tmp_path / "unet_ema" / "config.json"))
    assert cfg["optimization_step"] == 3 and cfg["decay"] == 0.9999 and cfg["_class_name"] == "UNet2DConditionModel"
    assert "_extra" not in unet.config or "optimization_step" not in unet.config["_extra"]
    state = [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq, tr.state)]
    ema_saved = tr.ema.clone()
    # the saved folder loads as a plain diffusers UNet carrying the EMA weights
    from diffusion_e2e_ft_b200 import B200UNet2DConditionModel
    m = B200UNet2DConditionModel.from_pretrained(str(tmp_path / "unet_ema"))
    name, off, shape = tr._layout[-1]
    assert torch.equal(dict(m.named_parameters())[name].reshape(-1), ema_saved[off:off + math.prod(shape)])
    for s in seq[3:]:
        _step_with(tr, s)
    want = tr.ema.clone()
    # resume: a fresh trainer with the optimizer state of step 3 and the EMA from disk continues identically
    unet2, tr2 = _trainer()
    for dst, src in zip((tr2.flat_param, tr2.exp_avg, tr2.exp_avg_sq, tr2.state), state):
        dst.copy_(src)
    tr2.load_ema(str(tmp_path / "unet_ema"))
    assert tr2.ema_steps == 3 and torch.equal(tr2.ema, ema_saved)
    for s in seq[3:]:
        _step_with(tr2, s)
    assert torch.equal(tr2.ema, want)
