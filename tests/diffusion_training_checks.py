"""Graph-level parity of the diffusion-objective micro-step, the noisy-start E2E steps and the EMA trainer: the engine
(CUDA kernels, or their plain-torch contracts on the CPU) against torch.autograd through the fp32 oracle on identical
seeded weights, inputs, timesteps and noise.  Shared by tests/test_diffusion_training_cpu.py / _gpu.py and tools/."""
import random

import numpy as np
import torch

import diffusion_training_oracle as DO
import engine_checks as EC
from diffusion_e2e_ft_b200 import DDIMScheduler
from oracle import pipeline as OP
import make_golden as MG


def grad_report(unet, ref_named, scale):
    """global rel-L2 over all UNet parameter gradients, the worst parameter (ignoring vanishing ones), missing ones."""
    ref = dict(ref_named)
    num = den = 0.0
    missing = []
    pairs = []
    for n, p in unet.named_parameters():
        if p.grad is None:
            missing.append(n)
            continue
        ge, gr = p.grad.detach().float().cpu() / scale, ref[n].grad
        gr = torch.zeros_like(ge) if gr is None else gr
        pairs.append((n, ge, gr))
        num += (ge - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    worst, worst_name = 0.0, None
    for n, ge, gr in pairs:
        e = EC.rel_l2(ge, gr)
        if e > worst and gr.norm() > 1e-3 * den ** 0.5:
            worst, worst_name = e, n
    return dict(grad_global=(num / max(den, 1e-30)) ** 0.5, grad_worst=worst, worst_name=worst_name, missing=missing)


def _seed_all(seed):
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)


def diffusion_batch(B=2, hw=(64, 64), seed=31, empty=False):
    g = torch.Generator().manual_seed(seed)
    H, W = hw
    rgb = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    depth = (torch.rand(B, 1, H, W, generator=g) * 2 - 1).expand(-1, 3, -1, -1).contiguous()
    normals = torch.nn.functional.normalize(torch.randn(B, 3, H, W, generator=g), dim=1)
    mask = torch.rand(B, 1, H, W, generator=g) > 0.01           # most 8x8 blocks stay valid, some do not
    if empty:
        mask[:, :, ::8, ::8] = False                           # one invalid pixel in every block: empty latent mask
    emb = torch.randn(B, 1, 96, generator=g) * 0.5
    return rgb, depth, normals, mask, emb


def run_diffusion_step_tiny(device="cuda:0", prediction_type="v_prediction", noise_type="gaussian",
                            timesteps=(7, 613), hw=(64, 64), empty=False):
    """One diffusion-objective micro-step (train_depth_normal.py:600-717) on the tiny GeoWizard UNet / VAE: engine
    `training.diffusion_loss_geowizard` + backward vs the oracle graph + torch.autograd."""
    from diffusion_e2e_ft_b200.pipelines import geowizard_pyramid_noise_like
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, diffusion_loss_geowizard
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(gunet_ref, vae_ref, device)
    unet.requires_grad_(True)
    gunet_ref.requires_grad_(True)
    vae_ref.requires_grad_(False)
    B = 2
    rgb, depth, normals, mask, emb = diffusion_batch(B, hw, empty=empty)
    t = torch.tensor(list(timesteps), dtype=torch.long).repeat(2)
    sched = DDIMScheduler(prediction_type=prediction_type)
    gen = torch.Generator(device=device).manual_seed(5) if noise_type == "gaussian" else None
    _seed_all(11)
    loss, pred, target = diffusion_loss_geowizard(unet, vae, sched, rgb.to(device), depth.to(device), normals.to(device),
                                                  mask.to(device), emb.to(device), "indoor", noise_type=noise_type,
                                                  timesteps=t, generator=gen)
    (loss * LOSS_SCALE).backward()
    h, w = hw[0] // 8, hw[1] // 8
    shape = (2 * B, 4, h, w)
    if noise_type == "gaussian":                                  # the same draw, reproduced from the same seed
        noise = torch.randn(shape, device=device, generator=torch.Generator(device=device).manual_seed(5)).cpu()
    elif noise_type == "pyramid":
        _seed_all(11)
        noise = geowizard_pyramid_noise_like(torch.zeros(shape, device=device), t.to(device)).cpu()
    else:
        noise = None
    want, pred_o, target_o = DO.geowizard_diffusion_loss(gunet_ref, vae_ref, rgb, depth, normals, mask, emb, t, noise,
                                                         sched.alphas_cumprod, prediction_type)
    want.backward()
    out = dict(loss_engine=loss.item(), loss_oracle=want.item(),
               loss_rel=abs(loss.item() - want.item()) / max(abs(want.item()), 1e-30),
               target_rel=EC.rel_l2(target, target_o), pred_rel=EC.rel_l2(pred, pred_o))
    out.update(grad_report(unet, gunet_ref.named_parameters(), LOSS_SCALE))
    if empty:
        out["grad_abs_max"] = max(p.grad.abs().max().item() for p in unet.parameters() if p.grad is not None)
    return out


def _noise_like(noise_type, shape, device, seed, timesteps=None):
    """Reproduces the draw `training._start_latent` made after `_seed_all(seed)` / with a generator seeded `seed`."""
    from diffusion_e2e_ft_b200.pipelines import geowizard_pyramid_noise_like, pyramid_noise_like
    if noise_type == "zeros":
        return torch.zeros(shape)
    if noise_type == "gaussian":
        return torch.randn(shape, device=device, generator=torch.Generator(device=device).manual_seed(seed)).cpu()
    _seed_all(seed)
    z = torch.zeros(shape, device=device)
    if timesteps is None:
        return pyramid_noise_like(z, generator=torch.Generator(device=device).manual_seed(seed)).cpu()
    return geowizard_pyramid_noise_like(z, timesteps).cpu()


def run_noisy_e2e_step_tiny(device="cuda:0", noise_type="gaussian"):
    """Marigold depth E2E micro-step (train.py:469-556) from a noisy start x_t = noise at t = 999."""
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss
    unet_ref, vae_ref = MG.build_tiny()
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, device)
    unet.requires_grad_(True)
    unet_ref.requires_grad_(True)
    vae_ref.requires_grad_(False)
    g = torch.Generator().manual_seed(13)
    rgb = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    ctx = torch.randn(1, 77, 128, generator=g) * 0.5
    mask = torch.rand(2, 1, 64, 64, generator=g) > 0.2
    gt = torch.rand(2, 1, 64, 64, generator=g) * 9.9 + 0.1
    _seed_all(3)
    got, _ = e2e_ft_loss(unet, vae, DDIMScheduler(), rgb.to(device), gt.to(device), mask.to(device), ctx.to(device),
                         "depth", noise_type=noise_type, generator=torch.Generator(device=device).manual_seed(3))
    (got * LOSS_SCALE).backward()
    x_t = _noise_like(noise_type, (2, 4, 8, 8), device, 3)
    with torch.no_grad():
        lat = OP.encode_rgb(vae_ref, rgb)
    v = unet_ref(torch.cat([lat, x_t], 1), 999, ctx.repeat(2, 1, 1)).sample
    dec = OP.decode_latent(vae_ref, OP.DDIMOneStep().pred_original_sample(v, 999, x_t))
    want = OP.ssi_loss(dec.mean(1, keepdim=True).clamp(-1, 1), gt, mask)
    want.backward()
    out = dict(loss_engine=got.item(), loss_oracle=want.item(), loss_rel=abs(got.item() - want.item()) / abs(want.item()))
    out.update(grad_report(unet, unet_ref.named_parameters(), LOSS_SCALE))
    return out


def run_noisy_e2e_geowizard_tiny(device="cuda:0", noise_type="gaussian"):
    """GeoWizard joint E2E micro-step (train_depth_normal.py:640-766, `--e2e_ft`) from a noisy start."""
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss_geowizard
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(gunet_ref, vae_ref, device)
    unet.requires_grad_(True)
    gunet_ref.requires_grad_(True)
    vae_ref.requires_grad_(False)
    g = torch.Generator().manual_seed(17)
    B = 2
    rgb = torch.rand(B, 3, 64, 64, generator=g) * 2 - 1
    emb = torch.randn(B, 1, 96, generator=g) * 0.5
    mask = torch.rand(B, 1, 64, 64, generator=g) > 0.2
    gt_d = torch.rand(B, 1, 64, 64, generator=g) * 9.9 + 0.1
    gt_n = torch.nn.functional.normalize(torch.randn(B, 3, 64, 64, generator=g), dim=1)
    _seed_all(3)
    got, _, _ = e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb.to(device), gt_d.to(device), gt_n.to(device),
                                      mask.to(device), emb.to(device), "indoor", noise_type=noise_type,
                                      generator=torch.Generator(device=device).manual_seed(3))
    (got * LOSS_SCALE).backward()
    x_t = _noise_like(noise_type, (2 * B, 4, 8, 8), device, 3, torch.full((2 * B,), 999, device=device))
    with torch.no_grad():
        lat = OP.encode_rgb(vae_ref, rgb)
    x = torch.cat([lat.repeat(2, 1, 1, 1), x_t], 1)
    cls = OP.geowizard_class_embedding("indoor", rgb.dtype, B)
    v = gunet_ref(x, torch.full((2 * B,), 999), encoder_hidden_states=emb.repeat(2, 1, 1), class_labels=cls).sample
    dec = OP.decode_latent(vae_ref, OP.DDIMOneStep().pred_original_sample(v, 999, x_t))
    est_d = dec[:B].mean(1, keepdim=True).clamp(-1, 1)
    est_n = (dec[B:] / (dec[B:].norm(dim=1, keepdim=True) + 1e-5)).clamp(-1, 1)
    want = 0.5 * OP.ssi_loss(est_d, gt_d, mask) + OP.angular_loss(est_n, -gt_n, mask)
    want.backward()
    out = dict(loss_engine=got.item(), loss_oracle=want.item(), loss_rel=abs(got.item() - want.item()) / abs(want.item()))
    out.update(grad_report(unet, gunet_ref.named_parameters(), LOSS_SCALE))
    return out


def run_ema_loop_tiny(device="cuda:0", steps=3, lr=1e-4):
    """3 diffusion-objective steps through FlatTrainer(use_ema=True) vs torch AdamW + clip_grad_norm_ + EMARef on the
    oracle graph.  Reports the update cosine / norm ratio of the parameters and of the EMA weights."""
    from diffusion_e2e_ft_b200.training import FlatTrainer, diffusion_loss_geowizard
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(gunet_ref, vae_ref, device)
    unet.requires_grad_(True)
    gunet_ref.requires_grad_(True)
    vae_ref.requires_grad_(False)
    names = [n for n, _ in gunet_ref.named_parameters()]
    start = {n: p.detach().clone() for n, p in gunet_ref.named_parameters()}
    opt = torch.optim.AdamW(gunet_ref.parameters(), lr=lr, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    ema_ref = DO.EMARef([p.detach().numpy() for p in gunet_ref.parameters()])
    tr = FlatTrainer(unet, lr=lr, weight_decay=1e-2, max_grad_norm=1.0, use_ema=True)
    sched = DDIMScheduler()
    le, lo = [], []
    for k in range(steps):
        rgb, depth, normals, mask, emb = diffusion_batch(2, (64, 64), seed=40 + k)
        t = torch.tensor([100 + 300 * k, 850 - 200 * k]).repeat(2)
        gen = torch.Generator(device=device).manual_seed(50 + k)
        loss_e, _, _ = diffusion_loss_geowizard(unet, vae, sched, rgb.to(device), depth.to(device), normals.to(device),
                                                mask.to(device), emb.to(device), noise_type="gaussian", timesteps=t,
                                                generator=gen)
        tr.backward(loss_e)
        tr.step()
        noise = torch.randn((4, 4, 8, 8), device=device, generator=torch.Generator(device=device).manual_seed(50 + k)).cpu()
        loss_o, _, _ = DO.geowizard_diffusion_loss(gunet_ref, vae_ref, rgb, depth, normals, mask, emb, t, noise,
                                                   sched.alphas_cumprod)
        opt.zero_grad()
        loss_o.backward()
        torch.nn.utils.clip_grad_norm_(gunet_ref.parameters(), 1.0)
        opt.step()
        ema_ref.step([p.detach().numpy() for p in gunet_ref.parameters()])
        le.append(loss_e.item())
        lo.append(loss_o.item())
    ema_of = {}
    for name, off, shape in tr._layout:
        n = int(np.prod(shape))
        ema_of[name] = tr.ema[off:off + n].view(shape).float().cpu()
    out = dict(loss_engine=le, loss_oracle=lo, ema_steps=tr.ema_steps)
    for key, eng, ref in (("update", {n: p.detach().float().cpu() for n, p in unet.named_parameters()},
                           {n: p.detach() for n, p in gunet_ref.named_parameters()}),
                          ("ema", ema_of, {n: torch.from_numpy(s) for n, s in zip(names, ema_ref.shadow)})):
        dot = ne = no = 0.0
        for n in names:
            de, do = eng[n] - start[n], ref[n] - start[n]
            dot += (de * do).sum().item()
            ne += de.pow(2).sum().item()
            no += do.pow(2).sum().item()
        out[key + "_cosine"] = dot / (ne * no) ** 0.5
        out[key + "_norm_ratio"] = (ne / no) ** 0.5
    return out
