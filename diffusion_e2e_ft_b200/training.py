"""Forward half of the E2E fine-tuning step (training/train.py:469-556) on the engine.

    rgb -> VAE.encode * scaling -> UNet(t = T-1, zeros noise, ctx[B,77,1024]) -> x0 (v-prediction)
        -> / scaling -> VAE.decode -> depth: mean_c, clamp | normals: normalise, clamp -> SSI / angular loss

Everything runs in libb200_e2eft.so kernels (incl. the losses).  `e2e_ft_forward` is the no-grad forward (loss value
only); `e2e_ft_loss` is the differentiable one: `e2e_ft_loss(...)[0].backward()` fills `.grad` of the UNet
parameters through the autograd blocks (autograd_blocks.py), `optimizer_step_` then does the gradient all-reduce,
clipping and AdamW on flat buffers.
"""
import math

import torch

from . import ops


def _check_noise_type(noise_type):
    from .pipelines import NOISE_TYPES
    if noise_type not in NOISE_TYPES:
        raise ValueError(f"Unknown noise type {noise_type}")


def _start_latent(noise_type, like, generator=None, timesteps=None):
    """The noisy start x_t of an E2E fine-tuning step (train.py:484-491, train_depth_normal.py:656-668): None for
    zeros (the x_t = 0 graph), `randn` with `generator`, or the recipe's pyramid noise (Marigold's when `timesteps`
    is None, GeoWizard's scaled by timesteps / 1000 otherwise)."""
    from .pipelines import geowizard_pyramid_noise_like, pyramid_noise_like
    if noise_type == "zeros":
        return None
    if noise_type == "gaussian":
        return torch.randn(like.shape, device=like.device, dtype=like.dtype, generator=generator)
    if timesteps is None:
        return pyramid_noise_like(like, generator=generator)
    return geowizard_pyramid_noise_like(like, timesteps)


def _e2e_unet_input(rgb_latents, x_t):
    return torch.cat((rgb_latents, torch.zeros_like(rgb_latents) if x_t is None else x_t), dim=1)


def _decode_x0(vae, model_pred, a_t, x_t):
    """x0 = sqrt(a) x_t - sqrt(1 - a) v (v_prediction, train.py:509-511), folded into post_quant_conv, then decoded."""
    if x_t is None:
        return vae.decode_from_prediction(model_pred, -math.sqrt(1.0 - a_t))
    return vae.decode_from_prediction(model_pred, -math.sqrt(1.0 - a_t), noisy=x_t.float().contiguous(),
                                      c_noisy=math.sqrt(a_t))


@torch.no_grad()
def e2e_ft_forward(unet, vae, scheduler, rgb, ground_truth, val_mask, empty_encoding, modality="depth",
                   noise_type="zeros", generator=None):
    """Returns (loss [0-d fp32 tensor], current_estimate).  rgb [B,3,H,W] in [-1,1]; ground_truth [B,1,H,W]
    metric depth or [B,3,H,W] normals; val_mask [B,1,H,W] bool; empty_encoding [1,77,1024].  `noise_type`: the
    start latent x_t at t = T-1 (zeros, gaussian drawn with `generator`, or pyramid)."""
    _check_noise_type(noise_type)
    B = rgb.shape[0]
    rgb_latents = vae.encode_scaled_mean(rgb)                                   # train.py:473-474
    T = scheduler.config["num_train_timesteps"]
    t = T - 1                                                                   # :480-481
    x_t = _start_latent(noise_type, rgb_latents, generator)                     # :484-491
    ctx = empty_encoding.to(rgb.device).repeat(B, 1, 1)
    model_pred = unet(_e2e_unet_input(rgb_latents, x_t), t, ctx, return_dict=False)[0]     # :494-500
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = _decode_x0(vae, model_pred, a_t, x_t)                                 # :509-529
    est = ops.decode_post(dec.float().contiguous(), normals=(modality == "normals"), training=True)   # :532-540
    if modality == "depth":
        loss = ops.ssi_loss(est, ground_truth, val_mask)                        # :545
    elif modality == "normals":
        loss = ops.angular_loss(est, ground_truth, val_mask)                    # :549
    else:
        raise ValueError(f"Unknown modality {modality}")
    return loss, est


LOSS_SCALE = 1024.0       # static loss scale: incoming gradients are fp16 GEMM operands in the backward pass


def e2e_ft_loss(unet, vae, scheduler, rgb, ground_truth, val_mask, empty_encoding, modality="depth",
                noise_type="zeros", generator=None):
    """Differentiable training micro-step (training/train.py:469-556).  Returns (loss, estimate); call
    `(loss * LOSS_SCALE).backward()` and divide the gradients by LOSS_SCALE (or pass `grad_unscale` to the
    optimizer step).  VAE encode runs without grad (frozen, train.py:473 under no_grad).  `noise_type` as in
    `e2e_ft_forward` (train.py:484-491); the default zeros keeps the x_t = 0 graph."""
    from . import autograd_blocks as ab
    _check_noise_type(noise_type)
    if modality not in ("depth", "normals"):
        raise ValueError(f"Unknown modality {modality}")
    B = rgb.shape[0]
    with torch.no_grad():
        rgb_latents = vae.encode_scaled_mean(rgb)
        x_t = _start_latent(noise_type, rgb_latents, generator)
    T = scheduler.config["num_train_timesteps"]
    t = T - 1
    ctx = empty_encoding.to(rgb.device).repeat(B, 1, 1)
    model_pred = unet(_e2e_unet_input(rgb_latents, x_t), t, ctx, return_dict=False)[0]
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = _decode_x0(vae, model_pred, a_t, x_t)
    normals = modality == "normals"
    est = ab.decode_post(dec, normals)
    return ab.task_loss(est, ground_truth, val_mask, normals), est


def e2e_ft_loss_geowizard(unet, vae, scheduler, rgb, depth_gt, normal_gt, val_mask, img_embed, domain="indoor",
                          depth_scale=0.5, normal_scale=1.0, noise_type="zeros", generator=None):
    """Differentiable joint depth + normal micro-step of the GeoWizard recipe
    (GeoWizard/geowizard/training/train_depth_normal.py:640-766, `--e2e_ft`, zeros noise): one UNet call on the
    [depth x B | normal x B] batch with the hybrid class embedding and joint self-attention, x0 by the v-prediction closed
    form, ONE decoder pass over both halves, depth = clamp(mean_c), normals = clamp(x / (|x| + 1e-5)),
    loss = depth_scale * SSI(depth) + normal_scale * angular(normals, -normal_gt)   (the reference trains on inverted
    normals, :742).  rgb [B,3,H,W], depth_gt [B,1,H,W], normal_gt [B,3,H,W], val_mask [B,1,H,W] bool, img_embed
    [B,1,768] (CLIP image embedding).  `noise_type` (:656-668): the start x_t at t = T-1 over both halves — zeros
    (default, today's graph), gaussian (one independent draw over the [2B] batch, :661, with `generator`) or GeoWizard's
    pyramid noise.  Returns (loss, depth_estimate, normal_estimate)."""
    from . import autograd_blocks as ab
    from .pipelines import DepthNormalEstimationPipeline
    _check_noise_type(noise_type)
    B = rgb.shape[0]
    dev = rgb.device
    T = scheduler.config["num_train_timesteps"]
    t = T - 1                                                                             # :646-648
    timesteps = torch.full((2 * B,), t, device=dev, dtype=torch.long)
    with torch.no_grad():
        rgb_latents = vae.encode_scaled_mean(rgb)
        rgb2 = rgb_latents.repeat(2, 1, 1, 1)
        x_t = _start_latent(noise_type, rgb2, generator, timesteps)
    x = _e2e_unet_input(rgb2, x_t)                                                        # :705
    ctx = img_embed.to(dev).repeat(2, 1, 1)                                               # :683
    cls = DepthNormalEstimationPipeline.class_embedding(domain, B, dev, rgb_latents.dtype)                   # :686-703
    pred = unet(x, timesteps, ctx, class_labels=cls, return_dict=False)[0]
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = _decode_x0(vae, pred, a_t, x_t)                                                 # :722-737, one decoder pass
    est_d = ab.decode_post(dec[:B].contiguous(), False)                                   # :739-741
    est_n = ab.decode_post(dec[B:].contiguous(), True)                                    # :743-746
    loss_d = ab.task_loss(est_d, depth_gt, val_mask, False)
    loss_n = ab.task_loss(est_n, -normal_gt, val_mask, True)
    return depth_scale * loss_d + normal_scale * loss_n, est_d, est_n


def _latent_hw(vae, H, W):
    """Latent size of an H x W image: every encoder down block pads (0, 1, 0, 1) and runs a pad-0 stride-2 conv
    (Downsample2D with padding 0), i.e. floor(H / 2) per level."""
    for _ in range(len(vae.config["block_out_channels"]) - 1):
        H, W = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    return H, W


def _randn(shape, device, generator):
    """randn on `device` with `generator`; a generator on another device (e.g. a CPU generator for a CUDA run) draws
    where it lives and the result is copied over."""
    if generator is None or generator.device.type == torch.device(device).type:
        return torch.randn(shape, device=device, dtype=torch.float32, generator=generator)
    return torch.randn(shape, device=generator.device, dtype=torch.float32, generator=generator).to(device)


def _device_alphas_cumprod(scheduler, device):
    cache = scheduler.__dict__.setdefault("_ac_device", {})
    key = str(device)
    if key not in cache:
        cache[key] = scheduler.alphas_cumprod.to(device=device, dtype=torch.float32).contiguous()
    return cache[key]


def diffusion_loss_geowizard(unet, vae, scheduler, rgb, depth, normals, val_mask, img_embed, domain="indoor",
                             noise_type="gaussian", timesteps=None, generator=None):
    """Differentiable micro-step of GeoWizard's diffusion objective (GeoWizard/geowizard/training/train_depth_normal.py
    :600-717 without `--e2e_ft`, the script's default).  rgb [B,3,H,W] and depth [B,3,H,W] (or [B,1,H,W], stacked to
    3 channels as the dataset does) in [-1, 1]; normals [B,3,H,W] as the dataset gives them (inverted here, :606);
    val_mask [B,1,H,W] bool; img_embed [B,1,768].

    One frozen VAE encode of cat(rgb, depth, normals) (:633-639); per-image timesteps shared by the two halves
    (`timesteps=None`: randint(0, T, (B,)).repeat(2) drawn on the host — with `generator` when it is a CPU generator,
    else with torch's default CPU generator — so the range check needs no device sync; or pass [B] / [2B] host
    integers); noise (:656-668): zeros, gaussian (randn with `generator`) or GeoWizard's pyramid noise scaled by the
    [2B] timesteps;
    then one `b200_diffusion_inputs` kernel (add_noise, the epsilon / velocity target, the UNet-input concatenation),
    the UNet with the hybrid class embedding, and the masked latent MSE (:712-714).  The prediction type comes from
    `scheduler.config["prediction_type"]` (epsilon or v_prediction).  Returns (loss, noise_pred, target).  An empty
    latent mask gives loss 0 and an all-zero gradient, which FlatTrainer's zero-gradient skip turns into no update."""
    from . import autograd_blocks as ab
    from .pipelines import DepthNormalEstimationPipeline, geowizard_pyramid_noise_like
    _check_noise_type(noise_type)
    pt = scheduler.config["prediction_type"]
    if pt not in ops.DIFFUSION_PREDICTION_TYPES:
        raise ValueError(f"Unknown prediction type {pt}")
    B, _, H, W = rgb.shape
    dev = rgb.device
    T = scheduler.config["num_train_timesteps"]
    h, w = _latent_hw(vae, H, W)
    ops.latent_mask_shape(val_mask, torch.empty((2 * B, vae.config["latent_channels"], h, w), device="meta"))
    if timesteps is None:
        host_gen = generator if generator is not None and generator.device.type == "cpu" else None
        timesteps = torch.randint(0, T, (B,), generator=host_gen).repeat(2)
    t_host = torch.as_tensor(timesteps).to("cpu", torch.long).reshape(-1)
    if t_host.numel() == B:
        t_host = t_host.repeat(2)
    if t_host.numel() != 2 * B or not bool(((t_host >= 0) & (t_host < T)).all()):
        raise ValueError(f"timesteps {t_host.tolist()} must be B or 2B integers in [0, {T})")
    t_dev = t_host.to(dev)
    if depth.shape[1] == 1:
        depth = depth.expand(-1, 3, -1, -1)
    with torch.no_grad():
        lat = vae.encode_scaled_mean(torch.cat((rgb, depth, -normals), dim=0).float())           # :633-639
        rgb_latents, geo = lat[:B].contiguous(), lat[B:].contiguous()
        if noise_type == "zeros":
            noise = None
        elif noise_type == "gaussian":
            noise = _randn(geo.shape, dev, generator)
        else:
            noise = geowizard_pyramid_noise_like(geo, t_dev).float().contiguous()
        x, target = ops.diffusion_inputs(rgb_latents, geo, noise, t_dev, _device_alphas_cumprod(scheduler, dev), pt,
                                         timesteps_host=t_host)
    ctx = img_embed.to(dev).repeat(2, 1, 1)                                                        # :683
    cls = DepthNormalEstimationPipeline.class_embedding(domain, B, dev, torch.float32)             # :686-703
    pred = unet(x, t_dev, ctx, class_labels=cls, return_dict=False)[0]
    return ab.masked_latent_mse(pred, target, val_mask), pred, target


def allreduce_mean_(flat_grad, group=None):
    """DDP gradient exchange of the fine-tuning step (training/train.py:470,563 via accelerate): one all-reduce
    of the flat gradient buffer over the data-parallel ranks, averaged.  NCCL over NVLink on the GPU box, gloo
    in the CPU tests.  No-op without an initialised process group."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return flat_grad
    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    flat_grad.div_(dist.get_world_size(group))
    return flat_grad


def optimizer_step_(flat_param, flat_grad, exp_avg, exp_avg_sq, step, lr=3e-5, weight_decay=1e-2, max_grad_norm=1.0,
                    group=None, grad_unscale=1.0):
    """all-reduce -> clip_grad_norm_(max_grad_norm) -> AdamW, fused on the device without host syncs
    (training/train.py:563-566 with the recipe of training/scripts/train_marigold_e2e_ft_depth.sh).
    `grad_unscale` = 1 / loss scale when the gradient buffer is loss-scaled."""
    from .modules import bump_weights_epoch
    allreduce_mean_(flat_grad, group)
    nsq = ops.grad_norm_sq(flat_grad)
    ops.adamw_step(flat_param, flat_grad, exp_avg, exp_avg_sq, step, lr=lr, weight_decay=weight_decay,
                   grad_norm_sq_t=nsq, max_grad_norm=max_grad_norm, grad_unscale=grad_unscale)
    bump_weights_epoch()
    return nsq


EMA_DECAY = 0.9999        # train_depth_normal.py:353: EMAModel defaults (min_decay 0, update_after_step 0, no warmup)


def ema_decay(step, decay=EMA_DECAY):
    """diffusers EMAModel.get_decay for the recipe's settings; `step` = EMA steps so far, this one included (1-based)."""
    s = max(0, step - 1)
    if s <= 0:
        return 0.0
    return max(0.0, min((1 + s) / (10 + s), decay))


def ema_config(step, decay=EMA_DECAY):
    """The EMAModel state that diffusers stores in the unet_ema config next to the weights."""
    return dict(decay=decay, min_decay=0.0, optimization_step=int(step), update_after_step=0, use_ema_warmup=False,
                inv_gamma=1.0, power=2 / 3)


ADAM_BETAS, ADAM_EPS = (0.9, 0.999), 1e-8        # train.py:346-353 / train_depth_normal.py:437-444 defaults


class IterExponential:
    """Marigold's iteration-wise LR factor (training/util/lr_scheduler.py, used by both recipes through LambdaLR):
    linear warm-up 0 -> 1 over `warmup_steps`, then exp(t / (total - warmup) * log(final_ratio)) in float64, held at
    `final_ratio` from `total_iter_length` on.  The attribute names are the reference's, so LambdaLR.state_dict()
    stores the same `lr_lambdas` entry and either side loads the other's scheduler.bin."""

    def __init__(self, total_iter_length, final_ratio, warmup_steps=0):
        self.total_length = total_iter_length
        self.effective_length = total_iter_length - warmup_steps
        self.final_ratio = final_ratio
        self.warmup_steps = warmup_steps

    def __call__(self, n_iter):
        import numpy as np
        if n_iter < self.warmup_steps:
            return 1.0 * n_iter / self.warmup_steps
        if n_iter >= self.total_length:
            return self.final_ratio
        return np.exp((n_iter - self.warmup_steps) / self.effective_length * np.log(self.final_ratio))


class ConstantLR:
    """GeoWizard's `--lr_scheduler constant` (diffusers get_scheduler("constant")): factor 1 on every step; the
    warm-up argument is ignored, as diffusers ignores it for this choice."""

    def __init__(self, *unused, **unused_kw):
        pass

    def __call__(self, n_iter):
        return 1.0


def geowizard_param_groups(class_embedding_lr_mult=10.0):
    """The two AdamW parameter groups of train_depth_normal.py:428-444: every parameter without `class_embedding` in
    its name at the base learning rate, then the `class_embedding.*` parameters at base * class_embedding_lr_mult
    (the script's default is 10).  Pass as FlatTrainer(..., param_groups=geowizard_param_groups())."""
    return [dict(name="params", select=lambda n: "class_embedding" not in n, lr_mult=1.0),
            dict(name="params_class_embedding", select=lambda n: "class_embedding" in n,
                 lr_mult=float(class_embedding_lr_mult))]


_CHECKPOINT_RE = r"checkpoint-(\d+)$"


def _checkpoints(output_dir):
    import os
    import re
    if not os.path.isdir(output_dir):
        return []
    found = [(int(m.group(1)), d) for d in os.listdir(output_dir) if (m := re.match(_CHECKPOINT_RE, d))]
    return [d for _, d in sorted(found)]


def latest_checkpoint(output_dir):
    """`--resume_from_checkpoint latest` (train.py:416-425): the path of the `checkpoint-N` folder in `output_dir`
    with the largest N (numeric order, so checkpoint-1000 follows checkpoint-900), or None when there is none."""
    import os
    cps = _checkpoints(output_dir)
    return os.path.join(output_dir, cps[-1]) if cps else None


def prune_checkpoints(output_dir, total_limit):
    """`--checkpoints_total_limit` (train.py:581-596), called BEFORE a save: delete the oldest `checkpoint-N` folders
    so that at most total_limit - 1 remain, making room for the one about to be written.  Returns the removed paths;
    total_limit None keeps everything."""
    import os
    import shutil
    if total_limit is None:
        return []
    cps = _checkpoints(output_dir)
    removed = [os.path.join(output_dir, d) for d in cps[:max(0, len(cps) - int(total_limit) + 1)]]
    for d in removed:
        shutil.rmtree(d)
    return removed


class FlatTrainer:
    """The optimizer side of training/train.py:346-353,560-568 for one module (the UNet): all trainable parameters
    and their gradients are re-homed as views of two flat fp32 buffers, so `backward()` accumulates straight into
    the buffer the gradient all-reduce and the fused clip + AdamW kernel work on.

        tr = FlatTrainer(unet, lr=3e-5, accumulation_steps=16)
        for batch in loader:                                      # one micro-batch per iteration
            loss, _ = e2e_ft_loss(unet, vae, scheduler, rgb, gt, mask, empty_encoding, "depth")
            tr.micro_step(loss)      # backward; on every `accumulation_steps`-th call also all-reduce + clip + AdamW

    (`tr.backward(loss); tr.step()` is the same thing spelled out for accumulation_steps == 1.)

    Gradient accumulation (`accelerator.accumulate`, train.py:470): micro-steps are counted here; only the LAST backward
    of an accumulation window exchanges gradients (DDP `no_sync` on the others), and `step()` refuses to run in the
    middle of a window.  Data parallel (one process per GPU, `torch.distributed` initialised): the flat gradient is cut
    into buckets of `bucket_mb` in gradient-ready order — the parameters whose gradients only arrive at the very end
    of backward (every resnet's `time_emb_proj` and the time / class embedding MLPs, produced by the embedding block
    that runs first in forward) get their own bucket, so they do not hold the others back.  With `overlap=True` a
    bucket's SUM all-reduce is launched asynchronously (NCCL stream) the moment autograd has accumulated its last
    parameter, as accelerate's DDP does for the reference; the DEFAULT is `overlap=False` — all buckets are reduced in
    `step()` after backward — because on this engine overlap can be a large loss: the GEMM / conv kernels are persistent
    with one ~200 KB-smem CTA per SM, so while NCCL's channel CTAs occupy SMs a 132-CTA grid no longer fits in one wave
    and the backward kernels take two.  Exposing the all-reduce of the 3.46 GB gradient buffer after backward is the
    safe choice at every N.  The 1/world_size of the average is folded into the optimizer kernel's
    gradient multiplier (no extra pass over the 3.46 GB buffer).

    Mixed precision: backward GEMM operands are fp16, so the loss is multiplied by a loss scale held ON THE DEVICE
    (`state[0]`); the fused optimizer kernel skips the step and halves the scale when the gradient norm is non-finite,
    doubles it after `growth_interval` good steps, and also skips when the gradient is exactly zero (all masks empty:
    train.py:503,546-551) — all without a host sync.  `skipped_steps()` / `loss_scale()` read the state back.

    Parameter groups (`param_groups`, torch.optim.AdamW's groups): None is one group over every trainable parameter
    (train.py:346-353).  Otherwise an ordered list of dicts `dict(name=..., select=lambda param_name: bool,
    lr_mult=1.0, weight_decay=None)`; each parameter joins the first group that selects it, trains at lr * lr_mult
    with the group's weight decay (None: the trainer's), and every parameter must land in a group.
    `geowizard_param_groups()` gives train_depth_normal.py:428-444.  The flat layout is not reordered: the fused
    kernel finds each element's group from a table of contiguous runs.  Group order, then named_parameters order
    within a group, numbers the parameters in the saved optimizer state, as torch numbers them.

    LR schedule (`lr_schedule`, e.g. `IterExponential(20000 * N, 0.01, 100 * N)` built with the reference's own
    arguments, or `ConstantLR()`): optimizer step k (0-based, every step() call counted) runs at
    lr_g = lr * lr_mult_g * lr_schedule(k * N), N = `num_processes` (default: the world size).  That is what LambdaLR
    gives under accelerate, whose scheduler wrapper steps it N times per optimizer step — INCLUDING lr = 0 on step 0
    with a warm-up, because LambdaLR applies lambda(0) before the first step.  Steps the device skips (zero or
    non-finite gradient) still advance the schedule, as the reference's scheduler steps after an AdamW step that
    updated nothing; so the rates are known on the host without a sync.  `get_last_lr()` is the rates of the next step.

    Checkpoints: `save_state(dir)` / `load_state(dir)` write and read accelerate's `checkpoint-N` folder (unet/,
    unet_ema/, optimizer.bin, scheduler.bin, random_states_{rank}.pkl) plus the engine's flat_trainer.pt;
    `latest_checkpoint` and `prune_checkpoints` are the scripts' folder logic."""

    LATE_GRAD_KEYS = ("time_emb_proj", "time_embedding", "class_embedding")

    def __init__(self, module, lr=3e-5, weight_decay=1e-2, max_grad_norm=1.0, accumulation_steps=1, group=None,
                 loss_scale=LOSS_SCALE, bucket_mb=256, dynamic_loss_scale=True, growth_interval=2000, overlap=False,
                 use_ema=False, param_groups=None, lr_schedule=None, num_processes=None):
        import torch.distributed as dist
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if not named:
            raise ValueError("no trainable parameters")
        self._group_def = self._resolve_groups(named, param_groups, weight_decay)
        late = [(n, p) for n, p in named if any(k in n for k in self.LATE_GRAD_KEYS)]
        rest = [(n, p) for n, p in named if not any(k in n for k in self.LATE_GRAD_KEYS)]
        ps = [p for _, p in late] + [p for _, p in rest]          # flat order == reverse gradient-ready order
        dev = ps[0].device
        sizes = [(p.numel() + 3) // 4 * 4 for p in ps]                     # keep every view 16-byte aligned
        total = sum(sizes)
        self.flat_param = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=dev)
        self.state = torch.zeros(8, dtype=torch.float32, device=dev)
        self.state[0] = float(loss_scale)
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        cap = max(1, int(bucket_mb * 2 ** 20 / 4))
        self._buckets, self._bucket_of = [], {}
        off = start = count = 0
        name_of = {id(p): n for n, p in named}
        self._layout = []                                          # (diffusers name, offset, shape) per parameter
        with torch.no_grad():
            for idx, (p, n) in enumerate(zip(ps, sizes)):
                if p.dtype != torch.float32:
                    raise TypeError("FlatTrainer expects fp32 master parameters")
                self._layout.append((name_of[id(p)], off, tuple(p.shape)))
                view = self.flat_param[off:off + p.numel()].view(p.shape)
                view.copy_(p.data)
                p.data = view
                p.grad = self.flat_grad[off:off + p.numel()].view(p.shape)
                self._bucket_of[id(p)] = len(self._buckets)
                off += n
                count += 1
                if off - start >= cap or idx == len(ps) - 1 or idx == len(late) - 1:
                    self._buckets.append(dict(lo=start, hi=off, n=count))
                    start, count = off, 0
        self.params, self.step_count = ps, 0
        # contiguous runs of one group along the flat layout, for the fused kernel
        group_of = {n: k for k, g in enumerate(self._group_def) for n in g["params"]}
        runs = []
        for name, off, _ in self._layout:
            if not runs or runs[-1][1] != group_of[name]:
                runs.append((off, group_of[name]))
        self._runs = runs
        self._run_table = None if len(runs) == 1 else ops.adamw_run_table(
            [r[0] for r in runs], [r[1] for r in runs], total, len(self._group_def), dev)
        self.lr_schedule = lr_schedule
        self.num_processes = int(num_processes) if num_processes is not None else self.world
        self._init_loss_scale = float(loss_scale)
        self.lr, self.weight_decay, self.max_grad_norm = lr, weight_decay, max_grad_norm
        self.accumulation_steps, self.group = max(1, int(accumulation_steps)), group
        self.dynamic_loss_scale, self.growth_interval, self.overlap = dynamic_loss_scale, growth_interval, overlap
        self._sync, self._ready, self._handles, self._micro, self._synced = True, [0] * len(self._buckets), {}, 0, True
        if self.world > 1:
            for p in ps:
                p.register_post_accumulate_grad_hook(self._on_grad)
        # EMA of the weights (train_depth_normal.py:351-353 `--use_ema`): one more flat buffer, cloned from the
        # parameters as EMAModel clones them, advanced by every step()
        self.module = module
        self.ema = self.flat_param.clone() if use_ema else None
        self.ema_steps = 0
        self._stored = None

    # autograd calls this right after it has added a parameter's gradient into its view of the flat buffer
    def _on_grad(self, p):
        if not (self._sync and self.overlap):
            return
        b = self._bucket_of[id(p)]
        self._ready[b] += 1
        if self._ready[b] == self._buckets[b]["n"]:
            self._launch(b)

    def _launch(self, b):
        import torch.distributed as dist
        bk = self._buckets[b]
        self._handles[b] = dist.all_reduce(self.flat_grad[bk["lo"]:bk["hi"]], op=dist.ReduceOp.SUM, group=self.group,
                                           async_op=True)

    def backward(self, loss, sync=None):
        """(loss * loss_scale / accumulation_steps).backward().  `sync=None`: exchange gradients only on the last
        micro-step of the accumulation window (counted here); an explicit True / False overrides."""
        last = (self._micro + 1) % self.accumulation_steps == 0
        sync = last if sync is None else bool(sync)
        if self._handles:
            raise RuntimeError("FlatTrainer.backward: gradient all-reduces of the previous backward are still in flight "
                               "— call step() first (or backward(..., sync=False) on non-final micro-steps)")
        self._sync, self._synced = sync, sync
        self._ready = [0] * len(self._buckets)
        self._micro += 1
        (loss * (self.state[0] / self.accumulation_steps)).backward()

    @staticmethod
    def _resolve_groups(named, param_groups, weight_decay):
        if param_groups is None:
            param_groups = [dict(name="params", select=None)]
        if not 1 <= len(param_groups) <= ops.ADAMW_MAX_GROUPS:
            raise ValueError(f"1..{ops.ADAMW_MAX_GROUPS} parameter groups, got {len(param_groups)}")
        groups = []
        for k, g in enumerate(param_groups):
            wd = g.get("weight_decay")
            groups.append(dict(name=str(g.get("name", f"group_{k}")), lr_mult=float(g.get("lr_mult", 1.0)),
                               weight_decay=float(weight_decay if wd is None else wd), params=[]))
        for n, _ in named:
            k = next((k for k, g in enumerate(param_groups) if g.get("select") is None or g["select"](n)), None)
            if k is None:
                raise ValueError(f"parameter {n} is in no parameter group")
            groups[k]["params"].append(n)
        return groups

    def _lrs(self, k, lr=None):
        """Per-group learning rates of optimizer step k (0-based)."""
        if self.lr_schedule is not None:
            f = self.lr_schedule(k * self.num_processes)
            return [float(self.lr * g["lr_mult"] * f) for g in self._group_def]
        base = self.lr if lr is None else lr
        return [base * g["lr_mult"] for g in self._group_def]

    def get_last_lr(self):
        """The per-group learning rates the next step() will use (LambdaLR.get_last_lr(), logged at train.py:575 /
        train_depth_normal.py:791)."""
        return self._lrs(self.step_count)

    def _check_lr_arg(self, lr):
        if lr is not None and self.lr_schedule is not None:
            raise ValueError("lr= and lr_schedule are exclusive: the schedule sets every step's learning rate")

    def micro_step(self, loss, lr=None):
        """backward(); on the last micro-step of the accumulation window also step().  Returns True when it stepped
        (`accelerator.sync_gradients` of train.py:563-570)."""
        self._check_lr_arg(lr)
        self.backward(loss)
        if self._micro % self.accumulation_steps == 0:
            self.step(lr)
            return True
        return False

    def step(self, lr=None):
        self._check_lr_arg(lr)
        if self._micro % self.accumulation_steps != 0 or not self._synced:
            raise RuntimeError(f"FlatTrainer.step inside an accumulation window ({self._micro % self.accumulation_steps} of "
                               f"{self.accumulation_steps} micro-steps) or after backward(sync=False): gradients are not reduced")
        lrs, wds = self._lrs(self.step_count, lr), [g["weight_decay"] for g in self._group_def]
        self.step_count += 1
        if self.world > 1:
            for b in range(len(self._buckets)):                    # parameters without a gradient this step / overlap off
                if b not in self._handles:
                    self._launch(b)
            for h in self._handles.values():
                h.wait()
            self._handles = {}
        from .modules import bump_weights_epoch
        nsq = ops.grad_norm_sq(self.flat_grad)
        if self._run_table is None:                                # one run: the whole buffer is one group
            k = self._runs[0][1]
            ops.adamw_step_state(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, self.state, nsq,
                                 lr=lrs[k], weight_decay=wds[k], max_grad_norm=self.max_grad_norm,
                                 inv_world=1.0 / self.world, dynamic_scale=self.dynamic_loss_scale,
                                 growth_interval=self.growth_interval)
        else:
            ops.adamw_step_state_groups(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, self.state, nsq,
                                        *self._run_table, lrs, wds, max_grad_norm=self.max_grad_norm,
                                        inv_world=1.0 / self.world, dynamic_scale=self.dynamic_loss_scale,
                                        growth_interval=self.growth_interval)
        bump_weights_epoch()
        self.flat_grad.zero_()
        if self.ema is not None:
            # diffusers steps the EMA whenever sync_gradients is true (:785-786), also when AdamW skipped the step
            self.ema_steps += 1
            ops.ema_update(self.ema, self.flat_param, 1.0 - ema_decay(self.ema_steps))
        return nsq

    # ---- EMA of the weights: EMAModel.store / copy_to / restore (:843-850) and unet_ema save / load (:380-391)
    def _need_ema(self):
        if self.ema is None:
            raise RuntimeError("FlatTrainer was built without use_ema=True")

    def store(self):
        """Keep a host copy of the current weights (EMAModel.store)."""
        self._need_ema()
        self._stored = self.flat_param.to("cpu", copy=True)

    def copy_to(self):
        """Load the EMA weights into the module's parameters (EMAModel.copy_to), e.g. for validation."""
        from .modules import bump_weights_epoch
        self._need_ema()
        self.flat_param.copy_(self.ema)
        bump_weights_epoch()

    def restore(self):
        """Put back the weights saved by store() (EMAModel.restore)."""
        from .modules import bump_weights_epoch
        self._need_ema()
        if self._stored is None:
            raise RuntimeError("restore() without a preceding store()")
        self.flat_param.copy_(self._stored)
        self._stored = None
        bump_weights_epoch()

    def save_ema(self, save_directory):
        """EMAModel.save_pretrained: the module in the diffusers layout with the EMA weights, the EMA settings in its
        config (`optimization_step` included, so a resumed run continues the decay schedule).  Written straight from
        the EMA buffer: the live weights and a pending store() are left alone."""
        self._need_ema()
        sd = self.module.state_dict()
        for name, off, shape in self._layout:
            sd[name] = self.ema[off:off + math.prod(shape)].view(shape)
        self.module.save_pretrained(save_directory, state_dict=sd, extra_config=ema_config(self.ema_steps))

    def load_ema(self, directory):
        """EMAModel.from_pretrained + load_state_dict: the EMA weights and step count written by save_ema (or by
        diffusers' EMAModel.save_pretrained) into the EMA buffer."""
        self._need_ema()
        step, flat = self._read_ema(directory)
        self.ema.copy_(flat)
        self.ema_steps = step

    def _read_ema(self, directory):
        import json
        import os
        from .checkpoint import CONFIG_NAME
        with open(os.path.join(directory, CONFIG_NAME)) as f:
            step = int(json.load(f).get("optimization_step", 0))
        return step, self._flat_from(self._load_checked(directory, "EMA weight"))

    def _load_checked(self, directory, what):
        """The weights of a diffusers folder, checked against the trainer's parameter names and shapes."""
        from .checkpoint import load_weights
        sd = load_weights(directory)
        for name, _, shape in self._layout:
            if name not in sd or tuple(sd[name].shape) != shape:
                raise ValueError(f"{directory}: no {what} {name} of shape {list(shape)}")
        return sd

    def _flat_from(self, per_param):
        """A host flat buffer in the trainer's layout from {name: tensor} (padding zero)."""
        flat = torch.zeros(self.flat_param.numel(), dtype=torch.float32)
        for name, off, shape in self._layout:
            flat[off:off + math.prod(shape)].copy_(per_param[name].reshape(-1))
        return flat

    # ---- save / resume of the whole training state (accelerator.save_state / load_state, train.py:416-438,578-598,
    # train_depth_normal.py:376-404,540-563,811-831)
    def _torch_order(self):
        """(group, diffusers name) per torch parameter index: group order, then named_parameters order."""
        return [(k, n) for k, g in enumerate(self._group_def) for n in g["params"]]

    def _check_boundary(self, what):
        if self._micro % self.accumulation_steps != 0 or self._handles:
            raise RuntimeError(f"FlatTrainer.{what} inside an accumulation window ({self._micro % self.accumulation_steps} "
                               f"of {self.accumulation_steps} micro-steps): call it after the step")

    def _torch_param_groups(self):
        """torch.optim.AdamW param_groups as the reference's optimizer holds them after `step_count` scheduler steps:
        torch's own defaults for this version, plus lr / initial_lr / betas / eps / weight_decay and the indices."""
        template = torch.optim.AdamW([torch.zeros(1)], lr=1.0, betas=ADAM_BETAS, eps=ADAM_EPS,
                                     weight_decay=0.0).state_dict()["param_groups"][0]
        lrs, out, idx = self.get_last_lr(), [], 0
        for k, g in enumerate(self._group_def):
            d = dict(template)
            d.update(lr=lrs[k], initial_lr=self.lr * g["lr_mult"], betas=ADAM_BETAS, eps=ADAM_EPS,
                     weight_decay=g["weight_decay"], params=list(range(idx, idx + len(g["params"]))))
            idx += len(g["params"])
            out.append(d)
        return out

    def _scheduler_state_dict(self):
        """LambdaLR.state_dict() of the reference's scheduler after step_count optimizer steps (last_epoch = k * N),
        produced by torch's own LambdaLR so the layout is this torch version's."""
        lam = self.lr_schedule if self.lr_schedule is not None else ConstantLR()
        base = [self.lr * g["lr_mult"] for g in self._group_def]
        dummy = torch.optim.AdamW([dict(params=[torch.zeros(1)], lr=b) for b in base])
        sched = torch.optim.lr_scheduler.LambdaLR(dummy, [lam] * len(base))
        sched.last_epoch = self.step_count * self.num_processes
        sched._step_count = sched.last_epoch + 1
        sched._last_lr = self.get_last_lr()
        sd = sched.state_dict()
        if isinstance(lam, ConstantLR):
            sd["lr_lambdas"] = [None] * len(base)      # diffusers' constant schedule is a plain lambda: torch stores None
        return sd

    def save_state(self, output_dir):
        """accelerator.save_state(output_dir) of the recipes: rank 0 writes unet/ (save_pretrained), unet_ema/ (with
        use_ema), optimizer.bin (torch.optim.AdamW.state_dict() layout), scheduler.bin (LambdaLR.state_dict() layout)
        and flat_trainer.pt (the device state block: loss scale, growth tracker, applied / skipped counts; step and
        EMA counts, world size, the group definition); every rank writes random_states_{rank}.pkl (python, numpy,
        torch CPU and CUDA generator states).  Only at an accumulation-window boundary.  The device buffers go to the
        host one at a time; no extra device copy is made.  Ends with a barrier when torch.distributed is up."""
        import os
        import random
        import numpy as np
        import torch.distributed as dist
        self._check_boundary("save_state")
        distributed = dist.is_available() and dist.is_initialized()
        rank = dist.get_rank() if distributed else 0
        os.makedirs(output_dir, exist_ok=True)
        if rank == 0:
            self.module.save_pretrained(os.path.join(output_dir, "unet"))
            if self.ema is not None:
                self.save_ema(os.path.join(output_dir, "unet_ema"))
            state_host = self.state.to("cpu", copy=True)
            applied = int(state_host[2])
            opt = dict(state={}, param_groups=self._torch_param_groups())
            if applied > 0:                   # torch keeps no per-parameter state before a parameter's first update
                where = {name: (off, shape) for name, off, shape in self._layout}
                m = self.exp_avg.to("cpu", copy=True)
                v = self.exp_avg_sq.to("cpu", copy=True)
                for i, (_, name) in enumerate(self._torch_order()):
                    off, shape = where[name]
                    n = math.prod(shape)
                    opt["state"][i] = dict(step=torch.tensor(float(applied)), exp_avg=m[off:off + n].view(shape),
                                           exp_avg_sq=v[off:off + n].view(shape))
                del m, v
            torch.save(opt, os.path.join(output_dir, "optimizer.bin"))
            del opt
            torch.save(self._scheduler_state_dict(), os.path.join(output_dir, "scheduler.bin"))
            torch.save(dict(state=state_host, step_count=self.step_count, ema_steps=self.ema_steps, world=self.world,
                            num_processes=self.num_processes, groups=self._group_def),
                       os.path.join(output_dir, "flat_trainer.pt"))
        rng = dict(random_state=random.getstate(), numpy_random_seed=np.random.get_state(),
                   torch_manual_seed=torch.get_rng_state())
        if torch.cuda.is_available():
            rng["torch_cuda_manual_seed"] = torch.cuda.get_rng_state_all()
        torch.save(rng, os.path.join(output_dir, f"random_states_{rank}.pkl"))
        if distributed:
            dist.barrier()

    def load_state(self, input_dir):
        """accelerator.load_state(input_dir): restores the weights, Adam moments, device state block, step / schedule
        position, the EMA (with use_ema) and this rank's RNG states, bumps the weights epoch (packed fp16 weights and
        CUDA graphs are rebuilt) and returns the checkpoint's global step (optimizer steps taken).  A folder the
        reference wrote (no flat_trainer.pt) loads with the trainer's initial loss scale and applied steps = the
        optimizer's `step`.  Everything is read and checked first: mismatched parameter names or shapes, another
        group definition, or per-parameter `step` values that differ raise ValueError before any buffer changes.
        random_states_{rank}.pkl holds numpy's state and is unpickled in full: load only checkpoints you trust."""
        import os
        import random
        import numpy as np
        import torch.distributed as dist
        from .modules import bump_weights_epoch
        self._check_boundary("load_state")
        path = lambda f: os.path.join(input_dir, f)                               # noqa: E731
        ft = torch.load(path("flat_trainer.pt"), map_location="cpu") if os.path.exists(path("flat_trainer.pt")) else None
        if ft is not None and ft["groups"] != self._group_def:
            raise ValueError(f"{input_dir}: saved with parameter groups "
                             f"{[(g['name'], g['lr_mult'], g['weight_decay'], len(g['params'])) for g in ft['groups']]}, "
                             f"this trainer has {[(g['name'], g['lr_mult'], g['weight_decay'], len(g['params'])) for g in self._group_def]}")
        weights = self._load_checked(path("unet"), "parameter")
        opt = torch.load(path("optimizer.bin"), map_location="cpu")
        pg = opt["param_groups"]
        if [len(g["params"]) for g in pg] != [len(g["params"]) for g in self._group_def] or \
                [float(g["weight_decay"]) for g in pg] != [g["weight_decay"] for g in self._group_def]:
            raise ValueError(f"{input_dir}: the optimizer's parameter groups (sizes "
                             f"{[len(g['params']) for g in pg]}) differ from this trainer's "
                             f"({[len(g['params']) for g in self._group_def]})")
        order = self._torch_order()
        index_of = [i for g in pg for i in g["params"]]
        shapes = {name: shape for name, _, shape in self._layout}
        steps, moments = set(), ({}, {})
        for pos, i in enumerate(index_of):
            st = opt["state"].get(i)
            name = order[pos][1]
            steps.add(float(st["step"]) if st is not None else 0.0)
            if st is not None:
                for d, key in zip(moments, ("exp_avg", "exp_avg_sq")):
                    if tuple(st[key].shape) != shapes[name]:
                        raise ValueError(f"{input_dir}: optimizer state of {name} has shape {list(st[key].shape)}, "
                                         f"the parameter {list(shapes[name])}")
                    d[name] = st[key]
        if len(steps) > 1:
            raise ValueError(f"{input_dir}: per-parameter AdamW steps {sorted(steps)} differ; the fused optimizer keeps "
                             "one step count (one bias correction) for all parameters")
        applied = int(steps.pop()) if steps else 0
        sched = torch.load(path("scheduler.bin"), map_location="cpu") if os.path.exists(path("scheduler.bin")) else None
        if ft is not None:
            step_count, state = int(ft["step_count"]), ft["state"].float()
        else:
            step_count = int(sched["last_epoch"]) // self.num_processes if sched is not None else applied
            state = torch.tensor([self._init_loss_scale, 0, applied, 0, 0, 0, 0, 0], dtype=torch.float32)
        ema = self._read_ema(path("unet_ema")) if self.ema is not None else None
        rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
        rng_file = path(f"random_states_{rank}.pkl")
        rng = torch.load(rng_file, weights_only=False) if os.path.exists(rng_file) else None
        # everything checked: write
        with torch.no_grad():
            self.flat_param.copy_(self._flat_from(weights))
            del weights
            for buf, d in zip((self.exp_avg, self.exp_avg_sq), moments):
                buf.copy_(self._flat_from(d) if d else torch.zeros(buf.numel()))
            self.state.copy_(state)
            if ema is not None:
                self.ema.copy_(ema[1])
                self.ema_steps = ema[0]
            self.flat_grad.zero_()
        self.step_count, self._micro, self._synced = step_count, 0, True
        if rng is not None:
            random.setstate(rng["random_state"])
            np.random.set_state(rng["numpy_random_seed"])
            torch.set_rng_state(rng["torch_manual_seed"])
            if "torch_cuda_manual_seed" in rng and torch.cuda.is_available():
                torch.cuda.set_rng_state_all(rng["torch_cuda_manual_seed"])
        bump_weights_epoch()
        return step_count

    # ---- host read-backs (each one is a device sync: for logging / tests, not for the training loop)
    def loss_scale(self):
        return float(self.state[0])

    def applied_steps(self):
        return int(self.state[2])

    def skipped_steps(self):
        return int(self.state[3])
