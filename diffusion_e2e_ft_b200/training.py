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
    train.py:503,546-551) — all without a host sync.  `skipped_steps()` / `loss_scale()` read the state back."""

    LATE_GRAD_KEYS = ("time_emb_proj", "time_embedding", "class_embedding")

    def __init__(self, module, lr=3e-5, weight_decay=1e-2, max_grad_norm=1.0, accumulation_steps=1, group=None,
                 loss_scale=LOSS_SCALE, bucket_mb=256, dynamic_loss_scale=True, growth_interval=2000, overlap=False,
                 use_ema=False):
        import torch.distributed as dist
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if not named:
            raise ValueError("no trainable parameters")
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

    def micro_step(self, loss, lr=None):
        """backward(); on the last micro-step of the accumulation window also step().  Returns True when it stepped
        (`accelerator.sync_gradients` of train.py:563-570)."""
        self.backward(loss)
        if self._micro % self.accumulation_steps == 0:
            self.step(lr)
            return True
        return False

    def step(self, lr=None):
        if self._micro % self.accumulation_steps != 0 or not self._synced:
            raise RuntimeError(f"FlatTrainer.step inside an accumulation window ({self._micro % self.accumulation_steps} of "
                               f"{self.accumulation_steps} micro-steps) or after backward(sync=False): gradients are not reduced")
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
        ops.adamw_step_state(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, self.state, nsq,
                             lr=self.lr if lr is None else lr, weight_decay=self.weight_decay,
                             max_grad_norm=self.max_grad_norm, inv_world=1.0 / self.world,
                             dynamic_scale=self.dynamic_loss_scale, growth_interval=self.growth_interval)
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
        import json
        import os
        from .checkpoint import CONFIG_NAME, load_weights
        self._need_ema()
        with open(os.path.join(directory, CONFIG_NAME)) as f:
            step = int(json.load(f).get("optimization_step", 0))
        sd = load_weights(directory)
        with torch.no_grad():
            for name, off, shape in self._layout:
                if name not in sd or tuple(sd[name].shape) != shape:
                    raise ValueError(f"{directory}: no EMA weight {name} of shape {list(shape)}")
                n = sd[name].numel()
                self.ema[off:off + n].copy_(sd[name].reshape(-1))
        self.ema_steps = step

    # ---- host read-backs (each one is a device sync: for logging / tests, not for the training loop)
    def loss_scale(self):
        return float(self.state[0])

    def applied_steps(self):
        return int(self.state[2])

    def skipped_steps(self):
        return int(self.state[3])
