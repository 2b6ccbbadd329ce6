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


@torch.no_grad()
def e2e_ft_forward(unet, vae, scheduler, rgb, ground_truth, val_mask, empty_encoding, modality="depth"):
    """Returns (loss [0-d fp32 tensor], current_estimate).  rgb [B,3,H,W] in [-1,1]; ground_truth [B,1,H,W]
    metric depth or [B,3,H,W] normals; val_mask [B,1,H,W] bool; empty_encoding [1,77,1024]."""
    B = rgb.shape[0]
    rgb_latents = vae.encode_scaled_mean(rgb)                                   # train.py:473-474
    T = scheduler.config["num_train_timesteps"]
    t = T - 1                                                                   # :480-481
    noisy = torch.zeros_like(rgb_latents)                                       # :484-485 (noise_type zeros)
    ctx = empty_encoding.to(rgb.device).repeat(B, 1, 1)
    model_pred = unet(torch.cat((rgb_latents, noisy), dim=1), t, ctx, return_dict=False)[0]     # :494-500
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = vae.decode_from_prediction(model_pred, -math.sqrt(1.0 - a_t))         # :509-529 (x_t = 0)
    est = ops.decode_post(dec.float().contiguous(), normals=(modality == "normals"), training=True)   # :532-540
    if modality == "depth":
        loss = ops.ssi_loss(est, ground_truth, val_mask)                        # :545
    elif modality == "normals":
        loss = ops.angular_loss(est, ground_truth, val_mask)                    # :549
    else:
        raise ValueError(f"Unknown modality {modality}")
    return loss, est


LOSS_SCALE = 1024.0       # static loss scale: incoming gradients are fp16 GEMM operands in the backward pass


def e2e_ft_loss(unet, vae, scheduler, rgb, ground_truth, val_mask, empty_encoding, modality="depth"):
    """Differentiable training micro-step (training/train.py:469-556).  Returns (loss, estimate); call
    `(loss * LOSS_SCALE).backward()` and divide the gradients by LOSS_SCALE (or pass `grad_unscale` to the
    optimizer step).  VAE encode runs without grad (frozen, train.py:473 under no_grad)."""
    from . import autograd_blocks as ab
    B = rgb.shape[0]
    with torch.no_grad():
        rgb_latents = vae.encode_scaled_mean(rgb)
    T = scheduler.config["num_train_timesteps"]
    t = T - 1
    ctx = empty_encoding.to(rgb.device).repeat(B, 1, 1)
    model_pred = unet(torch.cat((rgb_latents, torch.zeros_like(rgb_latents)), dim=1), t, ctx, return_dict=False)[0]
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = vae.decode_from_prediction(model_pred, -math.sqrt(1.0 - a_t))
    normals = modality == "normals"
    if modality not in ("depth", "normals"):
        raise ValueError(f"Unknown modality {modality}")
    est = ab.decode_post(dec, normals)
    return ab.task_loss(est, ground_truth, val_mask, normals), est


def e2e_ft_loss_geowizard(unet, vae, scheduler, rgb, depth_gt, normal_gt, val_mask, img_embed, domain="indoor",
                          depth_scale=0.5, normal_scale=1.0):
    """Differentiable joint depth + normal micro-step of the GeoWizard recipe
    (GeoWizard/geowizard/training/train_depth_normal.py:640-766, `--e2e_ft`, zeros noise): one UNet call on the
    [depth x B | normal x B] batch with the hybrid class embedding and joint self-attention, x0 by the v-prediction closed
    form, ONE decoder pass over both halves, depth = clamp(mean_c), normals = clamp(x / (|x| + 1e-5)),
    loss = depth_scale * SSI(depth) + normal_scale * angular(normals, -normal_gt)   (the reference trains on inverted
    normals, :742).  rgb [B,3,H,W], depth_gt [B,1,H,W], normal_gt [B,3,H,W], val_mask [B,1,H,W] bool, img_embed
    [B,1,768] (CLIP image embedding).  Returns (loss, depth_estimate, normal_estimate)."""
    from . import autograd_blocks as ab
    from .pipelines import DepthNormalEstimationPipeline
    B = rgb.shape[0]
    dev = rgb.device
    with torch.no_grad():
        rgb_latents = vae.encode_scaled_mean(rgb)
    T = scheduler.config["num_train_timesteps"]
    t = T - 1                                                                             # :646-648
    timesteps = torch.full((2 * B,), t, device=dev, dtype=torch.long)
    x = torch.cat((rgb_latents.repeat(2, 1, 1, 1), torch.zeros_like(rgb_latents).repeat(2, 1, 1, 1)), dim=1)   # :705
    ctx = img_embed.to(dev).repeat(2, 1, 1)                                               # :683
    cls = DepthNormalEstimationPipeline.class_embedding(domain, B, dev, rgb_latents.dtype)                   # :686-703
    pred = unet(x, timesteps, ctx, class_labels=cls, return_dict=False)[0]
    a_t = float(scheduler.alphas_cumprod[t])
    assert scheduler.config["prediction_type"] == "v_prediction"
    dec = vae.decode_from_prediction(pred, -math.sqrt(1.0 - a_t))                         # :722-737, one decoder pass
    est_d = ab.decode_post(dec[:B].contiguous(), False)                                   # :739-741
    est_n = ab.decode_post(dec[B:].contiguous(), True)                                    # :743-746
    loss_d = ab.task_loss(est_d, depth_gt, val_mask, False)
    loss_n = ab.task_loss(est_n, -normal_gt, val_mask, True)
    return depth_scale * loss_d + normal_scale * loss_n, est_d, est_n


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
                 loss_scale=LOSS_SCALE, bucket_mb=256, dynamic_loss_scale=True, growth_interval=2000, overlap=False):
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
        with torch.no_grad():
            for idx, (p, n) in enumerate(zip(ps, sizes)):
                if p.dtype != torch.float32:
                    raise TypeError("FlatTrainer expects fp32 master parameters")
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
        return nsq

    # ---- host read-backs (each one is a device sync: for logging / tests, not for the training loop)
    def loss_scale(self):
        return float(self.state[0])

    def applied_steps(self):
        return int(self.state[2])

    def skipped_steps(self):
        return int(self.state[3])
