"""TEST INFRASTRUCTURE ONLY: the diffusion-objective training math of the reference, restated in plain torch / numpy
on top of the single-step oracle in `oracle/pipeline.py` (encode / decode / class embedding), which it leaves unchanged.

* `add_noise` / `get_velocity`: diffusers (0.30.2) DDPMScheduler.add_noise / get_velocity, written the way diffusers
  writes them (`alphas_cumprod[t] ** 0.5`, `(1 - alphas_cumprod[t]) ** 0.5`, one product and one sum per element);
* `latent_mask`: GeoWizard/geowizard/training/train_depth_normal.py:607-609;
* `geowizard_diffusion_loss`: the same script's :600-717 without `--e2e_ft` (the script's default);
* `EMARef`: diffusers EMAModel with the recipe's defaults (:351-353), in numpy float32 with the same operation order.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import pipeline as OP


def _bcast(v, like):
    v = v.flatten()
    while v.dim() < like.dim():
        v = v.unsqueeze(-1)
    return v


def add_noise(alphas_cumprod, x0, noise, t):
    ac = alphas_cumprod.to(device=x0.device, dtype=x0.dtype)
    t = t.to(x0.device)
    sa = _bcast(ac[t] ** 0.5, x0)
    sb = _bcast((1 - ac[t]) ** 0.5, x0)
    return sa * x0 + sb * noise


def get_velocity(alphas_cumprod, x0, noise, t):
    ac = alphas_cumprod.to(device=x0.device, dtype=x0.dtype)
    t = t.to(x0.device)
    sa = _bcast(ac[t] ** 0.5, x0)
    sb = _bcast((1 - ac[t]) ** 0.5, x0)
    return sa * noise - sb * x0


def latent_mask(val_mask, channels=4):
    """~max_pool2d(~val_mask, 8, 8) repeated over the two halves and the channels -> [2B, C, H//8, W//8] bool."""
    invalid = ~val_mask
    lm = ~torch.max_pool2d(invalid.float(), 8, 8).bool()
    return lm.repeat((2, channels, 1, 1))


def masked_mse(pred, target, lm):
    return F.mse_loss(pred[lm].float(), target[lm].float(), reduction="mean")


def geowizard_diffusion_loss(unet, vae, rgb, depth, normals, val_mask, img_embed, timesteps, noise, alphas_cumprod,
                             prediction_type="v_prediction", domain="indoor"):
    """-> (loss, noise_pred, target).  `noise` None = zeros; timesteps [2B]; normals as the dataset gives them."""
    B = rgb.shape[0]
    with torch.no_grad():
        lat = OP.encode_rgb(vae, torch.cat((rgb, depth, -normals), dim=0))
    rgb_lat, geo = lat[:B], lat[B:]
    noise = torch.zeros_like(geo) if noise is None else noise
    noisy = add_noise(alphas_cumprod, geo, noise, timesteps)
    if prediction_type == "epsilon":
        target = noise
    elif prediction_type == "v_prediction":
        target = get_velocity(alphas_cumprod, geo, noise, timesteps)
    else:
        raise ValueError(prediction_type)
    cls = OP.geowizard_class_embedding(domain, rgb.dtype, B)
    pred = unet(torch.cat((rgb_lat.repeat(2, 1, 1, 1), noisy), 1), timesteps, encoder_hidden_states=img_embed.repeat(2, 1, 1),
                class_labels=cls).sample
    lm = latent_mask(val_mask, geo.shape[1])
    loss = masked_mse(pred, target, lm) if lm.any() else torch.tensor(0.0, requires_grad=True)
    return loss, pred, target


class EMARef:
    """diffusers EMAModel(decay=0.9999, min_decay=0, update_after_step=0, use_ema_warmup=False) over a list of float32
    numpy arrays: step() advances optimization_step, then shadow -= (1 - decay) * (shadow - param)."""

    def __init__(self, params, decay=0.9999):
        self.shadow = [np.array(p, dtype=np.float32, copy=True) for p in params]
        self.decay = decay
        self.optimization_step = 0

    def get_decay(self, optimization_step):
        step = max(0, optimization_step - 0 - 1)
        if step <= 0:
            return 0.0
        cur = (1 + step) / (10 + step)
        return max(min(cur, self.decay), 0.0)

    def step(self, params):
        self.optimization_step += 1
        omd = np.float32(1 - self.get_decay(self.optimization_step))
        for s, p in zip(self.shadow, params):
            s -= omd * (s - np.asarray(p, dtype=np.float32))
