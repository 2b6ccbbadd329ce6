"""TEST INFRASTRUCTURE ONLY: the multi-step DDIM oracle.  A plain-torch restatement of diffusers' (0.30.2)
DDIMScheduler (`set_timesteps` with trailing / leading / linspace spacing, `steps_offset`, `set_alpha_to_one`, and
`step()` with eta = 0) and of the reference's full denoising loops, built on the single-step oracle in
`oracle/pipeline.py` (encode / decode / class embedding), which it leaves unchanged:

* `marigold_infer`:  Marigold/marigold/marigold_pipeline.py:371-478 with any number of steps;
* `geowizard_infer`: GeoWizard/geowizard/models/geowizard_pipeline.py:251-344 with any number of steps.

The initial latent is an explicit argument (`init_latent`, None = zeros) so a test hands the oracle exactly the noise
the engine drew.  At one step with zeros both reduce to `oracle.pipeline.marigold_single_infer` /
`geowizard_single_infer` (checked against the golden fixtures in tests/test_multistep_cpu.py)."""
import numpy as np
import torch

from oracle import pipeline as OP


class DDIMRef:
    """diffusers.DDIMScheduler, scaled-linear betas, eta = 0, no clipping / thresholding."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, prediction_type="v_prediction",
                 timestep_spacing="trailing", steps_offset=1, set_alpha_to_one=True):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.prediction_type = prediction_type
        self.timestep_spacing = timestep_spacing
        self.steps_offset = steps_offset
        self.num_inference_steps = None
        self.timesteps = None

    def set_timesteps(self, n, device=None):
        T = self.num_train_timesteps
        self.num_inference_steps = n
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.int64)
            ts += self.steps_offset
        elif self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64)
            ts -= 1
        else:
            raise ValueError(self.timestep_spacing)
        self.timesteps = torch.from_numpy(ts).to(device)

    def prev_timestep(self, t):
        return int(t) - self.num_train_timesteps // self.num_inference_steps

    def step(self, model_output, timestep, sample):
        """-> (prev_sample, pred_original_sample), fp32 0-d coefficients as in diffusers."""
        t = int(timestep)
        prev = self.prev_timestep(t)
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        a_t, a_prev = a_t.to(sample.device), a_prev.to(sample.device)
        beta = 1 - a_t
        if self.prediction_type == "epsilon":
            x0 = (sample - beta ** 0.5 * model_output) / a_t ** 0.5
            eps = model_output
        elif self.prediction_type == "sample":
            x0 = model_output
            eps = (sample - a_t ** 0.5 * x0) / beta ** 0.5
        elif self.prediction_type == "v_prediction":
            x0 = a_t ** 0.5 * sample - beta ** 0.5 * model_output
            eps = a_t ** 0.5 * model_output + beta ** 0.5 * sample
        else:
            raise ValueError(self.prediction_type)
        return a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * eps, x0


@torch.no_grad()
def marigold_infer(unet, vae, scheduler, rgb_in, empty_text_embed, num_inference_steps=1, init_latent=None,
                   normals=False):
    scheduler.set_timesteps(num_inference_steps, device=rgb_in.device)
    rgb_latent = OP.encode_rgb(vae, rgb_in)
    latent = torch.zeros_like(rgb_latent) if init_latent is None else init_latent.to(rgb_latent)
    ctx = empty_text_embed.repeat(rgb_latent.shape[0], 1, 1)
    for i, t in enumerate(scheduler.timesteps):
        pred = unet(torch.cat([rgb_latent, latent], dim=1), t, encoder_hidden_states=ctx).sample
        prev, x0 = scheduler.step(pred, t, latent)
        latent = x0 if i == num_inference_steps - 1 else prev
    dec = OP.decode_latent(vae, latent)
    if normals:
        return dec / (torch.norm(dec, p=2, dim=1, keepdim=True) + 1e-5)
    return (torch.clip(dec.mean(dim=1, keepdim=True), -1.0, 1.0) + 1.0) / 2.0


@torch.no_grad()
def geowizard_infer(unet, vae, scheduler, rgb_in, img_embed, domain="indoor", num_inference_steps=1,
                    init_latent=None):
    """Batched ([depth x B, normal x B]) loop; `init_latent` is the [B] draw that the reference `.repeat(2)`s."""
    B = rgb_in.shape[0]
    scheduler.set_timesteps(num_inference_steps, device=rgb_in.device)
    rgb_latent = OP.encode_rgb(vae, rgb_in)
    geo = torch.zeros_like(rgb_latent) if init_latent is None else init_latent.to(rgb_latent)
    geo = geo.repeat(2, 1, 1, 1)
    rgb_latent = rgb_latent.repeat(2, 1, 1, 1)
    ctx = img_embed.repeat(2, 1, 1) if img_embed.shape[0] == B else img_embed.repeat(2 * B, 1, 1)
    cls = OP.geowizard_class_embedding(domain, rgb_in.dtype, B).to(rgb_in.device)
    for i, t in enumerate(scheduler.timesteps):
        pred = unet(torch.cat([rgb_latent, geo], 1), t.repeat(2 * B), encoder_hidden_states=ctx,
                    class_labels=cls).sample
        prev, x0 = scheduler.step(pred, t, geo)
        geo = x0 if i == num_inference_steps - 1 else prev
    depth = OP.decode_latent(vae, geo[:B]).mean(dim=1, keepdim=True)
    depth = (torch.clip(depth, -1.0, 1.0) + 1.0) / 2.0
    normal = OP.decode_latent(vae, geo[B:])
    normal = normal / (torch.norm(normal, p=2, dim=1, keepdim=True) + 1e-5)
    return depth, -normal
