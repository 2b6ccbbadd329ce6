"""Diffusers-free restatement of the reference's host pipelines on top of the engine modules.

`diffusers` (DiffusionPipeline, BaseOutput, DDIMScheduler) and `matplotlib` are not importable in
this image, so the reference pipeline files cannot even be imported; these classes keep their
public surface — `__call__`, `single_infer`, `encode_rgb`, `decode_depth`, `decode_normal`, the
output dataclasses — and route the arithmetic through B200UNet2DConditionModel / B200AutoencoderKL.

  MarigoldPipeline                 <- Marigold/marigold/marigold_pipeline.py:113-538
  DepthNormalEstimationPipeline    <- GeoWizard/geowizard/models/geowizard_pipeline.py:67-401
  DDIMScheduler (eta = 0, step on the b200_ddim_step kernel) <- diffusers DDIMScheduler as used at
                                   marigold_pipeline.py:401-402,457-465 and geowizard_pipeline.py:261,326-334
"""
import json
import math
import os
from dataclasses import dataclass
from typing import Optional, Union

import numpy as np
import torch

from . import ops


# ------------------------------------------------------------------------------------ scheduler
class SchedulerOutput:
    def __init__(self, prev_sample, pred_original_sample):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class DDIMScheduler:
    """diffusers' (0.30.2) DDIMScheduler as the reference uses it: `from_pretrained`, `set_timesteps` (trailing,
    leading, linspace), `timesteps`, `step(...).prev_sample / .pred_original_sample`, `alphas_cumprod`,
    `final_alpha_cumprod`, `config`.  Scaled-linear betas, eta = 0, no clipping / thresholding (the SD-2 and
    Marigold / GeoWizard configs); `from_pretrained` rejects a config that needs anything else."""

    # diffusers' constructor defaults: a key missing from scheduler_config.json takes these
    _DIFFUSERS_DEFAULTS = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                               trained_betas=None, clip_sample=True, set_alpha_to_one=True, steps_offset=0,
                               prediction_type="epsilon", thresholding=False, dynamic_thresholding_ratio=0.995,
                               clip_sample_range=1.0, sample_max_value=1.0, timestep_spacing="leading",
                               rescale_betas_zero_snr=False)
    _SPACINGS = ("trailing", "leading", "linspace")

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                 prediction_type="v_prediction", timestep_spacing="trailing", steps_offset=1, set_alpha_to_one=True):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        # the alpha of the step after the last one (diffusers: 1 with set_alpha_to_one, else alphas_cumprod[0])
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.config = dict(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           beta_schedule="scaled_linear", prediction_type=prediction_type,
                           timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                           set_alpha_to_one=set_alpha_to_one)
        self.num_inference_steps = None
        self.timesteps = None
        self._ac = [float(a) for a in self.alphas_cumprod]       # host copy: no device sync in step()
        self._final_ac = float(self.final_alpha_cumprod)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kwargs):
        """Read a diffusers `scheduler_config.json` (e.g. `from_pretrained(ckpt, subfolder="scheduler",
        timestep_spacing="trailing")`, Marigold/run.py:273, GeoWizard/run_infer.py:194-197).  Keyword arguments
        override the file.  A config whose math the engine does not implement raises ValueError naming the key."""
        d = pretrained_model_name_or_path if subfolder is None else os.path.join(pretrained_model_name_or_path, subfolder)
        with open(os.path.join(d, "scheduler_config.json")) as f:
            cfg = json.load(f)
        cfg.update(kwargs)
        return cls.from_config(cfg)

    @classmethod
    def from_config(cls, config):
        """Keys that are not DDIMScheduler arguments change no DDIM math and are kept, as diffusers ignores them (e.g.
        `skip_prk_steps` of the SD-2 scheduler configs, a PNDM key): they land in `config["_extra"]`."""
        cfg = dict(cls._DIFFUSERS_DEFAULTS)
        cfg.update({k: v for k, v in config.items() if k in cls._DIFFUSERS_DEFAULTS})
        extra = {k: v for k, v in config.items() if k not in cls._DIFFUSERS_DEFAULTS and k != "_class_name"}
        if cfg["beta_schedule"] != "scaled_linear":
            raise ValueError(f"beta_schedule={cfg['beta_schedule']!r}: the engine implements 'scaled_linear' only")
        if cfg["trained_betas"] is not None:
            raise ValueError("trained_betas: the engine implements the 'scaled_linear' schedule only")
        for k in ("clip_sample", "thresholding", "rescale_betas_zero_snr"):
            if cfg[k]:
                raise ValueError(f"{k}=True is not supported by the engine (DDIM with eta = 0 and no clipping only)")
        if cfg["prediction_type"] not in ops.PREDICTION_TYPES:
            raise ValueError(f"prediction_type={cfg['prediction_type']!r} is not one of {sorted(ops.PREDICTION_TYPES)}")
        if cfg["timestep_spacing"] not in cls._SPACINGS:
            raise ValueError(f"timestep_spacing={cfg['timestep_spacing']!r} is not one of {list(cls._SPACINGS)}")
        sched = cls(num_train_timesteps=int(cfg["num_train_timesteps"]), beta_start=float(cfg["beta_start"]),
                    beta_end=float(cfg["beta_end"]), prediction_type=cfg["prediction_type"],
                    timestep_spacing=cfg["timestep_spacing"], steps_offset=int(cfg["steps_offset"]),
                    set_alpha_to_one=bool(cfg["set_alpha_to_one"]))
        if extra:
            sched.config["_extra"] = extra
        return sched

    def set_timesteps(self, num_inference_steps, device=None):
        T = self.config["num_train_timesteps"]
        if not 1 <= num_inference_steps <= T:
            raise ValueError(f"num_inference_steps={num_inference_steps} must be in [1, num_train_timesteps={T}]")
        self.num_inference_steps = num_inference_steps
        if self.config["timestep_spacing"] == "trailing":
            ts = np.round(np.arange(T, 0, -T / num_inference_steps)) - 1
        elif self.config["timestep_spacing"] == "leading":
            ts = (np.arange(0, num_inference_steps) * (T // num_inference_steps)).round()[::-1].copy()
            ts = ts + self.config["steps_offset"]
        elif self.config["timestep_spacing"] == "linspace":
            ts = np.linspace(0, T - 1, num_inference_steps).round()[::-1].copy()
        else:
            raise ValueError(self.config["timestep_spacing"])
        self._host_timesteps = [int(t) for t in ts]
        self.timesteps = torch.tensor(self._host_timesteps, dtype=torch.long, device=device)

    def prev_timestep(self, timestep):
        """diffusers' `t - T // num_inference_steps` (so e.g. 3-step trailing 999 -> 666 -> 332 steps 666 to 333)."""
        return int(timestep) - self.config["num_train_timesteps"] // self.num_inference_steps

    def coefficients(self, t_index):
        """(t, t_prev, a_t, a_prev) for the i-th inference step, all host floats/ints."""
        t = self._host_timesteps[t_index]
        prev = self.prev_timestep(t)
        a_t = self._ac[t]
        a_prev = self._ac[prev] if prev >= 0 else self._final_ac
        return t, prev, a_t, a_prev

    def step(self, model_output, timestep, sample, eta=0.0, return_dict=True):
        """One DDIM update on the `b200_ddim_step` kernel -> SchedulerOutput(prev_sample, pred_original_sample), both
        fp32 (the engine keeps the DDIM state in fp32 whatever the model dtype).  `timestep` is an int or a 0-d tensor
        (a device tensor costs one host sync)."""
        if eta != 0.0:
            raise NotImplementedError("DDIMScheduler.step: eta != 0 (stochastic DDIM) is not implemented")
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps before step")
        t = int(timestep)
        T = self.config["num_train_timesteps"]
        if not 0 <= t < T:
            raise ValueError(f"timestep {t} is outside [0, num_train_timesteps={T})")
        prev = self.prev_timestep(t)
        a_prev = self._ac[prev] if prev >= 0 else self._final_ac
        x = sample if sample.dtype == torch.float32 else sample.float()           # dtype cast at the API boundary
        prev_sample, x0 = ops.ddim_step(model_output, x, self._ac[t], a_prev, self.config["prediction_type"],
                                        want_x0=True)
        if not return_dict:
            return prev_sample, x0
        return SchedulerOutput(prev_sample, x0)


def _x0_coefficients(prediction_type, a_t):
    """x0 = c_x * x_t + c_m * model_out: the scheduler's pred_original_sample as a linear map (fused into
    post_quant_conv on the last step)."""
    sa, sb = math.sqrt(a_t), math.sqrt(1.0 - a_t)
    if prediction_type == "v_prediction":
        return sa, -sb
    if prediction_type == "epsilon":
        return 1.0 / sa, -sb / sa
    if prediction_type == "sample":
        return 0.0, 1.0
    raise ValueError(prediction_type)


# ------------------------------------------------------------------------------------ base
class PipelineBase:
    """Minimal `DiffusionPipeline` surface the reference relies on: register_modules, to, device, dtype."""

    def register_modules(self, **modules):
        self._module_names = list(modules)
        for k, v in modules.items():
            setattr(self, k, v)

    def to(self, *args, **kwargs):
        for k in self._module_names:
            m = getattr(self, k)
            if isinstance(m, torch.nn.Module):
                m.to(*args, **kwargs)
        return self

    @property
    def device(self):
        return next(self.unet.parameters()).device

    # ---- diffusers' memory-efficient attention switch (Marigold/run.py:285), forwarded like DiffusionPipeline does
    def enable_xformers_memory_efficient_attention(self, attention_op=None):
        for k in self._module_names:
            fn = getattr(getattr(self, k), "enable_xformers_memory_efficient_attention", None)
            if fn is not None:
                fn(attention_op)

    def disable_xformers_memory_efficient_attention(self):
        for k in self._module_names:
            fn = getattr(getattr(self, k), "disable_xformers_memory_efficient_attention", None)
            if fn is not None:
                fn()

    @property
    def dtype(self):
        return next(self.unet.parameters()).dtype

    # ---- CUDA-graph replay of a fixed-shape step (launch-bound inner loop: ~1800 kernels / step)
    use_cuda_graph = True

    def _weights_key(self):
        """Identity of every weight a captured graph has baked in: storage pointers + torch version counters of the
        parameters AND the engine's weights epoch (`modules.bump_weights_epoch`: the flat-buffer optimizer kernel
        updates parameters with raw device writes that version counters do not see — without the epoch a validation
        `single_infer` after a training step would replay a graph that points at freed packed-weight buffers)."""
        from .modules import _WEIGHTS_EPOCH
        ps = self.__dict__.get("_wk_params")
        mods = (id(self.unet), id(self.vae), id(getattr(self.unet, "conv_in", None)))
        if ps is None or self.__dict__.get("_wk_mods") != mods:
            ps = list(self.unet.parameters()) + list(self.vae.parameters())
            self.__dict__["_wk_params"], self.__dict__["_wk_mods"] = ps, mods
        return (_WEIGHTS_EPOCH[0], hash(tuple((p.data_ptr(), p._version) for p in ps)))

    def _graphed(self, key, fn, *xs):
        """Capture `fn(*static_xs)` once per (key, weights version) and replay it; returns a fresh tensor.  Every input
        (the image batch, and the initial latent when the call draws noise) is copied into its static buffer first."""
        graphs = self.__dict__.setdefault("_graphs", {})
        wkey = self._weights_key()
        ent = graphs.get(key)
        if ent is None or ent["wkey"] != wkey:
            static_xs = [x.clone() for x in xs]
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for _ in range(2):                         # warm-up: packs weights, sets func attributes
                    fn(*static_xs)
            cur.wait_stream(side)
            torch.cuda.synchronize()
            before = (ops.STATS.launches, dict(ops.STATS.flops), dict(ops.STATS.count))
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = fn(*static_xs)
            delta = dict(launches=ops.STATS.launches - before[0],
                         flops={k: ops.STATS.flops[k] - before[1][k] for k in before[1]},
                         count={k: ops.STATS.count[k] - before[2][k] for k in before[2]})
            ent = dict(g=g, xs=static_xs, out=out, wkey=wkey, delta=delta)
            graphs[key] = ent
        for s, x in zip(ent["xs"], xs):
            s.copy_(x, non_blocking=True)
        ent["g"].replay()
        d = ent["delta"]
        ops.STATS.launches += d["launches"]
        for k in d["flops"]:
            ops.STATS.flops[k] += d["flops"][k]
            ops.STATS.count[k] += d["count"][k]
        return ent["out"].clone()


@dataclass
class MarigoldDepthOutput:
    depth_np: Optional[np.ndarray]
    depth_colored: Optional[object]
    uncertainty: Optional[np.ndarray]
    normal_np: Optional[np.ndarray]
    normal_colored: Optional[object]


from .ensemble import (check_color_map, colorize_depth, colorize_normals, ensemble_depths,  # noqa: E402
                       ensemble_normals, minmax_normalise_, minmax_rows, normalise_rgb, resize_bicubic_aa,
                       resize_bilinear_aa, resize_nearest, resize_nearest_exact)


def pyramid_noise_like(x, discount=0.9, generator=None):
    """Multi-resolution noise of marigold_pipeline.py:76-86 (also training/train.py:486-487): white noise plus
    bilinearly up-sampled coarser noise maps with geometrically decaying weights, renormalised to unit std.  The
    random draws (torch.randn, python `random`) are host-pipeline code as in the reference; they are not part of
    the measured hot path (E2E-FT uses zeros noise)."""
    import random
    b, c, w, h = x.shape
    u = torch.nn.Upsample(size=(w, h), mode="bilinear")
    noise = torch.randn(x.shape, device=x.device, dtype=x.dtype, generator=generator)
    for i in range(10):
        r = random.random() * 2 + 2
        w, h = max(1, int(w / (r ** i))), max(1, int(h / (r ** i)))
        noise += u(torch.randn(b, c, w, h, device=x.device, dtype=x.dtype, generator=generator)) * discount ** i
        if w == 1 or h == 1:
            break
    return noise / noise.std()


NOISE_TYPES = ("gaussian", "pyramid", "zeros")


def _check_noise(noise, num_inference_steps):
    """Argument checks of the denoising loop, raised before anything is launched."""
    if noise not in NOISE_TYPES:
        raise ValueError(f"Unknown noise type: {noise}")
    if int(num_inference_steps) < 1:
        raise ValueError(f"num_inference_steps={num_inference_steps} must be >= 1")


def _check_geowizard_noise(noise, num_inference_steps):
    """GeoWizard's pyramid noise adds `[T,1,1,1]`-shaped timesteps / 1000 in place into a `[B,...]` map: with T > 1 the
    reference raises, except when B == T, where it silently scales each sample of the batch by a different timestep.
    Neither is a defined schedule, so the engine refuses pyramid noise with more than one step."""
    _check_noise(noise, num_inference_steps)
    if noise == "pyramid" and num_inference_steps > 1:
        raise ValueError("GeoWizard's pyramid noise (geowizard_pipeline.py:33-43) scales the noise by timesteps / 1000 "
                         f"with an in-place broadcast that is only defined for one step; with {num_inference_steps} "
                         "steps the reference raises (or, when the batch size equals the step count, scales each sample "
                         "by a different timestep). Use noise='gaussian' or 'zeros', or num_inference_steps=1")


def geowizard_pyramid_noise_like(x, timesteps, discount=0.9):
    """GeoWizard's own multi-resolution noise (geowizard_pipeline.py:33-43): the coarser maps are scaled by
    timesteps / 1000, r is drawn from numpy in [1.5, 3) and the coarse draws come from torch's CPU generator.  Not
    Marigold's `pyramid_noise_like`.  Host-pipeline code; only defined for one timestep (see _check_geowizard_noise)."""
    b, c, w_ori, h_ori = x.shape
    u = torch.nn.Upsample(size=(w_ori, h_ori), mode="bilinear")
    noise = torch.randn_like(x)
    scale = 1.5
    for i in range(10):
        r = np.random.random() * scale + scale
        w, h = max(1, int(w_ori / (r ** i))), max(1, int(h_ori / (r ** i)))
        noise += u(torch.randn(b, c, w, h).to(x)) * (timesteps[..., None, None, None] / 1000) * discount ** i
        if w == 1 or h == 1:
            break
    return noise / noise.std()


def _check_image_size(H, W):
    """The kernels index one image's activations with 32-bit unsigned element offsets; the largest is the VAE
    decoder's 256-channel full-resolution tensor, so one image must stay under 2^32 / 256 pixels (16.7 MP)."""
    if 256 * H * W >= 2 ** 32:
        raise ValueError(f"a {W}x{H} input ({H * W / 1e6:.1f} MP) is over the engine's per-image limit of "
                         f"{(2 ** 32 - 1) // 256 / 1e6:.1f} MP (256 * H * W < 2^32 elements); pass a "
                         f"processing_res > 0 to run at a lower resolution")


def _max_res_size(h, w, max_edge):
    """(height, width) after resize_max_res; processing_res = 0 keeps the input size."""
    if max_edge <= 0:
        return h, w
    s = min(max_edge / w, max_edge / h)
    return int(h * s), int(w * s)


RESAMPLE_METHODS = ("bilinear", "bicubic", "nearest")


def _check_resample_method(method):
    """Marigold/marigold/util/image_util.py:111-120 get_tv_resample_method, raised before anything is launched."""
    if method not in RESAMPLE_METHODS:
        raise ValueError(f"Unknown resampling method: {method!r} (one of {list(RESAMPLE_METHODS)})")


def _resize(x, size, method):
    """torchvision `resize(x, size, method, antialias=True)` of a [..., H, W] fp32 tensor on the device:
    "bilinear" / "bicubic" antialiased, "nearest" = NEAREST_EXACT (antialias does not apply)."""
    if method == "bilinear":
        return resize_bilinear_aa(x, size)
    if method == "bicubic":
        return resize_bicubic_aa(x, size)
    return resize_nearest_exact(x, size)


def _resize_max_res(img, max_edge, method="bilinear"):
    """Marigold/marigold/util/image_util.py:79-108 resize_max_res: down-scale to a maximum edge length with the
    chosen resampling (antialiased bilinear by default), on the device (csrc/postproc.cu)."""
    _, h, w = img.shape
    return _resize(img, _max_res_size(h, w, max_edge), method)


def _to_pil(u8_hwc):
    """uint8 [H, W, 3] device tensor -> PIL image (one device-to-host copy)."""
    from PIL import Image
    return Image.fromarray(u8_hwc.cpu().numpy())


class MarigoldPipeline(PipelineBase):
    rgb_latent_scale_factor = 0.18215
    depth_latent_scale_factor = 0.18215

    def __init__(self, unet, vae, scheduler, text_encoder=None, tokenizer=None, empty_text_embed=None):
        self.register_modules(unet=unet, vae=vae, scheduler=scheduler, text_encoder=text_encoder,
                              tokenizer=tokenizer)
        self.empty_text_embed = empty_text_embed          # [1, 2, 1024]; CLIP weights are not available offline

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: int = 10, ensemble_size: int = 10,
                 processing_res: int = 768, match_input_res: bool = True, resample_method: str = "bilinear",
                 batch_size: int = 0, color_map: Optional[str] = "Spectral", show_progress_bar: bool = True,
                 ensemble_kwargs=None, noise="gaussian", normals=False) -> MarigoldDepthOutput:
        assert processing_res >= 0 and ensemble_size >= 1
        _check_resample_method(resample_method)
        check_color_map(color_map)
        _check_noise(noise, denoising_steps)
        if isinstance(input_image, torch.Tensor):
            rgb = input_image.squeeze()
        else:                                              # PIL.Image
            rgb = torch.from_numpy(np.asarray(input_image.convert("RGB")).copy()).permute(2, 0, 1)
        input_size = rgb.shape
        assert rgb.dim() == 3 and input_size[0] == 3, f"Wrong input shape {input_size}, expected [rgb, H, W]"
        _check_image_size(*_max_res_size(input_size[-2], input_size[-1], processing_res))   # before any launch
        # pre-processing on the device (SURVEY.md §8 f2): the raw (uint8) image is uploaded once; resize + [0,255] ->
        # [-1,1] run as kernels (marigold_pipeline.py:237-247).  torchvision resizes a uint8 tensor as a float resize
        # followed by clamp (bicubic) and round back to uint8: normalise_rgb(round_u8) does both.
        was_u8 = rgb.dtype == torch.uint8
        rgb = rgb.to(self.device)
        rgb = rgb.to(torch.float32)                        # dtype cast at the API boundary
        if processing_res > 0:
            rgb = _resize_max_res(rgb, processing_res, resample_method)
        rgb_norm = normalise_rgb(rgb, round_u8=was_u8 and processing_res > 0)
        lo, hi = minmax_rows(rgb_norm.view(1, -1))[0].tolist()
        assert lo >= -1.0 and hi <= 1.0
        rgb_norm = rgb_norm.to(self.dtype)
        duplicated = torch.stack([rgb_norm] * ensemble_size)
        bs = batch_size if batch_size > 0 else ensemble_size
        preds = []
        for i in range(0, ensemble_size, bs):
            preds.append(self.single_infer(duplicated[i:i + bs], denoising_steps, show_progress_bar,
                                           noise=noise, normals=normals).detach())
        preds = torch.concat(preds, dim=0).squeeze()
        pred_uncert = None
        if ensemble_size > 1:                              # test-time ensembling on the device (:288-294)
            if normals:
                pred, pred_uncert = ensemble_normals(preds)
            else:
                pred, pred_uncert = ensemble_depths(preds, **(ensemble_kwargs or {}))
        else:
            pred = preds
        return self._postprocess(pred, pred_uncert, tuple(input_size[-2:]), normals=normals,
                                 match_input_res=match_input_res, resample_method=resample_method, color_map=color_map)

    def _postprocess(self, pred, pred_uncert, input_hw, normals=False, match_input_res=True,
                     resample_method="bilinear", color_map="Spectral") -> MarigoldDepthOutput:
        """marigold_pipeline.py:298-350 on the device, from the (ensembled) prediction to the output: unit normals or
        [0, 1] depth, resize back with the call's resampling, one copy to the host, clip; the colour image is built
        by a kernel from the same device tensor and copied to the host once as uint8."""
        pred = pred.to(torch.float32).contiguous()
        if normals:
            pred = ops.decode_post(pred[None], normals=True)[0]            # pred / (|pred| + 1e-5)   (:300-303)
        else:
            pred, mm = minmax_normalise_(pred)                             # (pred - min) / (max - min)   (:305-312)
            lo, hi = mm.tolist()
            if hi == lo:
                pred = torch.zeros_like(pred)
        if match_input_res:
            pred = _resize(pred if normals else pred.unsqueeze(0), input_hw, resample_method).squeeze()
        # colours of the clipped map (:327-343): the kernels clip as numpy does, so they read the same device tensor
        if normals:
            colored = _to_pil(colorize_normals(pred))
        else:
            colored = None if color_map is None else _to_pil(colorize_depth(pred, color_map))
        pred = pred.cpu().numpy()
        if pred_uncert is not None:
            pred_uncert = pred_uncert.cpu().numpy() if torch.is_tensor(pred_uncert) else pred_uncert
        pred = pred.clip(-1.0, 1.0) if normals else pred.clip(0, 1)
        return MarigoldDepthOutput(depth_np=None if normals else pred, depth_colored=None if normals else colored,
                                   uncertainty=pred_uncert, normal_np=pred if normals else None,
                                   normal_colored=colored if normals else None)

    def encode_empty_text(self):
        if self.text_encoder is None:
            raise RuntimeError("no text encoder: pass `empty_text_embed` ([1,2,1024]) to MarigoldPipeline")
        ids = self.tokenizer("", padding="do_not_pad", max_length=self.tokenizer.model_max_length,
                             truncation=True, return_tensors="pt").input_ids.to(self.text_encoder.device)
        self.empty_text_embed = self.text_encoder(ids)[0].to(self.dtype)

    @torch.no_grad()
    def single_infer(self, rgb_in, num_inference_steps: int, show_pbar: bool = False, noise="gaussian",
                     normals=False, generator=None):
        device = self.device
        rgb_in = rgb_in.to(device)
        # the kernels index each tensor with 32-bit element offsets: split batches whose largest activation
        # (256 channels at full resolution in the VAE decoder) would exceed 2^32 elements
        B, _, H, W = rgb_in.shape
        _check_image_size(H, W)
        max_b = max(1, (2 ** 32 - 1) // (256 * H * W))
        if B > max_b:
            return torch.cat([self.single_infer(rgb_in[i:i + max_b], num_inference_steps, show_pbar, noise=noise,
                                                normals=normals, generator=generator)
                              for i in range(0, B, max_b)], dim=0)
        _check_noise(noise, num_inference_steps)
        graph = self.use_cuda_graph and rgb_in.is_cuda and not torch.cuda.is_current_stream_capturing()
        mem_eff = bool(getattr(self.vae, "memory_efficient_attention", False))
        if graph and noise == "zeros" and num_inference_steps == 1:
            key = ("marigold", tuple(rgb_in.shape), rgb_in.dtype, bool(normals), mem_eff)
            return self._graphed(key, lambda x: self._single_infer_impl(x, 1, noise, normals, None), rgb_in)
        # the initial latent is drawn here, outside any graph, on every call (marigold_pipeline.py:410-423)
        init = None if noise == "zeros" else self._initial_latent(rgb_in, noise, generator)
        if graph:
            self.scheduler.set_timesteps(num_inference_steps)
            sched = self.scheduler
            key = ("marigold-ddim", tuple(rgb_in.shape), rgb_in.dtype, bool(normals), mem_eff,
                   tuple(sched._host_timesteps), sched.config["prediction_type"], sched._final_ac, init is None,
                   tuple(sched.coefficients(i) for i in range(num_inference_steps)))
            if init is None:
                return self._graphed(key, lambda x: self._single_infer_impl(x, num_inference_steps, noise, normals,
                                                                            None), rgb_in)
            return self._graphed(key, lambda x, z: self._single_infer_impl(x, num_inference_steps, noise, normals,
                                                                           None, init_latent=z), rgb_in, init)
        return self._single_infer_impl(rgb_in, num_inference_steps, noise, normals, generator, init_latent=init)

    def _latent_shape(self, rgb_in):
        """[B, latent_channels, h, w] of encode_rgb(rgb_in): every VAE down-sampling conv (pad (0,1,0,1), stride 2)
        floors the size."""
        B, _, h, w = rgb_in.shape
        for _ in range(len(self.vae.config["block_out_channels"]) - 1):
            h, w = h // 2, w // 2
        return B, self.vae.config["latent_channels"], h, w

    def _initial_latent(self, rgb_in, noise, generator):
        """The reference's initial latent (marigold_pipeline.py:410-423), in the module dtype; host-pipeline code."""
        shape = self._latent_shape(rgb_in)
        if noise == "gaussian":
            return torch.randn(shape, device=rgb_in.device, dtype=self.dtype, generator=generator)
        return pyramid_noise_like(torch.empty(shape, device=rgb_in.device, dtype=self.dtype), generator=generator)

    def _single_infer_impl(self, rgb_in, num_inference_steps, noise, normals, generator, init_latent=None):
        device = rgb_in.device
        self.scheduler.set_timesteps(num_inference_steps)        # host-side only: graph-capture safe
        rgb_latent = self.encode_rgb(rgb_in)
        if noise != "zeros" and init_latent is None:
            init_latent = self._initial_latent(rgb_in, noise, generator)
        if self.empty_text_embed is None:
            self.encode_empty_text()
        # one context for the whole batch (marigold_pipeline.py:428-432 `.repeat`s it): passed as a broadcast view so
        # the UNet can take its constant-context cross-attention path (same values, no copy)
        ctx = self.empty_text_embed.to(device).expand(rgb_latent.shape[0], -1, -1)
        spec = getattr(self.unet, "single_step_specialisations", False)
        pt = self.scheduler.config["prediction_type"]
        # DDIM state x_t in fp32 whatever the module dtype; None = exact zeros (never materialised)
        latent = None if init_latent is None else init_latent.to(torch.float32, memory_format=torch.contiguous_format,
                                                                  copy=True)
        unet_in = None
        if latent is not None or not spec or num_inference_steps > 1:
            # one persistent [B, 8, h, w] UNet input: [rgb_latent | x_t] (this order is important, :447-449); every
            # intermediate DDIM step writes x_{t-1} into channels 4..7 in the UNet operand dtype
            B, c, h, w = rgb_latent.shape
            unet_in = torch.empty((B, 2 * c, h, w), dtype=rgb_latent.dtype, device=device)
            unet_in[:, :c].copy_(rgb_latent)
            if init_latent is None:
                unet_in[:, c:].zero_()
            else:
                unet_in[:, c:].copy_(init_latent)
        for i in range(num_inference_steps):
            t, _, a_t, a_prev = self.scheduler.coefficients(i)
            if latent is None and spec:
                unet_input = rgb_latent                               # the zero half is never materialised: conv_in on 4 channels
            else:
                unet_input = unet_in
            pred = self.unet(unet_input, t, encoder_hidden_states=ctx).sample
            if i == num_inference_steps - 1:
                # last step: latent = pred_original_sample, x0 = c_x * x_t + c_m * model_out fused with /scale +
                # post_quant_conv + decoder
                c_x, c_m = _x0_coefficients(pt, a_t)
                dec = self.vae.decode_from_prediction(pred, c_m, noisy=latent, c_noisy=c_x)
                break
            # intermediate DDIM step (eta = 0), one kernel: x_t -> x_{t-1} in place and into the next UNet input
            latent, _ = ops.ddim_step(pred, latent, a_t, a_prev, pt, out=latent, unet_in=unet_in[:, rgb_latent.shape[1]:])
        if normals:
            return ops.decode_post(dec.float().contiguous(), normals=True).to(dec.dtype)
        return ops.decode_post(dec.float().contiguous(), normals=False).to(dec.dtype)

    def encode_rgb(self, rgb_in):
        return self.vae.encode_scaled_mean(rgb_in)

    def decode_depth(self, depth_latent):
        z = self.vae.post_quant_conv(depth_latent, scale_in=1.0 / self.depth_latent_scale_factor)
        return self.vae.decoder(z).mean(dim=1, keepdim=True)

    def decode_normal(self, normal_latent):
        z = self.vae.post_quant_conv(normal_latent, scale_in=1.0 / self.depth_latent_scale_factor)
        return self.vae.decoder(z)


# ------------------------------------------------------------------------------------ GeoWizard
@dataclass
class DepthNormalPipelineOutput:
    depth_np: np.ndarray
    depth_colored: Optional[object]
    normal_np: np.ndarray
    normal_colored: Optional[object]
    uncertainty: Optional[np.ndarray] = None


class DepthNormalEstimationPipeline(PipelineBase):
    """GeoWizard joint depth+normal pipeline (geowizard_pipeline.py).  The image context comes from `image_encoder`
    (clip_vision.B200CLIPVisionModelWithProjection, or any object with the transformers interface) through
    `encode_img_embed` (:232-248), or is passed in as `img_embed` ([B or 1, 1, 768])."""

    latent_scale_factor = 0.18215

    def __init__(self, unet, vae, scheduler, image_encoder=None, feature_extractor=None):
        self.register_modules(unet=unet, vae=vae, scheduler=scheduler, image_encoder=image_encoder,
                              feature_extractor=feature_extractor)
        self.img_embed = None

    @staticmethod
    def class_embedding(domain, batch, device, dtype):
        """geowizard_pipeline.py:290-302 batched as train_depth_normal.py:684-704 -> [2B, 10]."""
        geo_class = torch.tensor([[0., 1.], [1., 0.]], device=device, dtype=dtype)
        geo = torch.cat([torch.sin(geo_class), torch.cos(geo_class)], dim=-1).repeat_interleave(batch, 0)
        dom = {"indoor": [1., 0., 0.], "outdoor": [0., 1., 0.], "object": [0., 0., 1.]}[domain]
        dom = torch.tensor([dom], device=device, dtype=dtype).repeat(2 * batch, 1)
        return torch.cat((geo, torch.cat([torch.sin(dom), torch.cos(dom)], dim=-1)), dim=-1)

    @torch.no_grad()
    def single_infer(self, input_rgb, num_inference_steps: int, domain: str, show_pbar: bool = False,
                     noise="zeros", img_embed=None, generator=None):
        """geowizard_pipeline.py:251-344: any number of DDIM steps on the joint [depth x B, normal x B] latent, from
        zeros, gaussian (one draw shared by both halves, :271-272) or GeoWizard's pyramid noise (:33-43)."""
        _check_geowizard_noise(noise, num_inference_steps)
        device = input_rgb.device
        B = input_rgb.shape[0]
        _check_image_size(input_rgb.shape[-2], input_rgb.shape[-1])
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        rgb_latent = self.encode_RGB(input_rgb)
        if noise == "gaussian":
            geo_init = torch.randn(rgb_latent.shape, device=device, dtype=self.dtype,
                                   generator=generator).repeat(2, 1, 1, 1)
        elif noise == "pyramid":
            geo_init = geowizard_pyramid_noise_like(rgb_latent, self.scheduler.timesteps).repeat(2, 1, 1, 1)
        else:
            geo_init = None
        rgb_latent = rgb_latent.repeat(2, 1, 1, 1)
        emb = img_embed if img_embed is not None else self.img_embed
        if emb is None and self.image_encoder is not None:
            emb = self.encode_img_embed(input_rgb)
        if emb is None:
            raise RuntimeError("no image_encoder registered: pass img_embed ([B or 1,1,768])")
        ctx = emb.to(device)
        ctx = ctx.repeat(2, 1, 1) if ctx.shape[0] == B else ctx.repeat(2 * B, 1, 1)
        cls = self.class_embedding(domain, B, device, rgb_latent.dtype)
        if num_inference_steps == 1 and geo_init is None:
            # the E2E-FT setting (1 step, zeros): x_t = 0, so x0 = c_m * model_out
            geo_latent = torch.zeros_like(rgb_latent)
            t, _, a_t, _ = self.scheduler.coefficients(0)
            pred = self.unet(torch.cat([rgb_latent, geo_latent], dim=1), torch.full((2 * B,), t, device=device),
                             encoder_hidden_states=ctx, class_labels=cls).sample
            assert self.scheduler.config["prediction_type"] == "v_prediction"
            c_m = -math.sqrt(1.0 - a_t)
            d = self.vae.decode_from_prediction(pred[:B].contiguous(), c_m)
            n = self.vae.decode_from_prediction(pred[B:].contiguous(), c_m)
        else:
            d, n = self._denoise(rgb_latent, geo_init, num_inference_steps, ctx, cls)
        depth = ops.decode_post(d.float().contiguous(), normals=False).to(d.dtype)
        normal = ops.decode_post(n.float().contiguous(), normals=True, sign=-1.0).to(n.dtype)   # :342 sign flip
        return depth, normal

    def _denoise(self, rgb_latent, geo_init, num_inference_steps, ctx, cls):
        """The DDIM loop of :319-334 on the [2B] state (eager): unet(.., t.repeat(2B), class_labels) then one
        `ddim_step` kernel per intermediate step; the last step's x0 is fused into post_quant_conv for both halves.
        Returns the decoded (depth, normal) halves."""
        device = rgb_latent.device
        B2, c = rgb_latent.shape[:2]
        B = B2 // 2
        pt = self.scheduler.config["prediction_type"]
        latent = None if geo_init is None else geo_init.to(torch.float32, memory_format=torch.contiguous_format,
                                                             copy=True)
        unet_in = torch.empty((B2, 2 * c) + tuple(rgb_latent.shape[2:]), dtype=rgb_latent.dtype, device=device)
        unet_in[:, :c].copy_(rgb_latent)
        if geo_init is None:
            unet_in[:, c:].zero_()
        else:
            unet_in[:, c:].copy_(geo_init)
        for i in range(num_inference_steps):
            t, _, a_t, a_prev = self.scheduler.coefficients(i)
            pred = self.unet(unet_in, torch.full((B2,), t, device=device), encoder_hidden_states=ctx,
                             class_labels=cls).sample
            if i == num_inference_steps - 1:
                c_x, c_m = _x0_coefficients(pt, a_t)
                halves = []
                for sl in (slice(0, B), slice(B, B2)):
                    noisy = None if latent is None else latent[sl]
                    halves.append(self.vae.decode_from_prediction(pred[sl].contiguous(), c_m, noisy=noisy,
                                                                  c_noisy=c_x))
                return halves[0], halves[1]
            latent, _ = ops.ddim_step(pred, latent, a_t, a_prev, pt, out=latent, unet_in=unet_in[:, c:])

    @torch.no_grad()
    def encode_img_embed(self, rgb):
        """geowizard_pipeline.py:232-248: bicubic-antialiased resize of (rgb + 1) / 2 to the crop size, CLIP mean / std,
        image_encoder(...).image_embeds.unsqueeze(1) -> [B, 1, 768] (one context row per input image)."""
        enc = self.image_encoder
        if hasattr(enc, "preprocess"):                                    # the engine encoder: device kernels
            x = enc.preprocess(rgb.float().contiguous(), self.feature_extractor)
        else:
            raise RuntimeError("image_encoder has no device `preprocess`; use B200CLIPVisionModelWithProjection or pass img_embed")
        return enc(x.to(enc.dtype)).image_embeds.unsqueeze(1).to(self.dtype)

    def encode_RGB(self, rgb_in):
        return self.vae.encode_scaled_mean(rgb_in)

    def decode_depth(self, depth_latent):
        z = self.vae.post_quant_conv(depth_latent, scale_in=1.0 / self.latent_scale_factor)
        return self.vae.decoder(z).mean(dim=1, keepdim=True)

    def decode_normal(self, normal_latent):
        z = self.vae.post_quant_conv(normal_latent, scale_in=1.0 / self.latent_scale_factor)
        return self.vae.decoder(z)

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: int = 1, ensemble_size: int = 1, processing_res: int = 768,
                 match_input_res: bool = True, domain: str = "indoor", color_map: Optional[str] = None,
                 show_progress_bar: bool = False, noise="zeros", img_embed=None,
                 batch_size: int = 0, ensemble_kwargs=None) -> DepthNormalPipelineOutput:
        _check_geowizard_noise(noise, denoising_steps)
        check_color_map(color_map)
        assert ensemble_size >= 1 and batch_size >= 0
        if isinstance(input_image, torch.Tensor):
            rgb = input_image.squeeze()
        else:
            rgb = torch.from_numpy(np.asarray(input_image.convert("RGB")).copy()).permute(2, 0, 1)
        input_size = rgb.shape
        _check_image_size(*_max_res_size(input_size[-2], input_size[-1], processing_res))   # before any launch
        was_u8 = rgb.dtype == torch.uint8
        rgb = rgb.to(self.device).to(torch.float32)
        if processing_res > 0:
            rgb = _resize_max_res(rgb, processing_res)
        rgb_norm = normalise_rgb(rgb, round_u8=was_u8 and processing_res > 0).to(self.dtype)
        dl, nl = [], []
        bs = batch_size if batch_size > 0 else 1            # geowizard_pipeline.py:139-176 (0 -> one member per batch)
        for i in range(0, ensemble_size, bs):
            batch = rgb_norm[None].expand(min(bs, ensemble_size - i), -1, -1, -1).contiguous()
            d, n = self.single_infer(batch, denoising_steps, domain, show_progress_bar, noise, img_embed)
            dl.append(d)
            nl.append(n)
        depth, normal = torch.cat(dl).squeeze(), torch.cat(nl).squeeze()
        uncert = None
        if ensemble_size > 1:                               # :179-188
            depth, uncert = ensemble_depths(depth, **(ensemble_kwargs or {}))
            normal, _ = ensemble_normals(normal)
        depth, _ = minmax_normalise_(depth.to(torch.float32).contiguous())      # :192-194
        normal = normal.to(torch.float32)
        if match_input_res:
            # the reference resizes on the host (PIL for depth, cv2 INTER_NEAREST for normals, :201-206); here on the device
            depth = resize_bilinear_aa(depth[None], tuple(input_size[-2:]))[0]
            normal = resize_nearest(normal, tuple(input_size[-2:]))
        # colours (:210-220) from the device tensors that become depth_np / normal_np; the kernels clip as numpy does
        depth_colored = None if color_map is None else _to_pil(colorize_depth(depth, color_map))
        normal_colored = _to_pil(colorize_normals(normal))
        return DepthNormalPipelineOutput(depth_np=depth.cpu().numpy().clip(0, 1), depth_colored=depth_colored,
                                         normal_np=normal.cpu().numpy().clip(-1, 1), normal_colored=normal_colored,
                                         uncertainty=None if uncert is None else uncert.cpu().numpy())
