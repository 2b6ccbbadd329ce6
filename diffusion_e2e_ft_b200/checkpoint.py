"""Checkpoint I/O in the diffusers directory layout (SURVEY.md §8 b / f4): `save_pretrained(dir)` writes
`config.json` + `diffusion_pytorch_model.safetensors`, `from_pretrained(dir, subfolder=...)` reads them back (a
`.bin` state dict is accepted too).  This is what the reference's accelerate hooks call on the UNet
(training/train.py:322-339: `model.save_pretrained(os.path.join(output_dir, "unet"))`,
`UNet2DConditionModel.from_pretrained(input_dir, subfolder="unet")` then `register_to_config(**load_model.config)` +
`load_state_dict`), and what `StableDiffusionPipeline.save_pretrained` does per module at :610-630.  Parameter names
are the diffusers names (App. A.8), so a real SD-2 / Marigold / E2E-FT checkpoint directory loads unchanged; config
keys the engine does not model (e.g. `_class_name`, `dropout`, `upcast_attention`) are kept aside in `config["_extra"]`
and written back on save."""
import json
import os

import torch

WEIGHTS_SAFE = "diffusion_pytorch_model.safetensors"
WEIGHTS_BIN = "diffusion_pytorch_model.bin"
CONFIG_NAME = "config.json"


def load_weights(directory):
    """The state dict of a diffusers model folder (safetensors, else .bin), on the CPU."""
    safe, binp = os.path.join(directory, WEIGHTS_SAFE), os.path.join(directory, WEIGHTS_BIN)
    if os.path.exists(safe):
        from safetensors.torch import load_file
        return load_file(safe)
    if os.path.exists(binp):
        return torch.load(binp, map_location="cpu")
    raise FileNotFoundError(f"no {WEIGHTS_SAFE} / {WEIGHTS_BIN} in {directory}")


class PretrainedMixin:
    _diffusers_class_name = None       # e.g. "UNet2DConditionModel"
    _config_defaults = None            # dict of the keys the engine models

    def save_pretrained(self, save_directory, safe_serialization=True, state_dict=None, extra_config=None, **unused):
        """`state_dict`: weights to write instead of the module's own (e.g. an EMA copy, same names and shapes);
        `extra_config`: keys added to config.json (e.g. EMAModel's settings)."""
        os.makedirs(save_directory, exist_ok=True)
        cfg = {k: (list(v) if isinstance(v, tuple) else v) for k, v in self.config.items() if k != "_extra"}
        cfg.update(self.config.get("_extra", {}))
        cfg.update(extra_config or {})
        cfg["_class_name"] = self._diffusers_class_name
        cfg.setdefault("_diffusers_version", "0.30.2")
        with open(os.path.join(save_directory, CONFIG_NAME), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)
        sd = {k: v.detach().to("cpu").contiguous() for k, v in (state_dict or self.state_dict()).items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, WEIGHTS_SAFE), metadata={"format": "pt"})
        else:
            torch.save(sd, os.path.join(save_directory, WEIGHTS_BIN))

    @classmethod
    def load_config(cls, directory):
        with open(os.path.join(directory, CONFIG_NAME)) as f:
            raw = json.load(f)
        known = {k: raw[k] for k in cls._config_defaults if k in raw}
        for k, v in known.items():
            if isinstance(cls._config_defaults[k], tuple) and isinstance(v, list):
                known[k] = tuple(v)
        # a scalar attention_head_dim (diffusers' SD-1 configs) stays a scalar: the model expands it per block and
        # save_pretrained writes it back as it was read
        extra = {k: v for k, v in raw.items() if k not in cls._config_defaults and k != "_class_name"}
        return known, extra

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, torch_dtype=None, **kwargs):
        d = pretrained_model_name_or_path if subfolder is None else os.path.join(pretrained_model_name_or_path, subfolder)
        if not os.path.isdir(d):
            raise FileNotFoundError(f"{d}: not a directory (the engine loads local diffusers checkpoint folders; there is "
                                    "no hub access)")
        known, extra = cls.load_config(d)
        known.update({k: v for k, v in kwargs.items() if k in cls._config_defaults})
        stream = kwargs.get("stream_dtype", torch.float32)
        model = cls(stream_dtype=stream, **known)
        if extra:
            model.config["_extra"] = extra
        model.load_state_dict(load_weights(d), strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()
