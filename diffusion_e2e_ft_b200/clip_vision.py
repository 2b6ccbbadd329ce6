"""CLIP image encoder on the engine kernels (SURVEY.md §8 f4, the vision half).

Drop-in for `transformers.CLIPVisionModelWithProjection` where GeoWizard uses it, once per input image —
GeoWizard/geowizard/models/geowizard_pipeline.py:232-248: `TF.resize((rgb + 1) / 2, crop_size, BICUBIC, antialias=True)`,
CLIP mean / std normalisation, `self.image_encoder(x).image_embeds.unsqueeze(1)` -> the [1, 1, 768] context of every
cross-attention.  Parameter names are transformers' (`vision_model.embeddings.patch_embedding.weight`,
`vision_model.pre_layrnorm.weight` (sic), `visual_projection.weight`, ...), so `image_encoder/model.safetensors` of
the GeoWizard checkpoint loads with `load_state_dict` / `from_pretrained`.

Arithmetic (transformers==4.37.2 models/clip/modeling_clip.py, restated in oracle/clip_vision.py):
patch embedding = one wgmma GEMM over the 14x14x3 patches (K 588 zero-padded to 640) whose epilogue adds the
position embedding and writes straight into rows 1.. of the token matrix; class token + its position row is a
packed constant; pre-LayerNorm; N x the encoder layer of clip_text.py (non-causal: one flash-attention launch over
the 257 tokens, head_dim 64; quick_gelu on the SiLU epilogue); post-LayerNorm of the class token; bias-free projection
GEMM.  torch only rearranges memory (patch gather, dtype casts).  `preprocess` is geowizard_pipeline.py:236-245 on the
device: b200_resize_bicubic_aa + the per-channel affine map (b200_pointwise_nchw).  No CPU fallback.
"""
import json
import os
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .clip_text import _Encoder
from .ensemble import resize_bicubic_aa
from .modules import ConfigDict, Packed, _f16, _f32
from .ops import F16, F32

CLIP_IMAGE_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_IMAGE_STD = (0.26862954, 0.26130258, 0.27577711)


class CLIPImageProcessorConfig:
    """What geowizard_pipeline.py:236-241 reads from its `feature_extractor`: image_mean, image_std, crop_size."""

    def __init__(self, size=224, image_mean=CLIP_IMAGE_MEAN, image_std=CLIP_IMAGE_STD):
        self.image_mean, self.image_std = list(image_mean), list(image_std)
        self.crop_size = {"height": size, "width": size}

    @classmethod
    def from_pretrained(cls, directory, subfolder=None):
        d = directory if subfolder is None else os.path.join(directory, subfolder)
        with open(os.path.join(d, "preprocessor_config.json")) as f:
            raw = json.load(f)
        cs = raw.get("crop_size", 224)
        size = cs["height"] if isinstance(cs, dict) else cs
        return cls(size, raw.get("image_mean", CLIP_IMAGE_MEAN), raw.get("image_std", CLIP_IMAGE_STD))


class _VisionEmbeddings(nn.Module):
    def __init__(self, C, patch, n_pos):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(C))
        self.patch_embedding = nn.Conv2d(3, C, patch, stride=patch, bias=False)
        self.position_embedding = nn.Embedding(n_pos, C)


class _VisionTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        C, eps = cfg["hidden_size"], cfg["layer_norm_eps"]
        self.embeddings = _VisionEmbeddings(C, cfg["patch_size"], (cfg["image_size"] // cfg["patch_size"]) ** 2 + 1)
        self.pre_layrnorm = nn.LayerNorm(C, eps=eps)
        self.encoder = _Encoder(cfg["num_hidden_layers"], C, cfg["intermediate_size"], eps, cfg["hidden_act"])
        self.post_layernorm = nn.LayerNorm(C, eps=eps)


class CLIPVisionOutput(SimpleNamespace):
    """`.image_embeds` [B, proj], `.last_hidden_state` [B, 1 + patches, C] (transformers CLIPVisionModelOutput)."""

    def __getitem__(self, i):
        return (self.image_embeds, self.last_hidden_state)[i]


_CFG_KEYS = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size", "patch_size",
             "projection_dim", "layer_norm_eps", "hidden_act")


class B200CLIPVisionModelWithProjection(nn.Module):
    def __init__(self, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                 image_size=224, patch_size=14, projection_dim=768, layer_norm_eps=1e-5, hidden_act="quick_gelu", **extra):
        super().__init__()
        if hidden_size != 64 * num_attention_heads:
            raise NotImplementedError(f"head width {hidden_size // num_attention_heads}: the attention kernel is d=64")
        if hidden_act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"hidden_act={hidden_act!r}")
        if image_size % patch_size:
            raise ValueError("image_size must be a multiple of patch_size")
        self.config = ConfigDict(hidden_size=hidden_size, intermediate_size=intermediate_size,
                                 num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                                 image_size=image_size, patch_size=patch_size, projection_dim=projection_dim,
                                 layer_norm_eps=layer_norm_eps, hidden_act=hidden_act)
        if extra:
            self.config["_extra"] = dict(extra)
        self.vision_model = _VisionTransformer(self.config)
        self.visual_projection = nn.Linear(hidden_size, projection_dim, bias=False)
        self._pk = Packed()

    @property
    def device(self):
        return self.visual_projection.weight.device

    @property
    def dtype(self):
        return self.visual_projection.weight.dtype

    def register_to_config(self, **kw):
        self.config.update(kw)

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = dict(state_dict)
        sd.pop("vision_model.embeddings.position_ids", None)      # a persistent buffer in transformers < 4.31 checkpoints
        return super().load_state_dict(sd, strict=strict, **kw)

    def save_pretrained(self, save_directory, safe_serialization=True, **unused):
        os.makedirs(save_directory, exist_ok=True)
        cfg = {k: v for k, v in self.config.items() if k != "_extra"}
        cfg.update(self.config.get("_extra", {}))
        cfg.update(architectures=["CLIPVisionModelWithProjection"], model_type="clip_vision_model")
        with open(os.path.join(save_directory, "config.json"), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)
        sd = {k: v.detach().to("cpu").contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, "model.safetensors"), metadata={"format": "pt"})
        else:
            torch.save(sd, os.path.join(save_directory, "pytorch_model.bin"))

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, torch_dtype=None, **unused):
        d = pretrained_model_name_or_path if subfolder is None else os.path.join(pretrained_model_name_or_path, subfolder)
        if not os.path.isdir(d):
            raise FileNotFoundError(f"{d}: not a directory (local checkpoint folders only; there is no hub access)")
        with open(os.path.join(d, "config.json")) as f:
            raw = json.load(f)
        raw = dict(raw.get("vision_config", {}), **{k: v for k, v in raw.items() if k != "vision_config"})
        model = cls(**{k: raw[k] for k in _CFG_KEYS if k in raw})
        extra = {k: v for k, v in raw.items() if k not in _CFG_KEYS and k not in ("architectures", "model_type")}
        if extra:
            model.config["_extra"] = extra
        safe, binp = os.path.join(d, "model.safetensors"), os.path.join(d, "pytorch_model.bin")
        if os.path.exists(safe):
            from safetensors.torch import load_file
            sd = load_file(safe)
        elif os.path.exists(binp):
            sd = torch.load(binp, map_location="cpu")
        else:
            raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin in {d}")
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()

    # ---------------------------------------------------------------------------------------------- arithmetic
    def _packed(self):
        vm, emb = self.vision_model, self.vision_model.embeddings
        params = [emb.class_embedding, emb.patch_embedding.weight, emb.position_embedding.weight, vm.pre_layrnorm.weight,
                  vm.pre_layrnorm.bias, vm.post_layernorm.weight, vm.post_layernorm.bias, self.visual_projection.weight]

        def build():
            C = self.config["hidden_size"]
            k = 3 * self.config["patch_size"] ** 2
            kpad = (k + 63) // 64 * 64
            wp = torch.zeros((C, kpad), dtype=F16, device=self.device)
            wp[:, :k] = emb.patch_embedding.weight.detach().reshape(C, k).to(F16)
            pos = _f32(emb.position_embedding.weight)
            return dict(wp=wp, k=k, kpad=kpad, pos_patches=pos[1:].contiguous(),
                        cls_pos=(emb.class_embedding.detach().float() + pos[0]).contiguous(),
                        pre=(_f32(vm.pre_layrnorm.weight), _f32(vm.pre_layrnorm.bias)),
                        post=(_f32(vm.post_layernorm.weight), _f32(vm.post_layernorm.bias)),
                        proj=_f16(self.visual_projection.weight))
        return self._pk.get(params, build)

    @torch.no_grad()
    def forward(self, pixel_values, **_ignored):
        """pixel_values [B, 3, image_size, image_size] (normalised; fp16 or fp32, CUDA) -> CLIPVisionOutput."""
        cfg = self.config
        ops._need_cuda(pixel_values)
        B, ch, S, S2 = pixel_values.shape
        P, C, H = cfg["patch_size"], cfg["hidden_size"], cfg["num_attention_heads"]
        if ch != 3 or S != cfg["image_size"] or S2 != S:
            raise ValueError(f"pixel_values {tuple(pixel_values.shape)}: expected [B, 3, {cfg['image_size']}, {cfg['image_size']}]")
        g = S // P
        n, L = g * g, g * g + 1
        pk = self._packed()
        # patch gather (memory rearrangement): [B,3,g,P,g,P] -> [B, g*g, 3*P*P] fp16, K zero-padded for the 64-wide k-blocks
        a = torch.zeros((B, n, pk["kpad"]), dtype=F16, device=pixel_values.device)
        a[..., :pk["k"]].copy_(pixel_values.view(B, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B, n, pk["k"]))
        h = torch.empty((B, L, C), dtype=F32, device=pixel_values.device)
        ops.linear(a, pk["wp"], residual=pk["pos_patches"].unsqueeze(0).expand(B, n, C), out=h[:, 1:, :], out_dtype=F32)
        h[:, 0, :].copy_(pk["cls_pos"])
        h = ops.layer_norm(h.view(B * L, C), *pk["pre"], eps=cfg["layer_norm_eps"]).to(F32)      # the residual stream
        for layer in self.vision_model.encoder.layers:
            h = layer.run(h, B, L, H, causal=False)
        last = h.view(B, L, C)
        pooled = ops.layer_norm(last[:, 0, :].contiguous(), *pk["post"], eps=cfg["layer_norm_eps"])
        embeds = ops.linear(pooled, pk["proj"], out_dtype=F32)
        return CLIPVisionOutput(image_embeds=embeds.to(self.dtype), last_hidden_state=last.to(self.dtype))

    @torch.no_grad()
    def preprocess(self, rgb, feature_extractor=None):
        """geowizard_pipeline.py:236-245: rgb in [-1, 1] [B, 3, H, W] (CUDA) -> normalised [B, 3, crop, crop] fp32.
        The resize is linear with weights summing to 1, so ((x + 1) / 2 resized - mean) / std is one per-channel affine
        map of the resized rgb: a = 0.5 / std, b = (0.5 - mean) / std."""
        fe = feature_extractor or CLIPImageProcessorConfig(self.config["image_size"])
        size = (fe.crop_size["height"], fe.crop_size["width"])
        x = resize_bicubic_aa(rgb, size)
        key = (str(rgb.device), tuple(fe.image_mean), tuple(fe.image_std))
        cache = self.__dict__.setdefault("_affine", {})
        if key not in cache:                                             # once per device: no per-image host->device copy
            std = torch.tensor(fe.image_std, dtype=F32)
            mean = torch.tensor(fe.image_mean, dtype=F32)
            cache[key] = (torch.diag(0.5 / std).to(rgb.device), ((0.5 - mean) / std).to(rgb.device))
        return ops.pointwise_nchw(x, 1.0, *cache[key])
