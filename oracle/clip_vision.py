"""ORACLE (test infrastructure) — fp32 PyTorch restatement of the CLIP IMAGE encoder GeoWizard conditions its UNet on
(GeoWizard/geowizard/models/geowizard_pipeline.py:232-248: bicubic antialiased resize of (rgb + 1) / 2 to the
feature extractor's crop size, CLIP mean / std normalisation, `self.image_encoder(x).image_embeds.unsqueeze(1)`
-> [1, 1, 768], once per input image).

The model is transformers==4.37.2 (requirements.txt:7) `CLIPVisionModelWithProjection`, absent from the reference checkout:
models/clip/modeling_clip.py — CLIPVisionEmbeddings (bias-free patch conv, class token, learned positions),
`pre_layrnorm` (sic), CLIPEncoderLayer x N (non-causal), `post_layernorm` of the class token, bias-free
`visual_projection`.  Restated from that published algorithm with the transformers `state_dict` names and PINNED in
tests/test_clip_vision.py against the installed transformers (5.5.0) on shared random weights.  Only tests/ may
import this module.
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from .clip_text import _act

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)      # CLIPImageProcessor defaults (feature_extractor/preprocessor_config.json)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@dataclass
class CLIPVisionCfg:
    hidden_size: int = 1024                 # lambdalabs/sd-image-variations-diffusers image_encoder (OpenAI ViT-L/14)
    intermediate_size: int = 4096
    num_hidden_layers: int = 24
    num_attention_heads: int = 16
    image_size: int = 224
    patch_size: int = 14
    projection_dim: int = 768
    layer_norm_eps: float = 1e-5
    hidden_act: str = "quick_gelu"


def tiny_vision_cfg(**kw):
    base = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, image_size=56,
                projection_dim=64)
    base.update(kw)
    return CLIPVisionCfg(**base)


def random_vision_state_dict(cfg: CLIPVisionCfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    C, I, P = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size
    n_pos = (cfg.image_size // P) ** 2 + 1

    def rn(*shape, s=1.0):
        return torch.randn(*shape, generator=g) * s
    sd = {"vision_model.embeddings.class_embedding": rn(C, s=0.5),
          "vision_model.embeddings.patch_embedding.weight": rn(C, 3, P, P, s=(3 * P * P) ** -0.5),
          "vision_model.embeddings.position_embedding.weight": rn(n_pos, C, s=0.5),
          "vision_model.pre_layrnorm.weight": 1.0 + rn(C, s=0.1), "vision_model.pre_layrnorm.bias": rn(C, s=0.1),
          "vision_model.post_layernorm.weight": 1.0 + rn(C, s=0.1), "vision_model.post_layernorm.bias": rn(C, s=0.1),
          "visual_projection.weight": rn(cfg.projection_dim, C, s=C ** -0.5)}
    for i in range(cfg.num_hidden_layers):
        p = f"vision_model.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{n}.weight"] = rn(C, C, s=C ** -0.5)
            sd[p + f"self_attn.{n}.bias"] = rn(C, s=0.1)
        for n in ("layer_norm1", "layer_norm2"):
            sd[p + n + ".weight"] = 1.0 + rn(C, s=0.1)
            sd[p + n + ".bias"] = rn(C, s=0.1)
        sd[p + "mlp.fc1.weight"] = rn(I, C, s=C ** -0.5)
        sd[p + "mlp.fc1.bias"] = rn(I, s=0.1)
        sd[p + "mlp.fc2.weight"] = rn(C, I, s=I ** -0.5)
        sd[p + "mlp.fc2.bias"] = rn(C, s=0.1)
    return sd


@torch.no_grad()
def clip_vision_forward(sd, cfg: CLIPVisionCfg, pixel_values: torch.Tensor):
    """pixel_values [B, 3, S, S] (already normalised) -> (image_embeds [B, proj], last_hidden_state [B, 1 + n, C])."""
    sd = {k: v.float() for k, v in sd.items()}
    x = pixel_values.float()
    B = x.shape[0]
    C, H, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps
    d = C // H
    pe = F.conv2d(x, sd["vision_model.embeddings.patch_embedding.weight"], stride=cfg.patch_size)   # [B, C, g, g]
    pe = pe.flatten(2).transpose(1, 2)
    cls = sd["vision_model.embeddings.class_embedding"].expand(B, 1, C)
    h = torch.cat([cls, pe], 1) + sd["vision_model.embeddings.position_embedding.weight"][None]
    L = h.shape[1]
    h = F.layer_norm(h, (C,), sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"], eps)
    for i in range(cfg.num_hidden_layers):
        p = f"vision_model.encoder.layers.{i}."
        y = F.layer_norm(h, (C,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], eps)
        q = F.linear(y, sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"]) * d ** -0.5
        k = F.linear(y, sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"])
        v = F.linear(y, sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"])
        q, k, v = (t.view(B, L, H, d).transpose(1, 2) for t in (q, k, v))
        o = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(B, L, C)
        h = h + F.linear(o, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
        y = F.layer_norm(h, (C,), sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], eps)
        m = _act(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]), cfg.hidden_act)
        h = h + F.linear(m, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    pooled = F.layer_norm(h[:, 0], (C,), sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"], eps)
    return F.linear(pooled, sd["visual_projection.weight"]), h


@torch.no_grad()
def geowizard_img_embed(sd, cfg: CLIPVisionCfg, rgb: torch.Tensor):
    """geowizard_pipeline.py:232-248: rgb in [-1, 1] [B, 3, H, W] -> img_embed [B, 1, proj]."""
    x = F.interpolate((rgb.float() + 1) / 2, size=(cfg.image_size, cfg.image_size), mode="bicubic", antialias=True,
                      align_corners=False)                                       # torchvision TF.resize(BICUBIC, antialias)
    mean = torch.tensor(CLIP_MEAN)[None, :, None, None]
    std = torch.tensor(CLIP_STD)[None, :, None, None]
    return clip_vision_forward(sd, cfg, (x - mean) / std)[0].unsqueeze(1)
