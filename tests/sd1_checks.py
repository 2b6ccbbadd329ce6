"""SD-1-shaped UNets (GeoWizard's: 8 heads of width 40 / 80 / 160, 1x1-conv projections) for the engine checks.

* The fp32 oracle of an SD-1 UNet: `unet_ref(cfg)` builds oracle.unet's UNet2DConditionRef and, for
  `use_linear_projection=False`, gives every Transformer2DModel the 1x1-conv projections of diffusers'
  transformer_2d.py (:152-155,214-217) and their NCHW forward (:332-339,408-414).  Its attention is already generic in
  the head width.  `sd1_config()` is the public SD-1.x UNet, `tiny_sd1_config()` a miniature with 320 channels over
  8 / 4 / 2 / 2 heads, so every level runs a new head width.
* `install_emulation(monkeypatch)`: tests/cpu_emulation.py's plain-torch kernel contracts plus those of the entry
  points for head widths other than 64 (ops.attention / ops.rowdot_heads_d).
* `sd1_tiny(monkeypatch)` points the tiny-model builders that tests/engine_checks.py uses (make_golden.build_tiny and
  engine_checks.engine_from_oracle) at the SD-1 miniature, with the context widths of the SD-2 miniature (128,
  GeoWizard 96).  The checks of engine_checks.py then run unchanged on it."""
from dataclasses import dataclass

import torch
import torch.nn as nn

import cpu_emulation
import engine_checks as EC
import make_golden as MG
from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, ops
from oracle import unet as OU
from oracle.unet import UNet2DConditionRef, UNetConfig, seeded_init
from oracle.vae import AutoencoderKLRef

# the GeoWizard SD-1 UNet as config.json stores it: one scalar head count, conv projections
GEOWIZARD_SD1 = dict(in_channels=8, attention_head_dim=8, use_linear_projection=False, cross_attention_dim=768,
                     class_embed_type="projection", projection_class_embeddings_input_dim=10, joint_attention=True)


# ----------------------------------------------------------------------------------------------- oracle
@dataclass
class SD1UNetConfig(UNetConfig):
    use_linear_projection: bool = False


def sd1_config(**kw):
    """SD-1.x UNet (lambdalabs/sd-image-variations-diffusers, the base of GeoWizard: train_depth_normal.py:343-345):
    8 heads of width 40 / 80 / 160 at 320 / 640 / 1280 channels, cross-attention width 768 (geowizard_pipeline.py:288),
    1x1-conv projections (unet_2d_condition.py:204-217 defaults)."""
    base = dict(in_channels=4, attention_head_dim=(8, 8, 8, 8), cross_attention_dim=768)
    base.update(kw)
    return SD1UNetConfig(**base)


def tiny_sd1_config(**kw):
    base = dict(block_out_channels=(320, 320, 320, 320), attention_head_dim=(8, 4, 2, 2), cross_attention_dim=128)
    base.update(kw)
    return SD1UNetConfig(**base)


class ConvProjTransformer2DModel(OU.Transformer2DModel):
    """transformer_2d.py:327-347,407-423 with use_linear_projection=False: GN -> 1x1 conv on NCHW -> flatten ->
    blocks -> unflatten -> 1x1 conv -> + residual."""

    def forward(self, x, ctx):
        B, C, H, W = x.shape
        h = self.proj_in(self.norm(x)).permute(0, 2, 3, 1).reshape(B, H * W, C)
        for blk in self.transformer_blocks:
            h = blk(h, ctx)
        h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
        return self.proj_out(h) + x


def unet_ref(cfg):
    unet = UNet2DConditionRef(cfg)
    if not getattr(cfg, "use_linear_projection", True):
        for m in [m for m in unet.modules() if isinstance(m, OU.Transformer2DModel)]:
            C = m.proj_in.in_features
            m.proj_in, m.proj_out = nn.Conv2d(C, C, 1), nn.Conv2d(C, C, 1)     # same state_dict positions
            m.__class__ = ConvProjTransformer2DModel
    return unet


def build_tiny_sd1(kind="marigold"):
    if kind == "geowizard":
        cfg = tiny_sd1_config(class_embed_type="projection", projection_class_embeddings_input_dim=10,
                              cross_attention_dim=96, joint_attention=True)
    else:
        cfg = tiny_sd1_config()
    unet = seeded_init(unet_ref(cfg), seed=1234).eval()
    vae = seeded_init(AutoencoderKLRef(MG.tiny_vae_config()), seed=77).eval()
    return unet, vae


# ----------------------------------------------------------------------------------------------- engine
def engine_unet(cfg, stream_dtype=torch.float32):
    """The engine UNet of an oracle config (every key the two share, projections included)."""
    return B200UNet2DConditionModel(
        stream_dtype=stream_dtype, in_channels=cfg.in_channels, out_channels=cfg.out_channels,
        block_out_channels=cfg.block_out_channels, attention_head_dim=cfg.attention_head_dim,
        cross_attention_dim=cfg.cross_attention_dim, class_embed_type=cfg.class_embed_type,
        projection_class_embeddings_input_dim=cfg.projection_class_embeddings_input_dim,
        joint_attention=cfg.joint_attention, use_linear_projection=getattr(cfg, "use_linear_projection", True))


def engine_from_oracle_sd1(unet_ref, vae_ref, device, stream_dtype=torch.float32, dtype=torch.float32,
                           vae_stream_dtype=None):
    """engine_checks.engine_from_oracle for any oracle UNet config."""
    unet = engine_unet(unet_ref.config, stream_dtype)
    unet.load_state_dict(unet_ref.state_dict(), strict=True)
    vae = None
    if vae_ref is not None:
        vae = B200AutoencoderKL(stream_dtype=vae_stream_dtype or stream_dtype,
                                block_out_channels=vae_ref.config.block_out_channels)
        vae.load_state_dict(vae_ref.state_dict(), strict=True)
        vae = vae.to(device=device, dtype=dtype).eval().requires_grad_(False)
    return unet.to(device=device, dtype=dtype).eval().requires_grad_(False), vae


def sd1_tiny(monkeypatch):
    monkeypatch.setattr(MG, "build_tiny", build_tiny_sd1)
    monkeypatch.setattr(EC, "engine_from_oracle", engine_from_oracle_sd1)


# ----------------------------------------------------------------------------------------------- emulation
def rowdot_heads_d(a, c, heads, head_dim):
    B, L, D = a.shape[0], a.shape[1], head_dim
    return (a[..., :heads * D].float() * c[..., :heads * D].float()).view(B, L, heads, D).sum(-1).permute(0, 2, 1).contiguous()


def attention(q, k, v, heads, scale, kv_segments=1, out=None, want_lse=False):
    B, Lq, C = q.shape
    D = C // heads
    if kv_segments == 2:                                   # batch b sees the keys of b % (B/2) then b % (B/2) + B/2
        h = B // 2
        k = torch.cat([torch.cat([k[:h], k[h:]], dim=1)] * 2, dim=0)
        v = torch.cat([torch.cat([v[:h], v[h:]], dim=1)] * 2, dim=0)

    def split(t):
        return t.float().unflatten(-1, (heads, D)).transpose(1, 2)
    k = k.expand(B, -1, -1) if k.shape[0] == 1 else k
    v = v.expand(B, -1, -1) if v.shape[0] == 1 else v
    logits = split(q) @ split(k).transpose(-1, -2) * scale
    o = (torch.softmax(logits, dim=-1) @ split(v)).transpose(1, 2).reshape(B, Lq, C).half()
    if out is not None:
        out.copy_(o)
        o = out
    if want_lse:
        return o, (torch.logsumexp(logits, dim=-1) * 1.4426950408889634).contiguous()      # log2 domain, [B, heads, Lq]
    return o


def install_emulation(monkeypatch):
    cpu_emulation.install(monkeypatch)
    monkeypatch.setattr(ops, "attention", attention)
    monkeypatch.setattr(ops, "rowdot_heads_d", rowdot_heads_d)
