"""ORACLE (test infrastructure) — fp32 PyTorch restatement of `UNet2DConditionModel`.

Follows the control flow of GeoWizard/geowizard/models/unet_2d_condition.py:845-1221
(identical to diffusers 0.30.2), unet_2d_blocks.py:634-777 (mid), :1027-1185
(CrossAttnDownBlock2D), :1188-1273 (DownBlock2D), :2201-2371 (CrossAttnUpBlock2D),
:2374-2481 (UpBlock2D), transformer_2d.py:327-423 and attention.py:292-413,430-513,
719-777.  Leaf ops (ResnetBlock2D, Downsample2D, Upsample2D, Attention, GEGLU,
Timesteps, TimestepEmbedding) are third-party diffusers code that is NOT under
the reference checkout; they are restated from their published 0.30.2 semantics (SURVEY.md App. A).

Parameter names reproduce the diffusers `state_dict` layout (SURVEY.md App. A.8).
"""
import math
import re
from dataclasses import dataclass, field
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class UNetConfig:
    # defaults = SD-2 / Marigold config.json (defaults visible at unet_2d_condition.py:179-234)
    in_channels: int = 8
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",)
    up_block_types: Tuple[str, ...] = ("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3
    layers_per_block: int = 2
    attention_head_dim: Tuple[int, ...] = (5, 10, 20, 20)   # used as NUMBER OF HEADS (:244-250)
    cross_attention_dim: int = 1024
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    class_embed_type: Optional[str] = None                   # "projection" for GeoWizard
    projection_class_embeddings_input_dim: Optional[int] = None
    joint_attention: bool = False                            # XFormersJointAttnProcessor (attention.py:425)
    flip_sin_to_cos: bool = True
    freq_shift: int = 0

    def __getitem__(self, k):
        return getattr(self, k)


def tiny_config(**kw):
    """Structurally complete miniature (same block types, 4 levels) for fast CPU tests."""
    base = dict(block_out_channels=(64, 128, 256, 256), attention_head_dim=(1, 2, 4, 4),
                cross_attention_dim=128)
    base.update(kw)
    return UNetConfig(**base)


# ----------------------------------------------------------------------------- leaves
def timestep_embedding(t: torch.Tensor, dim: int, flip_sin_to_cos=True, freq_shift=0):
    """diffusers `get_timestep_embedding` (App. A.3; called at unet_2d_condition.py:974)."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device)
    exponent = exponent / (half - freq_shift)
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return emb


class TimestepEmbedding(nn.Module):
    def __init__(self, in_dim, dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_dim, dim)
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class ResnetBlock2D(nn.Module):
    """App. A.2.  temb_channels=None for the VAE."""

    def __init__(self, cin, cout, temb_channels=1280, groups=32, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        if temb_channels is not None:
            self.time_emb_proj = nn.Linear(temb_channels, cout)
        else:
            self.time_emb_proj = None
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x, temb=None):
        h = self.conv1(F.silu(self.norm1(x)))
        if self.time_emb_proj is not None:
            h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    """App. A.4: pad=1 (UNet) or asymmetric (0,1,0,1) pad then pad=0 (VAE encoder)."""

    def __init__(self, ch, padding=1):
        super().__init__()
        self.padding = padding
        self.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=padding)

    def forward(self, x):
        if self.padding == 0:
            x = F.pad(x, (0, 1, 0, 1))
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, padding=1)

    def forward(self, x, output_size=None):
        if output_size is None:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
        else:
            x = F.interpolate(x, size=output_size, mode="nearest")
        return self.conv(x)


class Attention(nn.Module):
    """App. A.5.  `joint=True` restates XFormersJointAttnProcessor (attention.py:430-513)."""

    def __init__(self, dim, heads, cross_dim=None, bias=False, joint=False):
        super().__init__()
        self.heads = heads
        self.joint = joint
        self.to_q = nn.Linear(dim, dim, bias=bias)
        self.to_k = nn.Linear(cross_dim or dim, dim, bias=bias)
        self.to_v = nn.Linear(cross_dim or dim, dim, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim), nn.Dropout(0.0)])

    def forward(self, x, ctx=None):
        B, L, C = x.shape
        q = self.to_q(x)
        src = x if ctx is None else ctx
        k = self.to_k(src)
        v = self.to_v(src)
        if self.joint:
            assert ctx is None and B % 2 == 0
            k0, k1 = torch.chunk(k, 2, dim=0)              # attention.py:482
            v0, v1 = torch.chunk(v, 2, dim=0)
            k = torch.cat([torch.cat([k0, k1], dim=1)] * 2, dim=0)   # :487-491
            v = torch.cat([torch.cat([v0, v1], dim=1)] * 2, dim=0)
        h = self.heads
        d = C // h
        q = q.view(B, -1, h, d).transpose(1, 2)
        k = k.view(B, -1, h, d).transpose(1, 2)
        v = v.view(B, -1, h, d).transpose(1, 2)
        s = torch.matmul(q, k.transpose(-1, -2)) * (d ** -0.5)
        p = torch.softmax(s, dim=-1)
        o = torch.matmul(p, v).transpose(1, 2).reshape(B, L, C)
        return self.to_out[0](o)


class GEGLU(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner * 2)

    def forward(self, x):
        h, g = self.proj(x).chunk(2, dim=-1)
        return h * F.gelu(g)                               # erf GELU (attention.py:754-755)


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class BasicTransformerBlock(nn.Module):
    """attention.py:292-413."""

    def __init__(self, dim, heads, cross_dim, joint=False):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        self.attn1 = Attention(dim, heads, joint=joint)
        self.norm2 = nn.LayerNorm(dim, eps=1e-5)
        self.attn2 = Attention(dim, heads, cross_dim=cross_dim)
        self.norm3 = nn.LayerNorm(dim, eps=1e-5)
        self.ff = FeedForward(dim)

    def forward(self, x, ctx):
        x = x + self.attn1(self.norm1(x))
        x = x + self.attn2(self.norm2(x), ctx)
        x = x + self.ff(self.norm3(x))
        return x


class Transformer2DModel(nn.Module):
    """transformer_2d.py:327-347 (continuous input, use_linear_projection) and :407-423."""

    def __init__(self, dim, heads, cross_dim, groups=32, joint=False):
        super().__init__()
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        self.proj_in = nn.Linear(dim, dim)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, heads, cross_dim, joint)])
        self.proj_out = nn.Linear(dim, dim)

    def forward(self, x, ctx):
        B, C, H, W = x.shape
        res = x
        h = self.norm(x).permute(0, 2, 3, 1).reshape(B, H * W, C)
        h = self.proj_in(h)
        for blk in self.transformer_blocks:
            h = blk(h, ctx)
        h = self.proj_out(h)
        h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
        return h + res


# ----------------------------------------------------------------------------- blocks
class DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, n, heads, cross_dim, has_attn, add_down, groups, eps, joint):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(n)])
        if has_attn:
            self.attentions = nn.ModuleList(
                [Transformer2DModel(cout, heads, cross_dim, groups, joint) for _ in range(n)])
        else:
            self.attentions = None
        self.downsamplers = nn.ModuleList([Downsample2D(cout, 1)]) if add_down else None

    def forward(self, x, temb, ctx):
        outs = []
        for i, r in enumerate(self.resnets):
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class MidBlock(nn.Module):
    def __init__(self, ch, temb, heads, cross_dim, groups, eps, joint):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([Transformer2DModel(ch, heads, cross_dim, groups, joint)])

    def forward(self, x, temb, ctx):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb)


class UpBlock(nn.Module):
    def __init__(self, cin, cout, cprev, temb, n, heads, cross_dim, has_attn, add_up, groups, eps, joint):
        super().__init__()
        rs = []
        for i in range(n):
            skip = cin if i == n - 1 else cout            # unet_2d_blocks.py:2239-2240
            rin = cprev if i == 0 else cout
            rs.append(ResnetBlock2D(rin + skip, cout, temb, groups, eps))
        self.resnets = nn.ModuleList(rs)
        if has_attn:
            self.attentions = nn.ModuleList(
                [Transformer2DModel(cout, heads, cross_dim, groups, joint) for _ in range(n)])
        else:
            self.attentions = None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None

    def forward(self, x, skips, temb, ctx, upsample_size=None):
        for i, r in enumerate(self.resnets):
            x = torch.cat([x, skips.pop()], dim=1)          # unet_2d_blocks.py:2328,2456
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x, upsample_size)
        return x


class UNetOutput:
    def __init__(self, sample):
        self.sample = sample


class UNet2DConditionRef(nn.Module):
    def __init__(self, config: UNetConfig = None, **kw):
        super().__init__()
        cfg = config or UNetConfig(**kw)
        self.config = cfg
        boc = cfg.block_out_channels
        temb = boc[0] * 4
        g, eps, cd = cfg.norm_num_groups, cfg.norm_eps, cfg.cross_attention_dim
        J = cfg.joint_attention
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if cfg.class_embed_type == "projection":
            self.class_embedding = TimestepEmbedding(cfg.projection_class_embeddings_input_dim, temb)
        else:
            self.class_embedding = None
        n = cfg.layers_per_block
        downs = []
        ch = boc[0]
        for i, t in enumerate(cfg.down_block_types):
            cin, ch = ch, boc[i]
            downs.append(DownBlock(cin, ch, temb, n, cfg.attention_head_dim[i], cd,
                                   t == "CrossAttnDownBlock2D", i != len(boc) - 1, g, eps, J))
        self.down_blocks = nn.ModuleList(downs)
        self.mid_block = MidBlock(boc[-1], temb, cfg.attention_head_dim[-1], cd, g, eps, J)
        rev = list(reversed(boc))
        rheads = list(reversed(cfg.attention_head_dim))
        ups = []
        cout = rev[0]
        for i, t in enumerate(cfg.up_block_types):
            cprev, cout = cout, rev[i]
            cin = rev[min(i + 1, len(boc) - 1)]
            ups.append(UpBlock(cin, cout, cprev, temb, n + 1, rheads[i], cd,
                               t == "CrossAttnUpBlock2D", i != len(boc) - 1, g, eps, J))
        self.up_blocks = nn.ModuleList(ups)
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=eps)
        self.conv_out = nn.Conv2d(boc[0], cfg.out_channels, 3, padding=1)

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, return_dict=True):
        cfg = self.config
        B = sample.shape[0]
        n_up = len(cfg.block_out_channels) - 1
        factor = 2 ** n_up
        forward_size = any(d % factor != 0 for d in sample.shape[-2:])   # unet_2d_condition.py:920-930
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        elif timestep.dim() == 0:
            timestep = timestep[None].to(sample.device)
        t = timestep.expand(B)
        emb = timestep_embedding(t, cfg.block_out_channels[0], cfg.flip_sin_to_cos, cfg.freq_shift)
        emb = self.time_embedding(emb.to(sample.dtype))
        if self.class_embedding is not None:
            assert class_labels is not None
            emb = emb + self.class_embedding(class_labels.to(sample.dtype))  # :984-1000
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, emb, encoder_hidden_states)
            skips += outs
        x = self.mid_block(x, emb, encoder_hidden_states)
        for i, blk in enumerate(self.up_blocks):
            n = len(blk.resnets)
            mine, skips = skips[-n:], skips[:-n]
            up_size = None
            if i != len(self.up_blocks) - 1 and forward_size:
                up_size = skips[-1].shape[2:]                    # :1185-1186
            x = blk(x, list(mine), emb, encoder_hidden_states, up_size)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))
        if not return_dict:
            return (x,)
        return UNetOutput(x)


def seeded_init(module: nn.Module, seed: int = 1234, attn_gain: float = 1.5):
    """Deterministic synthetic weights (no checkpoints offline).

    PyTorch default init under a fixed seed; norm affine parameters are perturbed so the
    affine path is exercised; q/k projections of self-attention get `attn_gain` so the
    softmax is not trivially uniform: logit std ~ attn_gain**2 (1.5 -> ~2.3, the range of trained
    SD attention; 3.0 gave std ~9, a near-argmax softmax that amplifies fp16 operand rounding 50x
    and is not representative).
    """
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.named_parameters()):
            if p.dim() >= 2:
                fan_in = p[0].numel()
                bound = 1.0 / math.sqrt(fan_in) * math.sqrt(3.0)
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * bound)
                if re.search(r"(attn1|mid_block\.attentions\.0)\.to_(q|k)\.weight$", name):
                    p.mul_(attn_gain)
            else:
                is_norm_w = ("norm" in name and name.endswith("weight"))
                if is_norm_w:
                    p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
                else:
                    p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return module


def replace_unet_conv_in(unet: UNet2DConditionRef, repeat: int = 2):
    """training/util/unet_prep.py:6-21 — widen conv_in 4->8 ch, weights duplicated, weights AND bias divided by `repeat`."""
    w = unet.conv_in.weight.data.clone().repeat(1, repeat, 1, 1) / repeat
    b = unet.conv_in.bias.data.clone() / repeat          # unet_prep.py:12 scales the bias too
    new = nn.Conv2d(w.shape[1], w.shape[0], 3, padding=1)
    new.weight = nn.Parameter(w)
    new.bias = nn.Parameter(b)
    unet.conv_in = new
    if isinstance(unet.config, dict):                     # unet_prep.py:20 writes unet.config['in_channels']
        unet.config["in_channels"] = w.shape[1]
    else:                                                 # the oracle's own config is a dataclass
        unet.config.in_channels = w.shape[1]
    return unet
