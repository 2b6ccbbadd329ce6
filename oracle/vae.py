"""ORACLE (test infrastructure) — fp32 PyTorch restatement of the SD `AutoencoderKL`.

The AutoencoderKL source (diffusers 0.30.2) is NOT in the reference checkout; it is restated
per SURVEY.md App. A.6.  Block shapes follow the in-tree GeoWizard copies:
`DownEncoderBlock2D` unet_2d_blocks.py:1276-1333, `UNetMidBlock2D` :509-631 (attention
instantiated at :589-601), `UpDecoderBlock2D` :2484-2541.  Call sites:
Marigold/marigold/marigold_pipeline.py:493-494 (encoder, quant_conv) and :515-516
(post_quant_conv, decoder).  Parameter names = diffusers `state_dict` layout (App. A.8).
"""
from dataclasses import dataclass
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .unet import ResnetBlock2D, Downsample2D, Upsample2D


@dataclass
class VAEConfig:
    in_channels: int = 3
    out_channels: int = 3
    latent_channels: int = 4
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scaling_factor: float = 0.18215            # marigold_pipeline.py:134-135

    def __getitem__(self, k):
        return getattr(self, k)


def tiny_vae_config(**kw):
    base = dict(block_out_channels=(64, 64, 128, 128))
    base.update(kw)
    return VAEConfig(**base)


class VAEAttention(nn.Module):
    """Single-head attention with GroupNorm prologue, biased projections, residual (App. A.6)."""

    def __init__(self, ch, groups, eps=1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, ch, eps=eps)
        self.to_q = nn.Linear(ch, ch)
        self.to_k = nn.Linear(ch, ch)
        self.to_v = nn.Linear(ch, ch)
        self.to_out = nn.ModuleList([nn.Linear(ch, ch), nn.Dropout(0.0)])

    def forward(self, x):
        B, C, H, W = x.shape
        h = self.group_norm(x).view(B, C, H * W).transpose(1, 2)
        q, k, v = self.to_q(h), self.to_k(h), self.to_v(h)
        s = torch.matmul(q, k.transpose(-1, -2)) * (C ** -0.5)
        o = torch.matmul(torch.softmax(s, dim=-1), v)
        o = self.to_out[0](o).transpose(1, 2).reshape(B, C, H, W)
        return o + x


class VAEMidBlock(nn.Module):
    def __init__(self, ch, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, None, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([VAEAttention(ch, groups, eps)])

    def forward(self, x):
        x = self.resnets[0](x)
        x = self.attentions[0](x)
        return self.resnets[1](x)


class DownEncoderBlock(nn.Module):
    def __init__(self, cin, cout, n, add_down, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, None, groups, eps) for i in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout, padding=0)]) if add_down else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class UpDecoderBlock(nn.Module):
    def __init__(self, cin, cout, n, add_up, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, None, groups, eps) for i in range(n)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class Encoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        boc, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        blocks, ch = [], boc[0]
        for i, c in enumerate(boc):
            blocks.append(DownEncoderBlock(ch, c, cfg.layers_per_block, i != len(boc) - 1, g))
            ch = c
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = VAEMidBlock(boc[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * cfg.latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for b in self.down_blocks:
            x = b(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class Decoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        boc, g = cfg.block_out_channels, cfg.norm_num_groups
        rev = list(reversed(boc))
        self.conv_in = nn.Conv2d(cfg.latent_channels, rev[0], 3, padding=1)
        self.mid_block = VAEMidBlock(rev[0], g)
        blocks, ch = [], rev[0]
        for i, c in enumerate(rev):
            blocks.append(UpDecoderBlock(ch, c, cfg.layers_per_block + 1, i != len(boc) - 1, g))
            ch = c
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[0], cfg.out_channels, 3, padding=1)

    def forward(self, z):
        x = self.conv_in(z)
        x = self.mid_block(x)
        for b in self.up_blocks:
            x = b(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class AutoencoderKLRef(nn.Module):
    def __init__(self, config: VAEConfig = None, **kw):
        super().__init__()
        cfg = config or VAEConfig(**kw)
        self.config = cfg
        self.encoder = Encoder(cfg)
        self.decoder = Decoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)
