"""B200AutoencoderKL — drop-in for diffusers' `AutoencoderKL` as the reference uses it:
    vae.encoder(x), vae.quant_conv(h)            Marigold/marigold/marigold_pipeline.py:493-494
    vae.post_quant_conv(z), vae.decoder(z)       :515-516, :536-537
    vae.config.scaling_factor                    training/train.py:474,528
Graph per SURVEY.md App. A.6 (blocks shaped as GeoWizard/geowizard/models/unet_2d_blocks.py:
1276-1333 DownEncoderBlock2D, 509-631 UNetMidBlock2D, 2484-2541 UpDecoderBlock2D); diffusers
`state_dict` names.  All arithmetic runs in libb200_e2eft.so.
"""
import torch
import torch.nn as nn

from . import autograd_blocks as ab
from . import ops
from .modules import (ConfigDict, ConvInSmall, ConvOutSmall, Downsample2D, Packed, ResnetBlock2D,
                      Upsample2D, _f16, _f32, _view_cs)
from .checkpoint import PretrainedMixin
from .ops import F16, F32

_DEFAULTS = dict(in_channels=3, out_channels=3, latent_channels=4,
                 block_out_channels=(128, 256, 512, 512), layers_per_block=2, norm_num_groups=32,
                 scaling_factor=0.18215, sample_size=768, act_fn="silu")


# The unfused VAE attention stores S [B, L, Lp] fp32 and P fp16: 6 bytes per score.  Its GEMMs address one batch
# element of an output with 32-bit offsets (b200_linear rejects M * ldo >= 2^32 - 1; for S that is L * Lp), while batch
# offsets and the row softmax's offsets are 64-bit.  So the unfused path computes any batch size as long as one image's
# score matrix stays under 2^32 - 1 elements, and that bound (not B * L * Lp) is where the fused kernel must take over:
# every shape the unfused path can compute keeps it, bit for bit.
UNFUSED_MAX_SCORES = 0xFFFFFFFF


def use_fused_attention(B, L, ch, memory_efficient=False):
    """Which path `VAEAttention.run` takes for B images of L = H*W tokens and `ch` channels: the d=512 flash kernel
    (True) when memory-efficient attention is switched on or when the unfused path cannot index one image's scores;
    otherwise the unfused GEMM + row-softmax path.  The flash kernel exists for 512 channels only (every reference
    VAE); other widths always run unfused.  B does not enter: batch offsets are 64-bit on both paths."""
    if ch != 512:
        return False
    Lp = (L + 7) // 8 * 8
    return bool(memory_efficient) or L * Lp >= UNFUSED_MAX_SCORES


class VAEAttention(nn.Module):
    """Single-head mid-block attention (d = channels, 512 for SD): GN -> q,k,v Linear(+bias) ->
    softmax(QK^T/sqrt(C)) V -> out Linear -> + residual  (instantiated as unet_2d_blocks.py:589-601).
    Two paths (`use_fused_attention` picks one):
      unfused (default): S = QK^T (fp32), row softmax, O = P V^T^T on the wgmma GEMM; V^T comes directly out of a
        swapped-operand GEMM (bias along rows), so no transpose kernel is needed.  Needs 6 B per score (L^2 memory).
      fused (`memory_efficient`, or L too large for the unfused path): one [B*L, 3C] QKV GEMM, the d=512 flash kernel
        reading Q, K, V in place from it, then the same out-projection.  O(L) memory, in training too: the backward
        (autograd_blocks._VAEAttentionFn) recomputes P from the saved log-sum-exp in the fused d=512 backward kernels.
    Training takes the path inference takes (same rule, same forward), so both give the same bits."""

    def __init__(self, ch, groups, eps=1e-6):
        super().__init__()
        self.ch, self.groups, self.eps = ch, groups, eps
        self.group_norm = nn.GroupNorm(groups, ch, eps=eps)
        self.to_q = nn.Linear(ch, ch)
        self.to_k = nn.Linear(ch, ch)
        self.to_v = nn.Linear(ch, ch)
        self.to_out = nn.ModuleList([nn.Linear(ch, ch), nn.Dropout(0.0)])
        self._pk = Packed()
        self.memory_efficient = False       # B200AutoencoderKL.enable_xformers_memory_efficient_attention

    def _packed(self):
        return self._pk.get(list(self.parameters()), lambda: dict(
            g=_f32(self.group_norm.weight), b=_f32(self.group_norm.bias),
            wqk=_f16(torch.cat([self.to_q.weight, self.to_k.weight], 0)),
            bqk=_f32(torch.cat([self.to_q.bias, self.to_k.bias], 0)),
            wv=_f16(self.to_v.weight), bv=_f32(self.to_v.bias),
            wqkv=_f16(torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight], 0)),
            bqkv=_f32(torch.cat([self.to_q.bias, self.to_k.bias, self.to_v.bias], 0)),
            wo=_f16(self.to_out[0].weight), bo=_f32(self.to_out[0].bias)))

    def run(self, x, sdt=F32):
        B, H, W, C = x.shape
        if use_fused_attention(B, H * W, C, self.memory_efficient):
            return self.forward_fused(x, sdt)[0]
        return self.forward_unfused(x, sdt)[0]

    def forward_fused(self, x, sdt=F32, want_lse=False):
        """The fused path, also returning the intermediates its backward reads: (out, (hn, qkv, o, lse)); lse (the
        kernel's log2-domain log-sum-exp, [B, L] fp32) only with `want_lse`, else None.  Out is the same either way."""
        pk = self._packed()
        B, H, W, C = x.shape
        L = H * W
        hn = ops.group_norm(x, pk["g"], pk["b"], self.eps, self.groups, False).view(B * L, C)
        qkv = ops.linear(hn, pk["wqkv"], pk["bqkv"]).view(B, L, 3 * C)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        if want_lse:
            o, lse = ops.attention_d512(q, k, v, C ** -0.5, want_lse=True)                  # [B, L, C], [B, L]
        else:
            o, lse = ops.attention_d512(q, k, v, C ** -0.5), None
        out = ops.linear(o.view(B * L, C), pk["wo"], pk["bo"], residual=x.view(B * L, C), out_dtype=sdt,
                         stats_rows_per_img=L)
        return _view_cs(out, B, H, W, C), (hn, qkv, o, lse)

    def forward_unfused(self, x, sdt=F32):
        """The unfused path, also returning the intermediates its backward reads: (out, (hn, qk, p_buf, o))."""
        pk = self._packed()
        B, H, W, C = x.shape
        L = H * W
        Lp = (L + 7) // 8 * 8                       # leading dims must be multiples of 8 elements
        hn = ops.group_norm(x, pk["g"], pk["b"], self.eps, self.groups, False).view(B, L, C)
        qk = ops.linear(hn.view(B * L, C), pk["wqk"], pk["bqk"]).view(B, L, 2 * C)
        vt_buf = torch.empty((B, C, Lp), dtype=F16, device=x.device)
        vt = ops.linear(pk["wv"], hn, pk["bv"], bias_row=True, out=vt_buf[:, :, :L])        # V^T [B, C, L]
        s_buf = torch.empty((B, L, Lp), dtype=F32, device=x.device)
        ops.linear(qk[..., :C], qk[..., C:], out=s_buf[:, :, :L])                           # S [B, L, L] fp32
        p_buf = ops.softmax_rows(s_buf, C ** -0.5, cols=L)
        o = ops.linear(p_buf[:, :, :L], vt)                                                 # [B, L, C]
        out = ops.linear(o.view(B * L, C), pk["wo"], pk["bo"], residual=x.view(B * L, C), out_dtype=sdt,
                         stats_rows_per_img=L)
        return _view_cs(out, B, H, W, C), (hn, qk, p_buf, o)


class _MidBlock(nn.Module):
    def __init__(self, ch, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, None, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([VAEAttention(ch, groups, eps)])

    def run(self, x, resnet, attention):
        """resnet(block, x) / attention(block, x): the inference or the differentiable step of each block."""
        x = resnet(self.resnets[0], x)
        x = attention(self.attentions[0], x)
        return resnet(self.resnets[1], x)


class _DownEncoderBlock(nn.Module):
    def __init__(self, cin, cout, n, add_down, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, None, groups, eps) for i in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout, padding=0)]) if add_down else None


class _UpDecoderBlock(nn.Module):
    def __init__(self, cin, cout, n, add_up, groups, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, None, groups, eps) for i in range(n)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None


def _check_input(x, who):
    ops._need_cuda(x)                                  # sm_90a only, no CPU fallback
    if torch.is_grad_enabled() and x.requires_grad:
        raise NotImplementedError(f"backward through {who} is not implemented yet; wrap in torch.no_grad()")


class Encoder(nn.Module):
    """NCHW image in [-1,1] -> NCHW moments [B, 2*latent, H/8, W/8] (before quant_conv)."""

    def __init__(self, cfg, stream_dtype):
        super().__init__()
        boc, g = tuple(cfg["block_out_channels"]), cfg["norm_num_groups"]
        self.stream_dtype = stream_dtype
        self.conv_in = nn.Conv2d(cfg["in_channels"], boc[0], 3, padding=1)
        blocks, ch = [], boc[0]
        for i, c in enumerate(boc):
            blocks.append(_DownEncoderBlock(ch, c, cfg["layers_per_block"], i != len(boc) - 1, g))
            ch = c
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _MidBlock(boc[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * cfg["latent_channels"], 3, padding=1)
        self._in = ConvInSmall(self.conv_in)
        self._out = ConvOutSmall(self.conv_norm_out, self.conv_out)

    def forward(self, x):
        _check_input(x, "B200AutoencoderKL.encoder")
        sdt = self.stream_dtype
        h = self._in.run(x if x.dtype in (F16, F32) else x.float(), sdt)
        resnet = lambda r, h, f16_copy=False: r.run(h, None, None, sdt, f16_copy)         # noqa: E731
        for blk in self.down_blocks:
            for i, r in enumerate(blk.resnets):
                h = resnet(r, h, i == len(blk.resnets) - 1 and blk.downsamplers is not None)
            if blk.downsamplers is not None:
                h = blk.downsamplers[0].run(h, sdt)
        h = self.mid_block.run(h, resnet, lambda m, h: m.run(h, sdt))
        out = self._out.run(h)
        return out if out.dtype == x.dtype else out.to(x.dtype)


class Decoder(nn.Module):
    """NCHW latent (after post_quant_conv) -> NCHW image [B, 3, 8H, 8W]."""

    def __init__(self, cfg, stream_dtype):
        super().__init__()
        boc, g = tuple(cfg["block_out_channels"]), cfg["norm_num_groups"]
        rev = list(reversed(boc))
        self.stream_dtype = stream_dtype
        self.conv_in = nn.Conv2d(cfg["latent_channels"], rev[0], 3, padding=1)
        self.mid_block = _MidBlock(rev[0], g)
        blocks, ch = [], rev[0]
        for i, c in enumerate(rev):
            blocks.append(_UpDecoderBlock(ch, c, cfg["layers_per_block"] + 1, i != len(boc) - 1, g))
            ch = c
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[0], cfg["out_channels"], 3, padding=1)
        self._in = ConvInSmall(self.conv_in)
        self._out = ConvOutSmall(self.conv_norm_out, self.conv_out)
        self.gradient_checkpointing = False            # B200AutoencoderKL.enable_gradient_checkpointing

    def forward(self, z):
        """With grad enabled and `z.requires_grad` every block runs as its autograd Function (autograd_blocks.py);
        the VAE is frozen in training (training/train.py:323-326), so only the data gradient is produced."""
        ops._need_cuda(z)                                  # sm_90a only, no CPU fallback
        sdt = self.stream_dtype
        zin = z if z.dtype in (F16, F32) else z.float()
        train = torch.is_grad_enabled() and z.requires_grad
        if train:
            if sdt != F32:
                raise NotImplementedError("training runs with the fp32 residual stream (stream_dtype=torch.float32)")
            h = ab.conv_in(self._in, zin)
            # gradient checkpointing: the resnets and the attention block keep only their inputs.  An upsampler's
            # backward reads nothing but the fp16 copy of its input that its input carries anyway, so it keeps that.
            ck = bool(self.gradient_checkpointing)
            resnet = lambda r, h, f16_copy=False: ab.resnet(r, h, f16_copy=f16_copy, ckpt=ck)  # noqa: E731
            attention = lambda m, h: ab.vae_attention(m, h, ckpt=ck)                          # noqa: E731
            upsample = ab.upsample
        else:
            h = self._in.run(zin, sdt)
            resnet = lambda r, h, f16_copy=False: r.run(h, None, None, sdt, f16_copy)     # noqa: E731
            attention = lambda m, h: m.run(h, sdt)                                         # noqa: E731
            upsample = lambda m, h: m.run(h, None, sdt)                                    # noqa: E731
        h = self.mid_block.run(h, resnet, attention)
        for blk in self.up_blocks:
            for i, r in enumerate(blk.resnets):
                h = resnet(r, h, i == len(blk.resnets) - 1 and blk.upsamplers is not None)
            if blk.upsamplers is not None:
                h = upsample(blk.upsamplers[0], h)
        out = ab.conv_out(self._out, h) if train else self._out.run(h)
        return out if out.dtype == z.dtype else out.to(z.dtype)


class Conv1x1Small(nn.Conv2d):
    """quant_conv / post_quant_conv (1x1 on <= 8 channels, NCHW): one pointwise kernel."""

    def forward(self, x, scale_in=1.0, x2=None, scale_in2=0.0, rows=None, scale_out=1.0):
        _check_input(x, "B200AutoencoderKL.(post_)quant_conv")
        # the (row-sliced, pre-scaled) fp32 matrix is derived once per weights version, not per call
        cache = self.__dict__.setdefault("_wb_cache", {})
        pk = cache.setdefault((rows, float(scale_out)), Packed())

        def build():
            w = self.weight.detach().reshape(self.out_channels, self.in_channels).to(F32)
            b = self.bias.detach().to(F32)
            if rows is not None:
                w, b = w[:rows], b[:rows]
            if scale_out != 1.0:
                w, b = w * scale_out, b * scale_out
            return w.contiguous(), b.contiguous()
        w, b = pk.get([self.weight, self.bias], build)
        xin = x if x.dtype == F32 else x.float()
        x2in = None if x2 is None else (x2 if x2.dtype == F32 else x2.float())
        out = ops.pointwise_nchw(xin.contiguous(), scale_in, w, b,
                                 in2=None if x2in is None else x2in.contiguous(), a2=scale_in2,
                                 cin=self.in_channels)
        return out if out.dtype == x.dtype else out.to(x.dtype)


class B200AutoencoderKL(PretrainedMixin, nn.Module):
    _diffusers_class_name = "AutoencoderKL"
    _config_defaults = _DEFAULTS

    def __init__(self, stream_dtype=torch.float32, **config):
        super().__init__()
        cfg = ConfigDict(_DEFAULTS)
        unknown = set(config) - set(_DEFAULTS)
        if unknown:
            raise TypeError(f"unknown VAE config keys: {sorted(unknown)}")
        cfg.update(config)
        self.config = cfg
        self.encoder = Encoder(cfg, stream_dtype)
        self.decoder = Decoder(cfg, stream_dtype)
        lc = cfg["latent_channels"]
        self.quant_conv = Conv1x1Small(2 * lc, 2 * lc, 1)
        self.post_quant_conv = Conv1x1Small(lc, lc, 1)

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def register_to_config(self, **kw):
        self.config.update({k: v for k, v in kw.items() if k in _DEFAULTS})

    # ---- diffusers' memory-efficient attention switch (Marigold/run.py:285)
    def enable_xformers_memory_efficient_attention(self, attention_op=None):
        """Run both mid-block attentions (encoder and decoder) on the d=512 flash kernel, which never stores the
        L x L score matrix: what makes native-resolution (`processing_res=0`) inference on large photos fit.
        `attention_op` (an xformers operator in diffusers) is accepted and ignored: there is one kernel."""
        self._set_memory_efficient_attention(True)

    def disable_xformers_memory_efficient_attention(self):
        """Back to the default: the unfused path wherever it can index the scores (see `use_fused_attention`)."""
        self._set_memory_efficient_attention(False)

    def _set_memory_efficient_attention(self, on):
        for m in self.modules():
            if isinstance(m, VAEAttention):
                m.memory_efficient = bool(on)

    @property
    def memory_efficient_attention(self):
        return any(m.memory_efficient for m in self.modules() if isinstance(m, VAEAttention))

    # ---- diffusers' gradient checkpointing switch (ModelMixin.enable_gradient_checkpointing)
    def enable_gradient_checkpointing(self):
        """Checkpoint the decoder's blocks: a training forward then keeps only the input of every ResnetBlock2D and of
        the mid-block attention, and each block re-runs its training forward at the start of its backward, so the
        decoder's backward needs the block inputs plus one block's intermediates.  The recompute reproduces the saved
        intermediates bit for bit in practice.  The same kernels run on the same inputs; only the fp64-atomic GroupNorm
        statistics could round differently.  So the gradients are the plain backward's, bit for bit where that backward
        reproduces itself; its fp32-atomic sums vary in the last bits run to run.  Per block,
        not per diffusers segment (mid-block, each up block): at 768 x 768, bs 2 it peaks lower (DESIGN.md §7).  As in
        current diffusers it applies whenever grad is enabled, also to a frozen VAE in eval mode (the E2E recipes).
        The encoder has no backward (it runs under no_grad in training), so it has nothing to checkpoint."""
        self.decoder.gradient_checkpointing = True

    def disable_gradient_checkpointing(self):
        self.decoder.gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self):
        return any(getattr(m, "gradient_checkpointing", False) for m in self.modules())

    # ---- fused conveniences used by the engine's own pipelines (same math as the call sites above)
    def encode_scaled_mean(self, rgb):
        """`encode_rgb` of marigold_pipeline.py:481-498: quant_conv -> mean half -> * scaling_factor."""
        h = self.encoder(rgb)
        return self.quant_conv(h, rows=self.config["latent_channels"], scale_out=self.config["scaling_factor"])

    def decode_from_prediction(self, model_out, c_out, noisy=None, c_noisy=0.0):
        """x0 = c_noisy*noisy + c_out*model_out (scheduler closed form), / scaling_factor,
        post_quant_conv, decoder  (marigold_pipeline.py:457-465, 513-516)."""
        s = 1.0 / self.config["scaling_factor"]
        if torch.is_grad_enabled() and model_out.requires_grad:
            if noisy is None or c_noisy == 0.0:
                return self.decoder(ab.pointwise(self.post_quant_conv, model_out, c_out * s))
            # noisy-start E2E fine-tuning: c_noisy * x_t is a constant addend, so the backward is unchanged
            return self.decoder(ab.pointwise(self.post_quant_conv, model_out, c_out * s, noisy, c_noisy * s))
        z = self.post_quant_conv(model_out, scale_in=c_out * s, x2=noisy, scale_in2=c_noisy * s)
        return self.decoder(z)
