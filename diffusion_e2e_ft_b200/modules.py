"""Building blocks of the engine: diffusers-named parameter containers whose forward runs the
sm_90a kernels of libb200_e2eft.so (via ops.py) on NHWC activations.

Layout / precision contract inside the engine
  * activations are NHWC; GEMM/conv operands are fp16; accumulation fp32;
  * the residual stream (`sdt`) is fp32 (parity mode, default) or fp16 (fast mode);
  * GroupNorm / LayerNorm statistics and softmax are fp32.

Each block mirrors one diffusers/GeoWizard class (cited per class) and keeps its `state_dict`
names, so reference checkpoints load unchanged (SURVEY.md App. A.8).  Packed fp16 weights are
derived lazily from the fp32 master parameters and re-derived whenever a parameter changes
(`_version` / storage pointer), so optimizers and `load_state_dict` just work.
"""
import torch
import torch.nn as nn

from . import ops
from .ops import F16, F32


class ConfigDict(dict):
    """dict with attribute access — the reference reads both `unet.config.x` and `unet.config['x']`
    (training/train.py:299, training/util/unet_prep.py:20)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


_WEIGHTS_EPOCH = [0]


def bump_weights_epoch():
    """Invalidate every packed-weight cache: called after an optimizer kernel has updated the parameters through
    their flat buffer (a raw device write that torch's per-tensor version counters do not see)."""
    _WEIGHTS_EPOCH[0] += 1


class Packed:
    """Cache of derived (packed fp16 / fp32-contiguous) tensors keyed on parameter identity+version."""

    def __init__(self):
        self._key = None
        self._val = None

    def get(self, params, build):
        key = (_WEIGHTS_EPOCH[0],) + tuple((p.data_ptr(), p._version, p.device, p.dtype) for p in params)
        if key != self._key:
            with torch.no_grad():
                self._val = build()
            self._key = key
        return self._val


def _view_cs(t, *shape):
    """view() that keeps the producer-attached extras: fused GroupNorm channel sums (`._cs`) and the fp16
    twin (`._h16`)."""
    v = t.view(*shape)
    cs = getattr(t, "_cs", None)
    if cs is not None:
        v._cs = cs
    h = getattr(t, "_h16", None)
    if h is not None:
        v._h16 = h.view(*shape)
    return v


def _f32(p):
    return p.detach().to(F32).contiguous()


def _f16(p):
    return p.detach().to(F16).contiguous()


# ------------------------------------------------------------------------------------ resnet
class ResnetBlock2D(nn.Module):
    """diffusers ResnetBlock2D (SURVEY.md App. A.2): GN+SiLU -> conv3x3 (+temb) -> GN+SiLU ->
    conv3x3 (+1x1 shortcut fused as extra K columns) + residual.  Instantiated by the reference at
    GeoWizard/geowizard/models/unet_2d_blocks.py:1064-1076, 2242-2254, 667-679."""

    def __init__(self, cin, cout, temb_channels=1280, groups=32, eps=1e-5):
        super().__init__()
        self.cin, self.cout, self.groups, self.eps = cin, cout, groups, eps
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, cout) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self._pk = Packed()

    def _packed(self):
        ps = [p for p in self.parameters()]

        def build():
            d = dict(g1=_f32(self.norm1.weight), b1=_f32(self.norm1.bias),
                     g2=_f32(self.norm2.weight), b2=_f32(self.norm2.bias),
                     w1=ops.pack_conv(self.conv1.weight), c1b=_f32(self.conv1.bias))
            if self.conv_shortcut is not None:
                d["w2"] = ops.pack_conv(self.conv2.weight, self.conv_shortcut.weight)
                d["c2b"] = _f32(self.conv2.bias + self.conv_shortcut.bias)
            else:
                d["w2"] = ops.pack_conv(self.conv2.weight)
                d["c2b"] = _f32(self.conv2.bias)
            return d
        return self._pk.get(ps, build)

    def run(self, x, temb=None, skip=None, sdt=F32, f16_copy=False):
        """x (and optional skip, channel-concatenated after x): stream NHWC; temb: fp32 [B,cout] view.
        `f16_copy`: the output also gets an fp16 twin (the next op is a stride-2 / upsample conv)."""
        return self.forward_saved(x, temb, skip, sdt, f16_copy)[0]

    def forward_saved(self, x, temb=None, skip=None, sdt=F32, f16_copy=False):
        """`run`, also returning the intermediates its backward reads: (out, (a1, raw, h, a2))."""
        pk = self._packed()
        if self.conv_shortcut is not None and (skip is not None or x.dtype != F16):
            # the 1x1 shortcut needs the (concatenated) input as an fp16 operand: emitted by the GN pass
            a1, raw = ops.group_norm(x, pk["g1"], pk["b1"], self.eps, self.groups, True, x2=skip, want_raw=True)
        else:
            assert skip is None
            a1 = ops.group_norm(x, pk["g1"], pk["b1"], self.eps, self.groups, True)
            raw = x if self.conv_shortcut is not None else None     # fp16 stream: x itself is the operand
        h = ops.conv2d(a1, pk["w1"], self.cout, bias=pk["c1b"], rowvec=temb, stats=True)
        a2 = ops.group_norm(h, pk["g2"], pk["b2"], self.eps, self.groups, True)
        if raw is not None:
            out = ops.conv2d(a2, pk["w2"], self.cout, bias=pk["c2b"], x2=raw, out_dtype=sdt, stats=True,
                             f16_copy=f16_copy)
        else:
            out = ops.conv2d(a2, pk["w2"], self.cout, bias=pk["c2b"], residual=x, out_dtype=sdt, stats=True,
                             f16_copy=f16_copy)
        return out, (a1, raw, h, a2)


class Downsample2D(nn.Module):
    """diffusers Downsample2D (App. A.4): stride-2 conv, pad 1 (UNet) or (0,1,0,1) (VAE encoder)."""

    def __init__(self, ch, padding=1):
        super().__init__()
        self.ch, self.padding = ch, padding
        self.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=padding)
        self._pk = Packed()

    def _packed(self):
        return self._pk.get(list(self.parameters()),
                            lambda: dict(w=ops.pack_conv(self.conv.weight), b=_f32(self.conv.bias)))

    def run(self, x, sdt=F32):
        return self.forward_saved(x, sdt)[0]

    def forward_saved(self, x, sdt=F32):
        """`run`, also returning the fp16 conv operand its weight gradient reads: (out, x16)."""
        pk = self._packed()
        NB, H, W, C = x.shape
        if self.padding == 1:
            taps, Ho, Wo = ops.TAPS3, (H - 1) // 2 + 1, (W - 1) // 2 + 1
        else:
            taps, Ho, Wo = ops.TAPS3_PAD0, (H - 2) // 2 + 1, (W - 2) // 2 + 1
        x16 = x if x.dtype == F16 else ops.cast_f16(x)
        out = ops.conv2d(x16, pk["w"], C, bias=pk["b"], taps=taps, stride=2, out_hw=(Ho, Wo), out_dtype=sdt,
                         stats=True)
        return out, x16


class Upsample2D(nn.Module):
    """diffusers Upsample2D: nearest x2 (or explicit size, unet_2d_condition.py:1185-1186) + conv3x3."""

    def __init__(self, ch):
        super().__init__()
        self.ch = ch
        self.conv = nn.Conv2d(ch, ch, 3, padding=1)
        self._pk = Packed()
        self._pk2 = Packed()

    # exact 2x nearest upsample followed by a 3x3 conv == four 2x2 convs on the low-res input, one per output
    # parity (py, px): output row 2i+py reads upsampled rows 2i+py-1..2i+py+1, i.e. low-res rows
    #   py=0: {i-1: W[0], i: W[1]+W[2]}     py=1: {i: W[0]+W[1], i+1: W[2]}       (same along x)
    # 2.25x fewer MACs than convolving the 4x larger tensor, and the upsampled tensor is never written.
    _PHASE = {0: ((-1, (0,)), (0, (1, 2))), 1: ((0, (0, 1)), (1, (2,)))}

    def _pack_phases(self):
        w = self.conv.weight.detach().float()
        out = {}
        for py in (0, 1):
            for px in (0, 1):
                taps, mats = [], []
                for dy, kys in self._PHASE[py]:
                    for dx, kxs in self._PHASE[px]:
                        taps.append((dy, dx))
                        mats.append(sum(w[:, :, ky, kx] for ky in kys for kx in kxs))
                wp = torch.stack(mats, dim=1).reshape(w.shape[0], -1).to(F16).contiguous()   # [Cout, 4*Cin]
                out[(py, px)] = (taps, wp)
        return out

    def _packed_phases(self):
        return self._pk.get(list(self.parameters()), lambda: dict(ph=self._pack_phases(), b=_f32(self.conv.bias)))

    def _packed_resize(self):
        return self._pk2.get(list(self.parameters()),
                             lambda: dict(w=ops.pack_conv(self.conv.weight), b=_f32(self.conv.bias)))

    @staticmethod
    def resizes(x, out_hw):
        """True when `out_hw` is not the exact 2x of x: nearest resize to out_hw, then a plain conv3x3."""
        return out_hw is not None and tuple(out_hw) != (2 * x.shape[1], 2 * x.shape[2])

    def run(self, x, out_hw=None, sdt=F32):
        return self.forward_saved(x, out_hw, sdt)[0]

    def forward_saved(self, x, out_hw=None, sdt=F32):
        """`run`, also returning the fp16 conv operand its weight gradient reads: (out, x16) for the exact 2x,
        (out, resized input) otherwise."""
        NB, H, W, C = x.shape
        if not self.resizes(x, out_hw):
            pk = self._packed_phases()
            x16 = x if x.dtype == F16 else ops.cast_f16(x)
            out = torch.empty((NB, 2 * H, 2 * W, C), dtype=sdt, device=x.device)
            cs = ops._new_stats(NB, C, x.device) if ops.FUSE_GN_STATS else None
            for (py, px), (taps, wp) in pk["ph"].items():
                ops.conv2d(x16, wp, C, bias=pk["b"], taps=taps, out_hw=(H, W), out=out, out_mul=2, out_off=(py, px),
                           stats=cs)
            return out, x16
        pk = self._packed_resize()
        up = ops.upsample_nearest(x, out_hw)
        return ops.conv2d(up, pk["w"], C, bias=pk["b"], out_dtype=sdt, stats=True), up


# ------------------------------------------------------------------------------------ attention
class Attention(nn.Module):
    """Parameter container for diffusers `Attention` (to_q/to_k/to_v/to_out.0); the math runs in
    BasicTransformerBlock.run so projections can be fused (QKV in one GEMM)."""

    def __init__(self, dim, cross_dim=None, bias=False):
        super().__init__()
        self.to_q = nn.Linear(dim, dim, bias=bias)
        self.to_k = nn.Linear(cross_dim or dim, dim, bias=bias)
        self.to_v = nn.Linear(cross_dim or dim, dim, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim), nn.Dropout(0.0)])


class GEGLU(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner * 2)


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class BasicTransformerBlock(nn.Module):
    """GeoWizard/geowizard/models/attention.py:292-413: LN -> self-attn -> LN -> cross-attn -> LN ->
    GEGLU FF, each with residual.  `joint=True` = XFormersJointAttnProcessor (attention.py:430-513)."""

    def __init__(self, dim, heads, cross_dim, joint=False):
        super().__init__()
        if dim % heads or dim // heads not in ops.HEAD_DIMS:
            raise NotImplementedError(f"{dim} channels over {heads} heads is head width {dim / heads:g}; the engine's "
                                      f"attention kernel supports head widths {ops.HEAD_DIMS}")
        self.dim, self.heads, self.head_dim, self.joint = dim, heads, dim // heads, joint
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        self.attn1 = Attention(dim)
        self.norm2 = nn.LayerNorm(dim, eps=1e-5)
        self.attn2 = Attention(dim, cross_dim=cross_dim)
        self.norm3 = nn.LayerNorm(dim, eps=1e-5)
        self.ff = FeedForward(dim)
        self._pk = Packed()
        self._pk_ctx = Packed()

    # Exact single-step specialisation (SURVEY.md §8 f1): when every image attends to the SAME context tokens
    # (marigold_pipeline.py:428-432 repeats one [1,2,1024] empty-text embedding over the batch) the keys / values are
    # constants of (weights, context), so  softmax(q K^T) V W_o^T  with q = LN(h) W_q^T  collapses to two skinny GEMMs
    #     logits = LN(h) . A^T,   A[h*S+s] = scale * W_q[head h]^T k_{h,s}            [heads*S, C]
    #     out    = P . VW,        VW[h*S+s] = W_o[:, head h] v_{h,s}                   [heads*S, C]
    # instead of a C x C query GEMM, a 128-wide flash tile over 2 keys and a C x C output GEMM.  A and VW are folded
    # in fp32 once per (weights, context) and cached.
    CONST_CTX_MAX_J = 64

    def _packed_const_ctx(self, ctx1):
        """ctx1: [S, Dctx] (any float dtype) -> dict(a16 [Jp, C], vwt16 [C, Jp], J, Jp, S)."""
        a2 = self.attn2
        params = [a2.to_q.weight, a2.to_k.weight, a2.to_v.weight, a2.to_out[0].weight, ctx1]

        def build():
            C, heads, D = self.dim, self.heads, self.head_dim
            S = ctx1.shape[0]
            J = heads * S
            Jp = (J + 7) // 8 * 8
            c = ctx1.detach().to(F32)
            k = (c @ a2.to_k.weight.detach().to(F32).t()).view(S, heads, D)            # [S, heads, D]
            v = (c @ a2.to_v.weight.detach().to(F32).t()).view(S, heads, D)
            wq = a2.to_q.weight.detach().to(F32).view(heads, D, C)                     # rows of W_q per head
            wo = a2.to_out[0].weight.detach().to(F32).view(C, heads, D)                # columns of W_o per head
            A = torch.einsum("shd,hdc->hsc", k, wq).reshape(J, C) * (D ** -0.5)
            VW = torch.einsum("shd,chd->hsc", v, wo).reshape(J, C)
            a16 = torch.zeros((Jp, C), dtype=F16, device=c.device)
            a16[:J] = A.to(F16)
            vwt16 = torch.zeros((C, Jp), dtype=F16, device=c.device)
            vwt16[:, :J] = VW.t().to(F16)
            return dict(a16=a16, vwt16=vwt16, J=J, Jp=Jp, S=S, ctx_ref=ctx1)   # ctx_ref pins the storage the key names
        return self._pk_ctx.get(params, build)

    def _packed(self):
        def build():
            a1, a2 = self.attn1, self.attn2
            pw, pb = self.ff.net[0].proj.weight, self.ff.net[0].proj.bias
            half = pw.shape[0] // 2
            return dict(
                ln=[(_f32(n.weight), _f32(n.bias)) for n in (self.norm1, self.norm2, self.norm3)],
                wqkv=_f16(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], 0)),
                wo1=_f16(a1.to_out[0].weight), bo1=_f32(a1.to_out[0].bias),
                wq2=_f16(a2.to_q.weight), wkv2=_f16(torch.cat([a2.to_k.weight, a2.to_v.weight], 0)),
                wo2=_f16(a2.to_out[0].weight), bo2=_f32(a2.to_out[0].bias),
                wv=_f16(pw[:half]), bv=_f32(pb[:half]), wgt=_f16(pw[half:]), bgt=_f32(pb[half:]),
                wf=_f16(self.ff.net[2].weight), bf=_f32(self.ff.net[2].bias))
        return self._pk.get(list(self.parameters()), build)

    def forward_saved(self, h0, B, L, ctx16, sdt=F32, const_ctx=None, save=True):
        """h0: stream [B*L, C]; ctx16: fp16 [B, S, Dctx]; const_ctx: [S, Dctx] when all images share one context.
        Returns (out, saved): `saved` holds the intermediates the backward reads, None unless `save`."""
        assert not (save and const_ctx is not None), "the backward exists for the general cross-attention path only"
        pk = self._packed()
        C, heads = self.dim, self.heads
        scale = self.head_dim ** -0.5
        n1 = ops.layer_norm(h0, *pk["ln"][0])
        qkv = ops.linear(n1, pk["wqkv"]).view(B, L, 3 * C)
        o = ops.attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, scale,
                              kv_segments=2 if self.joint else 1)
        h1 = ops.linear(o.view(B * L, C), pk["wo1"], pk["bo1"], residual=h0, out_dtype=sdt)
        n2 = ops.layer_norm(h1, *pk["ln"][1])
        S = ctx16.shape[1]
        if const_ctx is not None and heads * S <= self.CONST_CTX_MAX_J:
            cc = self._packed_const_ctx(const_ctx)
            lg = ops.linear(n2, cc["a16"], out_dtype=F32)                              # [B*L, Jp] scaled logits
            p2 = ops.softmax_groups(lg, heads, S, cc["Jp"])
            h2 = ops.linear(p2, cc["vwt16"], pk["bo2"], residual=h1, out_dtype=sdt)
        else:
            q2 = ops.linear(n2, pk["wq2"]).view(B, L, C)
            c2d = ctx16.reshape(B * S, -1)
            kv = ops.linear(c2d, pk["wkv2"]).view(B, S, 2 * C)
            o2 = ops.attention(q2, kv[..., :C], kv[..., C:], heads, scale)
            h2 = ops.linear(o2.view(B * L, C), pk["wo2"], pk["bo2"], residual=h1, out_dtype=sdt)
        saved = (n1, qkv, o, h1, n2, q2, c2d, kv, o2) if save else None
        del h1                          # without `save`, the feed-forward below runs with h1 already freed
        n3 = ops.layer_norm(h2, *pk["ln"][2])
        # GEGLU (attention.py:754-755) as two swapped-operand GEMMs: gate = gelu(x Wg + bg), then
        # value = (x Wv + bv) * gate in the second epilogue (the fused single-GEMM variant is barrier-bound)
        gate = ops.linear(n3, pk["wgt"], pk["bgt"], act=ops.ACT_GELU)
        g = ops.linear(n3, pk["wv"], pk["bv"], residual=gate, res_mul=True)
        out = ops.linear(g, pk["wf"], pk["bf"], residual=h2, out_dtype=sdt, f16_copy=True)   # proj_out operand
        return out, None if saved is None else (*saved, h2, n3, g)


class Transformer2DModel(nn.Module):
    """GeoWizard/geowizard/models/transformer_2d.py:327-347,407-423 (continuous input): GN -> proj_in -> blocks ->
    proj_out -> + residual.  `use_linear_projection` (SD-2, Marigold) makes the projections nn.Linear; otherwise
    (SD-1, GeoWizard) they are 1x1 nn.Conv2d with [C, C, 1, 1] weights (transformer_2d.py:152-155,214-217).  On NHWC
    activations a 1x1 conv is the same [B*L, C] x [C, C]^T GEMM, so both run the same packed fp16 [C, C] weight."""

    def __init__(self, dim, heads, cross_dim, groups=32, joint=False, use_linear_projection=True):
        super().__init__()
        self.dim, self.groups = dim, groups
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        self.proj_in = nn.Linear(dim, dim) if use_linear_projection else nn.Conv2d(dim, dim, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, heads, cross_dim, joint)])
        self.proj_out = nn.Linear(dim, dim) if use_linear_projection else nn.Conv2d(dim, dim, 1)
        self._pk = Packed()

    def _packed(self):
        own = [self.norm.weight, self.norm.bias, self.proj_in.weight, self.proj_in.bias,
               self.proj_out.weight, self.proj_out.bias]
        C = self.dim
        return self._pk.get(own, lambda: dict(g=_f32(self.norm.weight), b=_f32(self.norm.bias),
                                              wi=_f16(self.proj_in.weight.reshape(C, C)), bi=_f32(self.proj_in.bias),
                                              wo=_f16(self.proj_out.weight.reshape(C, C)), bo=_f32(self.proj_out.bias)))

    def run(self, x, ctx16, sdt=F32, f16_copy=False, const_ctx=None):
        return self.forward_saved(x, ctx16, sdt, f16_copy, const_ctx, save=False)[0]

    def forward_saved(self, x, ctx16, sdt=F32, f16_copy=False, const_ctx=None, save=True):
        """`run`, also returning the intermediates its backward reads: (out, (hn, h0, block saved, h16))."""
        pk = self._packed()
        (blk,) = self.transformer_blocks
        B, H, W, C = x.shape
        L = H * W
        hn = ops.group_norm(x, pk["g"], pk["b"], 1e-6, self.groups, False)
        h0 = ops.linear(hn.view(B * L, C), pk["wi"], pk["bi"], out_dtype=sdt)
        h, saved = blk.forward_saved(h0, B, L, ctx16, sdt, const_ctx, save)
        h16 = h if h.dtype == F16 else ops.cast_f16(h)
        out = ops.linear(h16, pk["wo"], pk["bo"], residual=x.view(B * L, C), out_dtype=sdt, stats_rows_per_img=L,
                         f16_copy=f16_copy)
        return _view_cs(out, B, H, W, C), (hn, h0, saved, h16)


# ------------------------------------------------------------------------------------ small-Cin conv
class ConvInSmall:
    """Helper for conv_in layers with Cin in {3,4,8}: im2col kernel + GEMM straight from NCHW."""

    def __init__(self, conv: nn.Conv2d):
        self.conv = conv
        self._pk = Packed()

    def _packed(self, cin):
        """Weights for an input carrying the first `cin` channels: dict(w [cout, kpad] fp16, b, kpad)."""
        conv = self.conv
        kpad = (9 * cin + 7) // 8 * 8
        pks = self.__dict__.setdefault("_pks", {})
        return pks.setdefault(cin, Packed()).get(
            [conv.weight, conv.bias],
            lambda: dict(w=ops.pack_conv_small_cin(conv.weight[:, :cin], kpad), b=_f32(conv.bias), kpad=kpad))

    def run(self, x_nchw, sdt=F32):
        """x_nchw may carry only the LEADING channels of the layer's input: the missing trailing channels are exact
        zeros (single-step zeros-noise path, marigold_pipeline.py:418-423,447-449: conv_in on 4 of the 8 channels)."""
        return self.forward_saved(x_nchw, sdt)[0]

    def forward_saved(self, x_nchw, sdt=F32):
        """`run`, also returning the im2col patches its weight gradient reads: (out, patches)."""
        cout = self.conv.weight.shape[0]
        NB, cin, H, W = x_nchw.shape
        assert cin <= self.conv.weight.shape[1]
        pk = self._packed(cin)
        patches = ops.im2col3x3(x_nchw.contiguous(), pk["kpad"])
        out = ops.linear(patches, pk["w"], pk["b"], out_dtype=sdt, stats_rows_per_img=H * W)
        return _view_cs(out, NB, H, W, cout), patches


class ConvOutSmall:
    """GroupNorm+SiLU -> conv3x3 with tiny Cout (4 / 3 / 8), written as NCHW fp32."""

    def __init__(self, norm: nn.GroupNorm, conv: nn.Conv2d):
        self.norm, self.conv = norm, conv
        self._pk = Packed()

    def _packed(self):
        norm, conv = self.norm, self.conv
        direct = conv.weight.shape[0] <= 8 and conv.weight.shape[1] % 64 == 0
        return self._pk.get([norm.weight, norm.bias, conv.weight, conv.bias],
                            lambda: dict(g=_f32(norm.weight), b=_f32(norm.bias), cb=_f32(conv.bias), direct=direct,
                                         w=ops.pack_conv_small_cout(conv.weight) if direct else ops.pack_conv(conv.weight)))

    def run(self, x):
        return self.forward_saved(x)[0]

    def forward_saved(self, x):
        """`run`, also returning the normalised conv operand its backward reads: (out, a)."""
        norm, cout = self.norm, self.conv.weight.shape[0]
        pk = self._packed()
        a = ops.group_norm(x, pk["g"], pk["b"], norm.eps, norm.num_groups, True)
        if pk["direct"]:
            return ops.conv3x3_small_cout(a, pk["w"], pk["cb"], cout), a      # input read once (halo tile in smem)
        return ops.conv2d(a, pk["w"], cout, bias=pk["cb"], out_dtype=F32, out_nchw=True), a
