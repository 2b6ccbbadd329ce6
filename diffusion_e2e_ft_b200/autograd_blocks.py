"""Training-mode (differentiable) execution of the engine blocks — SURVEY.md §8 row a10.

The reference trains through `accelerator.backward(loss)` (training/train.py:563): plain torch.autograd over
the UNet and the frozen VAE decoder.  The engine keeps that boundary: every block of modules.py / unet.py / vae.py is
one `torch.autograd.Function`.  Its forward calls the block's inference forward (`forward_saved`, which also returns
the intermediates the backward reads) and adds only the GroupNorm mean / rstd of the saved inputs; its backward is
hand-written on the backward operators of backward.py / csrc/backward.cu and reads the weights through the same
`_packed*` methods as inference.  So a training forward launches the inference kernels by construction.
torch.autograd is used for what it is in the reference — graph bookkeeping between blocks (skip connections,
the shared time embedding, `.grad` accumulation) — never for arithmetic inside a block.

Precision: residual stream and its gradient fp32; GEMM operands (activations and incoming gradients) fp16 —
callers scale the loss (`training.LOSS_SCALE`) so fp16 gradients stay in range; parameter gradients fp32.
"""
import torch

from . import backward as bw
from . import ops
from .backward_packing import pack_conv_dgrad_s1, pack_conv_dgrad_s2, pack_upsample_conv_dgrad
from .modules import Packed, _f16, _f32
from .ops import F16, F32, TAPS3, TAPS3_PAD0


def _attach(out, box):
    """Function.apply hands back the tensor object created in forward, but re-attach the producer extras
    (fused GroupNorm sums / fp16 twin) explicitly so nothing depends on that."""
    for k in ("_cs", "_h16"):
        v = box.get(k)
        if v is not None and getattr(out, k, None) is None:
            setattr(out, k, v)
    return out


def _stash(out, box):
    for k in ("_cs", "_h16"):
        v = getattr(out, k, None)
        if v is not None:
            box[k] = v
    return out


def _bwd_cache(mod, kind=""):
    """The module's cache of the backward operand `kind` (re-packed weights), built by one function."""
    return mod.__dict__.setdefault("_pk_bwd", {}).setdefault(kind, Packed())


def _any(ctx, first):
    return any(ctx.needs_input_grad[first:])


# ----------------------------------------------------------------------------------------------- resnet
def _resnet_params(m):
    ps = [m.norm1.weight, m.norm1.bias, m.conv1.weight, m.conv1.bias, m.norm2.weight, m.norm2.bias,
          m.conv2.weight, m.conv2.bias]
    if m.conv_shortcut is not None:
        ps += [m.conv_shortcut.weight, m.conv_shortcut.bias]
    return ps


class _ResnetFn(torch.autograd.Function):
    """ResnetBlock2D + its backward.  inputs: x [NB,H,W,C1] fp32, skip [NB,H,W,C2] | None, temb [NB,cout] | None."""

    @staticmethod
    def run(m, f16_copy, x, skip, temb):
        out, (a1, raw, h, a2) = m.forward_saved(x, temb, skip, F32, f16_copy)
        mr1 = ops.group_norm_mean_rstd(x, m.eps, m.groups, skip)
        mr2 = ops.group_norm_mean_rstd(h, m.eps, m.groups)
        return out, ([x] if skip is None else [x, skip], mr1, a1, raw, h, mr2, a2)

    @staticmethod
    def forward(ctx, m, f16_copy, box, x, skip, temb, *params):
        out, saved = _ResnetFn.run(m, f16_copy, x, skip, temb)
        ctx.m, ctx.has_temb = m, temb is not None
        # gradient checkpointing (unet.enable_gradient_checkpointing, train.py:358-359): keep the block inputs only
        # and re-run the block's forward kernels at the start of its backward
        ctx.saved, ctx.inputs = (None, (f16_copy, x, skip, temb)) if box.get("ckpt") else (saved, None)
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        m = ctx.m
        xs, mr1, a1, raw, h, mr2, a2 = ctx.saved if ctx.saved is not None else _ResnetFn.run(m, *ctx.inputs)[1]
        pk = m._packed()
        train = _any(ctx, 6)
        short = m.conv_shortcut is not None
        cin = sum(t.shape[3] for t in xs)

        def build():
            d = dict(d1=pack_conv_dgrad_s1(m.conv1.weight), d2=pack_conv_dgrad_s1(m.conv2.weight))
            if short:
                d["st"] = ops.transpose_rows(_f16(m.conv_shortcut.weight.reshape(m.cout, cin)))      # [cin, cout]
            return d
        pb = _bwd_cache(m).get(_resnet_params(m), build)

        dout = dout.contiguous()
        NB, H, W, cout = dout.shape
        d16 = ops.cast_f16(dout)
        g = {}
        # ---- conv2 (+ 1x1 shortcut, fused in the forward as extra K columns)
        if train:
            dw2, db2 = bw.conv_wgrad(a2, d16, TAPS3)
            g["w2"], g["b2"] = bw.unpack_conv_grad(dw2, cout), db2
            if short:
                dws, _ = bw.conv_wgrad(raw, d16, [(0, 0)], bias=False)
                g["ws"], g["bs"] = dws.view(cout, cin, 1, 1), db2
        da2 = bw.conv_dgrad(d16, None, cout, "s1", out_dtype=F16, packed=pb["d2"])
        # ---- norm2 + SiLU
        (dh,), g["g2"], g["be2"] = ops.group_norm_bwd([h], da2, mr2, pk["g2"], pk["b2"], m.groups, True, None, F16)
        # ---- temb broadcast add and conv1 bias: per-image / total column sums of dh
        dtemb = None
        if ctx.has_temb and (ctx.needs_input_grad[5] or train):
            dtemb = torch.zeros((NB, cout), dtype=F32, device=dout.device)
            for n in range(NB):
                ops.col_sum(dh[n].view(H * W, cout), out=dtemb[n])
        # ---- conv1
        if train:
            dw1, db1 = bw.conv_wgrad(a1, dh, TAPS3, bias=dtemb is None)
            g["w1"] = bw.unpack_conv_grad(dw1, cin)
            g["b1"] = db1 if dtemb is None else dtemb.sum(0)
        da1 = bw.conv_dgrad(dh, None, cin, "s1", out_dtype=F16, packed=pb["d1"])
        # ---- norm1 + SiLU, plus the residual / shortcut path into the block inputs
        if short:
            adds, off = [], 0
            for t in xs:
                c = t.shape[3]
                adds.append(ops.conv2d(d16, pb["st"][off:off + c], c, taps=[(0, 0)], out_dtype=F32))
                off += c
        else:
            adds = [dout]
        dxs, g["g1"], g["be1"] = ops.group_norm_bwd(xs, da1, mr1, pk["g1"], pk["b1"], m.groups, True, adds, F32)
        grads = [g.get(k) for k in ("g1", "be1", "w1", "b1", "g2", "be2", "w2", "b2")]
        if short:
            grads += [g.get("ws"), g.get("bs")]
        if not train:
            grads = [None] * len(grads)
        return (None, None, None, dxs[0], dxs[1] if len(dxs) > 1 else None,
                dtemb if ctx.has_temb else None, *grads)


def resnet(m, x, temb=None, skip=None, f16_copy=False, ckpt=False):
    box = {"ckpt": ckpt}
    return _attach(_ResnetFn.apply(m, f16_copy, box, x, skip, temb, *_resnet_params(m)), box)


# ------------------------------------------------------------------------------------------ down / up sample
class _DownsampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, m, box, x, weight, bias):
        out, x16 = m.forward_saved(x)
        ctx.m, ctx.saved = m, (x16,)
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        m = ctx.m
        (x16,) = ctx.saved
        NB, H, W, C = x16.shape
        taps, kind = (TAPS3, "s2") if m.padding == 1 else (TAPS3_PAD0, "s2_vae")
        d16 = ops.cast_f16(dout.contiguous())
        gw = gb = None
        if _any(ctx, 3):
            dwp, gb = bw.conv_wgrad(x16, d16, taps, stride=2)
            gw = bw.unpack_conv_grad(dwp, C)
        pb = _bwd_cache(m).get([m.conv.weight], lambda: pack_conv_dgrad_s2(m.conv.weight, 1 if m.padding == 1 else 0))
        dx = bw.conv_dgrad(d16, None, C, kind, out_dtype=F32, packed=pb, in_hw=(H, W))
        return None, None, dx, gw, gb


def downsample(m, x):
    box = {}
    return _attach(_DownsampleFn.apply(m, box, x, m.conv.weight, m.conv.bias), box)


class _UpsampleFn(torch.autograd.Function):
    """Upsample2D + its backward: nearest-2x + conv3x3 as four 2x2 phase convs, or nearest to an explicit size
    (unet_2d_condition.py:1185-1186, latent sizes not divisible by 2^levels) + conv3x3."""

    @staticmethod
    def forward(ctx, m, out_hw, box, x, weight, bias):
        out, a = m.forward_saved(x, out_hw)
        ctx.m, ctx.saved, ctx.in_hw, ctx.resize = m, (a,), tuple(x.shape[1:3]), m.resizes(x, out_hw)
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        m = ctx.m
        (a,) = ctx.saved
        C = a.shape[3]
        d16 = ops.cast_f16(dout.contiguous())
        gw = gb = None
        if _any(ctx, 4):
            dwp, gb = bw.conv_wgrad(a, d16, TAPS3, up=1 if ctx.resize else 2)
            gw = bw.unpack_conv_grad(dwp, C)
        if ctx.resize:
            pb = _bwd_cache(m, "s1").get([m.conv.weight], lambda: pack_conv_dgrad_s1(m.conv.weight))
            da = bw.conv_dgrad(d16, None, C, "s1", out_dtype=F32, packed=pb)
            dx = ops.upsample_nearest_bwd(da, ctx.in_hw)
        else:
            pb = _bwd_cache(m, "up").get([m.conv.weight],
                                         lambda: pack_upsample_conv_dgrad(m._packed_phases()["ph"]))
            dx = bw.conv_dgrad(d16, None, C, "up", out_dtype=F32, packed=pb)
        return None, None, None, dx, gw, gb


def upsample(m, x, out_hw=None):
    box = {}
    return _attach(_UpsampleFn.apply(m, out_hw, box, x, m.conv.weight, m.conv.bias), box)


# ---------------------------------------------------------------------------------------- transformer block
def _transformer_params(m):
    b = m.transformer_blocks[0]
    a1, a2, ff = b.attn1, b.attn2, b.ff
    return [m.norm.weight, m.norm.bias, m.proj_in.weight, m.proj_in.bias, m.proj_out.weight, m.proj_out.bias,
            b.norm1.weight, b.norm1.bias, a1.to_q.weight, a1.to_k.weight, a1.to_v.weight,
            a1.to_out[0].weight, a1.to_out[0].bias,
            b.norm2.weight, b.norm2.bias, a2.to_q.weight, a2.to_k.weight, a2.to_v.weight,
            a2.to_out[0].weight, a2.to_out[0].bias,
            b.norm3.weight, b.norm3.bias, ff.net[0].proj.weight, ff.net[0].proj.bias,
            ff.net[2].weight, ff.net[2].bias]


class _TransformerFn(torch.autograd.Function):
    """Transformer2DModel (one BasicTransformerBlock; plain or GeoWizard joint self-attention) + its backward."""

    @staticmethod
    def run(m, f16_copy, x, ctx16):
        out, (hn, h0, blk_saved, h16) = m.forward_saved(x, ctx16, F32, f16_copy)     # general path: no const_ctx
        mr0 = ops.group_norm_mean_rstd(x, 1e-6, m.groups)
        return out, (x, mr0, hn, h0, *blk_saved, h16)

    @staticmethod
    def forward(ctx, m, f16_copy, box, x, ctx16, *params):
        out, saved = _TransformerFn.run(m, f16_copy, x, ctx16)
        ctx.m = m
        ctx.saved, ctx.inputs = (None, (f16_copy, x, ctx16)) if box.get("ckpt") else (saved, None)
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        m = ctx.m
        blk = m.transformer_blocks[0]
        saved = ctx.saved if ctx.saved is not None else _TransformerFn.run(m, *ctx.inputs)[1]
        x, mr0, hn, h0, n1, qkv, o, h1, n2, q2, c2d, kv, o2, h2, n3, gg, h16 = saved
        pk, bp = m._packed(), blk._packed()
        B, H, W, C = x.shape
        L, heads, scale = H * W, blk.heads, blk.head_dim ** -0.5
        S = kv.shape[1]
        train = _any(ctx, 5)
        proj = blk.ff.net[0].proj
        pb = _bwd_cache(m).get([proj.weight, proj.bias], lambda: dict(wcat=_f16(proj.weight), bcat=_f32(proj.bias)))
        dev = x.device
        dout = dout.contiguous().view(B * L, C)
        g = {}
        # ---- proj_out (+ residual x)
        dh3, g["wo"], g["bo"] = bw.linear_bwd(h16, pk["wo"], ops.cast_f16(dout), da_dtype=F32, need_dw=train)
        # ---- feed-forward: h3 = h2 + W_f (value * gelu(gate)) + b_f
        dgg, g["wf"], g["bf"] = bw.linear_bwd(gg, bp["wf"], ops.cast_f16(dh3), need_dw=train)
        hg = ops.linear(n3, pb["wcat"], pb["bcat"])                      # [value | gate] pre-activations (recomputed)
        dhg = ops.geglu_bwd(hg, dgg)
        del hg, dgg
        dn3, g["wp"], g["bp"] = bw.linear_bwd(n3, pb["wcat"], dhg, need_dw=train)
        del dhg
        dh2, g["ln3w"], g["ln3b"] = ops.layer_norm_bwd(h2, dn3, bp["ln"][2][0], 1e-5, add=dh3)
        # ---- cross attention: h2 = h1 + W_o2 attn(q2, k, v) + b_o2
        do2, g["wo2"], g["bo2"] = bw.linear_bwd(o2.view(B * L, C), bp["wo2"], ops.cast_f16(dh2), need_dw=train)
        dkv = torch.empty((B, S, 2 * C), dtype=F16, device=dev)
        dq2 = torch.empty((B, L, C), dtype=F16, device=dev)
        bw.attention_bwd(q2, kv[..., :C], kv[..., C:], do2.view(B, L, C), heads, scale,
                         outs=(dq2, dkv[..., :C], dkv[..., C:]))
        if train:
            _, dwkv, _ = bw.linear_bwd(c2d, bp["wkv2"], dkv.view(B * S, 2 * C), need_da=False, bias=False)
            g["wk2"], g["wv2"] = dwkv[:C], dwkv[C:]
        dn2, g["wq2"], _ = bw.linear_bwd(n2, bp["wq2"], dq2.view(B * L, C), need_dw=train, bias=False)
        dh1, g["ln2w"], g["ln2b"] = ops.layer_norm_bwd(h1, dn2, bp["ln"][1][0], 1e-5, add=dh2)
        # ---- self attention: h1 = h0 + W_o1 attn(q, k, v) + b_o1
        do1, g["wo1"], g["bo1"] = bw.linear_bwd(o.view(B * L, C), bp["wo1"], ops.cast_f16(dh1), need_dw=train)
        dqkv = torch.empty((B, L, 3 * C), dtype=F16, device=dev)
        # joint blocks (XFormersJointAttnProcessor, attention.py:430-513): images i and i + B/2 attend to the keys of
        # both, kv_segments = 2 as in the forward
        bw.attention_bwd(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], do1.view(B, L, C), heads, scale,
                         outs=(dqkv[..., :C], dqkv[..., C:2 * C], dqkv[..., 2 * C:]),
                         kv_segments=2 if blk.joint else 1)
        dn1, dwqkv, _ = bw.linear_bwd(n1, bp["wqkv"], dqkv.view(B * L, 3 * C), need_dw=train, bias=False)
        if train:
            g["wq1"], g["wk1"], g["wv1"] = dwqkv[:C], dwqkv[C:2 * C], dwqkv[2 * C:]
        dh0, g["ln1w"], g["ln1b"] = ops.layer_norm_bwd(h0, dn1, bp["ln"][0][0], 1e-5, add=dh1)
        # ---- proj_in and the GroupNorm in front of it; the block's residual x joins here
        dhn, g["wi"], g["bi"] = bw.linear_bwd(hn.view(B * L, C), pk["wi"], ops.cast_f16(dh0), need_dw=train)
        (dx,), g["gnw"], g["gnb"] = ops.group_norm_bwd([x], dhn.view(B, H, W, C), mr0, pk["g"], pk["b"], m.groups,
                                                       False, [dout.view(B, H, W, C)], F32)
        order = ("gnw", "gnb", "wi", "bi", "wo", "bo", "ln1w", "ln1b", "wq1", "wk1", "wv1", "wo1", "bo1",
                 "ln2w", "ln2b", "wq2", "wk2", "wv2", "wo2", "bo2", "ln3w", "ln3b", "wp", "bp", "wf", "bf")
        if train:                       # 1x1-conv projections: the [C, C] GEMM gradient in the [C, C, 1, 1] layout
            g["wi"], g["wo"] = g["wi"].view(m.proj_in.weight.shape), g["wo"].view(m.proj_out.weight.shape)
        grads = [g.get(k) if train else None for k in order]
        return (None, None, None, dx, None, *grads)


def transformer(m, x, ctx16, f16_copy=False, ckpt=False):
    box = {"ckpt": ckpt}
    return _attach(_TransformerFn.apply(m, f16_copy, box, x, ctx16, *_transformer_params(m)), box)


# ------------------------------------------------------------------------------------- conv_in / conv_out
class _ConvInFn(torch.autograd.Function):
    """ConvInSmall (im2col + GEMM from the NCHW sample); backward = weight/bias gradients (the sample is data)
    and, when the input needs it (VAE decoder), the data gradient through the small-Cout conv kernel."""

    @staticmethod
    def forward(ctx, runner, box, x_nchw, weight, bias):
        out, patches = runner.forward_saved(x_nchw)
        ctx.runner, ctx.saved, ctx.cin = runner, (patches,), x_nchw.shape[1]
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        conv, cin = ctx.runner.conv, ctx.cin
        (patches,) = ctx.saved
        NB, H, W, cout = dout.shape
        d16 = ops.cast_f16(dout.contiguous()).view(NB * H * W, cout)
        gw = gb = dx = None
        if ctx.needs_input_grad[3] or ctx.needs_input_grad[4]:
            _, dwp, gb = bw.linear_bwd(patches, ctx.runner._packed(cin)["w"], d16, need_da=False)
            gw = dwp[:, :9 * cin].reshape(cout, 3, 3, cin).permute(0, 3, 1, 2).contiguous()
        if ctx.needs_input_grad[2]:
            wq = _bwd_cache(ctx.runner).get([conv.weight], lambda: ops.pack_conv_small_cout(
                conv.weight.detach().flip(2, 3).transpose(0, 1).contiguous()))
            dx = ops.conv3x3_small_cout(d16.view(NB, H, W, cout), wq, None, cin)      # NCHW fp32 [NB, cin, H, W]
        return None, None, dx, gw, gb


def conv_in(runner, x_nchw):
    box = {}
    return _attach(_ConvInFn.apply(runner, box, x_nchw, runner.conv.weight, runner.conv.bias), box)


class _ConvOutFn(torch.autograd.Function):
    """ConvOutSmall: GroupNorm+SiLU -> conv3x3 with tiny Cout, NCHW fp32 out."""

    @staticmethod
    def forward(ctx, runner, x, nw, nb, weight, bias):
        out, a = runner.forward_saved(x)
        mr = ops.group_norm_mean_rstd(x, runner.norm.eps, runner.norm.num_groups)
        ctx.runner, ctx.saved = runner, (x, mr, a)
        return out

    @staticmethod
    def backward(ctx, dout):
        norm, conv = ctx.runner.norm, ctx.runner.conv
        x, mr, a = ctx.saved
        pk = ctx.runner._packed()
        NB, H, W, C = x.shape
        cout = conv.weight.shape[0]
        dout = dout.contiguous().float()
        kpad = (9 * cout + 7) // 8 * 8
        wd = _bwd_cache(ctx.runner).get([conv.weight], lambda: ops.pack_conv_small_cin(
            conv.weight.detach().flip(2, 3).transpose(0, 1).contiguous(), kpad))      # dgrad = conv with Cin = cout
        da = ops.linear(ops.im2col3x3(dout, kpad), wd).view(NB, H, W, C)
        gw = gb = None
        train = _any(ctx, 2)
        if train:
            dy_nhwc = dout.permute(0, 2, 3, 1).contiguous().to(F16)          # tiny (<= 8 channels): host re-layout
            dwp, gb = bw.conv_wgrad(a, dy_nhwc, TAPS3)
            gw = bw.unpack_conv_grad(dwp, C)
        (dx,), gg, gbeta = ops.group_norm_bwd([x], da, mr, pk["g"], pk["b"], norm.num_groups, True, None, F32)
        if not train:
            gg = gbeta = None
        return None, dx, gg, gbeta, gw, gb


def conv_out(runner, x):
    return _ConvOutFn.apply(runner, x, runner.norm.weight, runner.norm.bias, runner.conv.weight, runner.conv.bias)


# ------------------------------------------------------------------------------------- time / class embedding
def _embed_params(unet):
    te, ce = unet.time_embedding, unet.class_embedding
    ps = [te.linear_1.weight, te.linear_1.bias, te.linear_2.weight, te.linear_2.bias]
    if ce is not None:
        ps += [ce.linear_1.weight, ce.linear_1.bias, ce.linear_2.weight, ce.linear_2.bias]
    for r in unet._resnets():
        ps += [r.time_emb_proj.weight, r.time_emb_proj.bias]
    return ps


class _EmbedFn(torch.autograd.Function):
    """sinusoid -> linear_1 -> SiLU -> linear_2 (+ class embedding) -> SiLU -> every resnet's time_emb_proj in one GEMM
    (B200UNet2DConditionModel._time_embedding, unet_2d_condition.py:957-1000)."""

    @staticmethod
    def forward(ctx, unet, t, class_labels, *params):
        out, ctx.saved = unet._time_embedding(t, class_labels)
        ctx.unet = unet
        return out

    @staticmethod
    def backward(ctx, dall):
        unet = ctx.unet
        e0, e1, e2, cl, c1, c = ctx.saved
        ep = unet._embed_packed()
        de2, dwall, dball = bw.linear_bwd(e2, ep["wall"], ops.cast_f16(dall.contiguous()))
        z2 = ops.linear(e1, ep["w2"], ep["b2"], residual=c)                       # pre-activation, recomputed
        dz2 = ops.act_bwd(z2, de2, ops.ACT_SILU)
        de1, dw2, db2 = bw.linear_bwd(e1, ep["w2"], dz2)
        z1 = ops.linear(e0, ep["w1"], ep["b1"])
        _, dw1, db1 = bw.linear_bwd(e0, ep["w1"], ops.act_bwd(z1, de1, ops.ACT_SILU), need_da=False)
        grads = [dw1, db1, dw2, db2]
        if unet.class_embedding is not None:
            dc1, dcw2, dcb2 = bw.linear_bwd(c1, ep["cw2"], dz2)
            zc = ops.linear(cl, ep["cw1"], ep["cb1"])
            _, dcw1, dcb1 = bw.linear_bwd(cl, ep["cw1"], ops.act_bwd(zc, dc1, ops.ACT_SILU), need_da=False)
            kin = unet.class_embedding.linear_1.weight.shape[1]
            grads += [dcw1[:, :kin], dcb1, dcw2, dcb2]
        for r, o in zip(unet._resnets(), ep["offs"]):
            grads += [dwall[o:o + r.cout], dball[o:o + r.cout]]
        return (None, None, None, *grads)


def embed(unet, t, class_labels):
    return _EmbedFn.apply(unet, t, class_labels, *_embed_params(unet))


# ------------------------------------------------------------------------------------ VAE mid-block attention
class _VAEAttentionFn(torch.autograd.Function):
    """VAEAttention (single head, d = channels) + its data gradient, on the path inference takes for the same shape
    (vae.use_fused_attention): the unfused GEMM + row-softmax path, which saves P [B, L, Lp], or the d=512 flash
    kernel, which saves Q, K, V, O and the log-sum-exp and recomputes P in the fused backward (O(L) memory).  The VAE
    is frozen in the fine-tuning recipe (training/train.py:323-326), so only d/dx is produced."""

    @staticmethod
    def run(m, fused, x):
        out, saved = m.forward_fused(x, want_lse=True) if fused else m.forward_unfused(x)
        mr = ops.group_norm_mean_rstd(x, m.eps, m.groups)
        return out, (x, mr, *saved)

    @staticmethod
    def forward(ctx, m, box, x):
        from .vae import use_fused_attention
        B, H, W, C = x.shape
        ctx.fused = use_fused_attention(B, H * W, C, m.memory_efficient)
        out, saved = _VAEAttentionFn.run(m, ctx.fused, x)
        ctx.m = m
        # gradient checkpointing (B200AutoencoderKL.enable_gradient_checkpointing): keep the input only, as _ResnetFn
        ctx.saved, ctx.inputs = (None, (ctx.fused, x)) if box.get("ckpt") else (saved, None)
        return _stash(out, box)

    @staticmethod
    def backward(ctx, dout):
        m = ctx.m
        if any(p.requires_grad for p in m.parameters()):
            raise NotImplementedError("the VAE attention block is differentiable w.r.t. its input only (frozen VAE)")
        saved = ctx.saved if ctx.saved is not None else _VAEAttentionFn.run(m, *ctx.inputs)[1]
        x, mr = saved[:2]
        pk = m._packed()
        B, H, W, C = x.shape
        dout = dout.contiguous()
        dhn = (_VAEAttentionFn._dhn_fused if ctx.fused else _VAEAttentionFn._dhn_unfused)(pk, dout, *saved[2:])
        (dx,), _, _ = ops.group_norm_bwd([x], dhn.view(B, H, W, C), mr, pk["g"], pk["b"], m.groups, False, [dout], F32)
        return None, None, dx

    @staticmethod
    def _dhn_fused(pk, dout, hn, qkv, o, lse):
        """d(GroupNorm output) through the out-projection, the fused d=512 attention backward and the QKV projection."""
        B, L, C = o.shape
        do, _, _ = bw.linear_bwd(o.view(B * L, C), pk["wo"], ops.cast_f16(dout).view(B * L, C), need_dw=False)
        do = do.view(B, L, C)
        delta = ops.rowdot_d512(do, o)
        dqkv = torch.empty((B, L, 3 * C), dtype=F16, device=o.device)
        ops.attention_d512_bwd(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], do, lse, delta,
                               dqkv[..., :C], dqkv[..., C:2 * C], dqkv[..., 2 * C:], C ** -0.5)
        dhn, _, _ = bw.linear_bwd(hn, pk["wqkv"], dqkv.view(B * L, 3 * C), need_dw=False)
        return dhn

    @staticmethod
    def _dhn_unfused(pk, dout, hn, qk, p_buf, o):
        B, L, C = o.shape
        Lp = p_buf.shape[2]
        scale = C ** -0.5
        dev = o.device
        do, _, _ = bw.linear_bwd(o.view(B * L, C), pk["wo"], ops.cast_f16(dout).view(B * L, C), need_dw=False)
        do = do.view(B, L, C)
        v = ops.linear(hn.view(B * L, C), pk["wv"], pk["bv"]).view(B, L, C)            # recomputed (forward keeps V^T)
        dqk = torch.empty((B, L, 2 * C), dtype=F16, device=dev)
        dv = torch.empty((B, L, C), dtype=F16, device=dev)
        for b in range(B):
            q_b, k_b = qk[b, :, :C], qk[b, :, C:]
            dp = torch.zeros((L, Lp), dtype=F32, device=dev)
            ops.linear(do[b], v[b], out=dp[:, :L], out_dtype=F32)
            ds = ops.softmax_bwd_rows(p_buf[b], dp, scale, cols=L)                     # [L, Lp] fp16, padding 0
            del dp
            # dQ = dS K, dK = dS^T Q, dV = P^T dO with the row-major operands consumed MN-major as stored (no transposes)
            ops.linear(ds[:, :L], k_b, out=dqk[b, :, :C], w_t=True)
            ops.linear(ds[:, :L], q_b, out=dqk[b, :, C:], a_t=True, w_t=True)
            ops.linear(p_buf[b][:, :L], do[b], out=dv[b], a_t=True, w_t=True)
        dhn, _, _ = bw.linear_bwd(hn.view(B * L, C), pk["wqk"], dqk.view(B * L, 2 * C), need_dw=False)
        dhn, _, _ = bw.linear_bwd(hn.view(B * L, C), pk["wv"], dv.view(B * L, C), need_dw=False, da_add=dhn)
        return dhn


def vae_attention(m, x, ckpt=False):
    box = {"ckpt": ckpt}
    return _attach(_VAEAttentionFn.apply(m, box, x), box)


# --------------------------------------------------------------- latent -> decoder input, post-ops and losses
class _PointwiseFn(torch.autograd.Function):
    """Conv1x1Small (post_quant_conv with the x0 / scaling-factor coefficients folded in): out = W (a1 * x) + b."""

    @staticmethod
    def forward(ctx, conv, a1, x, const=None, a2=0.0):
        w = conv.weight.detach().reshape(conv.out_channels, conv.in_channels).to(F32).contiguous()
        b = conv.bias.detach().to(F32).contiguous()
        ctx.w, ctx.a1 = w, a1
        c = None if const is None else const.detach().float().contiguous()
        return ops.pointwise_nchw(x.float().contiguous(), a1, w, b, in2=c, a2=a2, cin=conv.in_channels)

    @staticmethod
    def backward(ctx, dout):
        wt = ctx.w.t().contiguous()
        zero = torch.zeros((wt.shape[0],), dtype=F32, device=dout.device)
        return None, None, ops.pointwise_nchw(dout.float().contiguous(), ctx.a1, wt, zero, cin=wt.shape[1]), None, None


def pointwise(conv, x, a1, const=None, a2=0.0):
    """W (a1 * x + a2 * const) + b; `const` (e.g. the noisy latent x_t of a noisy-start step) carries no gradient."""
    return _PointwiseFn.apply(conv, a1, x, const, a2)


class _DecodePostFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, normals):
        x = x.float().contiguous()
        ctx.saved, ctx.normals = (x,), normals
        return ops.decode_post(x, normals=normals, training=True)

    @staticmethod
    def backward(ctx, dout):
        return ops.decode_post_bwd(ctx.saved[0], dout.float().contiguous(), ctx.normals), None


def decode_post(x, normals):
    return _DecodePostFn.apply(x, normals)


class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, est, target, mask, normals):
        ctx.saved, ctx.normals = (est, target, mask), normals
        return (ops.angular_loss if normals else ops.ssi_loss)(est, target, mask)

    @staticmethod
    def backward(ctx, gout):
        est, target, mask = ctx.saved
        fn = ops.angular_loss_bwd if ctx.normals else ops.ssi_loss_bwd
        return fn(est, target, mask, gout).view_as(est), None, None, None


def task_loss(est, target, mask, normals):
    return _LossFn.apply(est, target, mask, normals)


class _MaskedLatentMSEFn(torch.autograd.Function):
    """Diffusion-objective loss (train_depth_normal.py:607-609,712-714): the latent mask is pooled from the pixel mask
    once, in the forward, and saved with the fp64 (sum, count) workspace for the backward."""

    @staticmethod
    def forward(ctx, pred, target, val_mask):
        pred = pred.contiguous()
        loss, lm, ws = ops.masked_latent_mse(pred, target, val_mask)
        ctx.saved = (pred, target, lm, ws)
        return loss

    @staticmethod
    def backward(ctx, gout):
        pred, target, lm, ws = ctx.saved
        return ops.masked_latent_mse_bwd(pred, target, lm, ws, gout), None, None


def masked_latent_mse(pred, target, val_mask):
    return _MaskedLatentMSEFn.apply(pred, target.detach(), val_mask)
