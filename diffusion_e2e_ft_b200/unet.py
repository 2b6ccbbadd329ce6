"""B200UNet2DConditionModel — drop-in for diffusers' / GeoWizard's `UNet2DConditionModel` on the
single-step denoising path.

Call-compatible with the reference call sites
    Marigold/marigold/marigold_pipeline.py:452-454   unet(x, t, encoder_hidden_states=E).sample
    training/train.py:500                            unet(x, t, E, return_dict=False)[0]
    GeoWizard/.../geowizard_pipeline.py:319-321      unet(x, t.repeat(2), encoder_hidden_states=E, class_labels=C).sample
Control flow restates GeoWizard/geowizard/models/unet_2d_condition.py:845-1221; parameters keep the
diffusers `state_dict` names (SURVEY.md App. A.8).  All arithmetic runs in libb200_e2eft.so.
"""
import torch
import torch.nn as nn

from . import autograd_blocks as ab
from . import ops
from .modules import (ConfigDict, ConvInSmall, ConvOutSmall, Downsample2D, Packed, ResnetBlock2D,
                      Transformer2DModel, Upsample2D, _f16, _f32)
from .checkpoint import PretrainedMixin
from .ops import F16, F32


class UNet2DConditionOutput:
    """Stand-in for diffusers' BaseOutput subclass: `.sample` plus tuple-style indexing."""

    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


class TimestepEmbedding(nn.Module):
    def __init__(self, in_dim, dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_dim, dim)
        self.linear_2 = nn.Linear(dim, dim)


class _DownBlock(nn.Module):
    """CrossAttnDownBlock2D (unet_2d_blocks.py:1027-1185) / DownBlock2D (:1188-1273)."""

    def __init__(self, cin, cout, temb, n, heads, cross_dim, has_attn, add_down, groups, eps, joint, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(n)])
        self.attentions = nn.ModuleList(
            [Transformer2DModel(cout, heads, cross_dim, groups, joint, linear_proj) for _ in range(n)]) if has_attn else None
        self.downsamplers = nn.ModuleList([Downsample2D(cout, 1)]) if add_down else None


class _MidBlock(nn.Module):
    """UNetMidBlock2DCrossAttn (unet_2d_blocks.py:634-777)."""

    def __init__(self, ch, temb, heads, cross_dim, groups, eps, joint, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([Transformer2DModel(ch, heads, cross_dim, groups, joint, linear_proj)])


class _UpBlock(nn.Module):
    """CrossAttnUpBlock2D (unet_2d_blocks.py:2201-2371) / UpBlock2D (:2374-2481)."""

    def __init__(self, cin, cout, cprev, temb, n, heads, cross_dim, has_attn, add_up, groups, eps, joint, linear_proj):
        super().__init__()
        rs = []
        for i in range(n):
            skip = cin if i == n - 1 else cout
            rin = cprev if i == 0 else cout
            rs.append(ResnetBlock2D(rin + skip, cout, temb, groups, eps))
        self.resnets = nn.ModuleList(rs)
        self.attentions = nn.ModuleList(
            [Transformer2DModel(cout, heads, cross_dim, groups, joint, linear_proj) for _ in range(n)]) if has_attn else None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None


_DEFAULTS = dict(
    in_channels=8, out_channels=4, block_out_channels=(320, 640, 1280, 1280),
    down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
    up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3,
    layers_per_block=2, attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024,
    norm_num_groups=32, norm_eps=1e-5, class_embed_type=None,
    projection_class_embeddings_input_dim=None, joint_attention=False,
    flip_sin_to_cos=True, freq_shift=0, sample_size=96, act_fn="silu", use_linear_projection=True)


class B200UNet2DConditionModel(PretrainedMixin, nn.Module):
    """`stream_dtype`: dtype of the residual stream inside the engine (fp32 = parity mode, fp16 = fast)."""
    _diffusers_class_name = "UNet2DConditionModel"
    _config_defaults = _DEFAULTS

    def __init__(self, stream_dtype=torch.float32, **config):
        super().__init__()
        cfg = ConfigDict(_DEFAULTS)
        unknown = set(config) - set(_DEFAULTS)
        if unknown:
            raise TypeError(f"unknown UNet config keys: {sorted(unknown)}")
        cfg.update(config)
        for k in ("block_out_channels", "down_block_types", "up_block_types", "attention_head_dim"):
            if isinstance(cfg[k], list):
                cfg[k] = tuple(cfg[k])
        if not cfg["flip_sin_to_cos"] or cfg["freq_shift"] != 0:
            raise NotImplementedError("engine supports the SD embedding config (flip_sin_to_cos, freq_shift 0) only")
        self.config = cfg
        self.stream_dtype = stream_dtype
        boc = tuple(cfg["block_out_channels"])
        # number of heads per block (unet_2d_condition.py:244-250); SD-1 configs store one scalar for all blocks
        heads = cfg["attention_head_dim"]
        heads = (heads,) * len(boc) if isinstance(heads, int) else tuple(heads)
        temb = boc[0] * 4
        g, eps, cd, J = cfg["norm_num_groups"], cfg["norm_eps"], cfg["cross_attention_dim"], cfg["joint_attention"]
        lp = bool(cfg["use_linear_projection"])         # False: 1x1-conv proj_in / proj_out (SD-1, GeoWizard)
        self.conv_in = nn.Conv2d(cfg["in_channels"], boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        self.class_embedding = (TimestepEmbedding(cfg["projection_class_embeddings_input_dim"], temb)
                                if cfg["class_embed_type"] == "projection" else None)
        n = cfg["layers_per_block"]
        downs, ch = [], boc[0]
        for i, t in enumerate(cfg["down_block_types"]):
            cin, ch = ch, boc[i]
            downs.append(_DownBlock(cin, ch, temb, n, heads[i], cd, t == "CrossAttnDownBlock2D",
                                    i != len(boc) - 1, g, eps, J, lp))
        self.down_blocks = nn.ModuleList(downs)
        self.mid_block = _MidBlock(boc[-1], temb, heads[-1], cd, g, eps, J, lp)
        rev, rheads = list(reversed(boc)), list(reversed(heads))
        ups, cout = [], rev[0]
        for i, t in enumerate(cfg["up_block_types"]):
            cprev, cout = cout, rev[i]
            cin = rev[min(i + 1, len(boc) - 1)]
            ups.append(_UpBlock(cin, cout, cprev, temb, n + 1, rheads[i], cd, t == "CrossAttnUpBlock2D",
                                i != len(boc) - 1, g, eps, J, lp))
        self.up_blocks = nn.ModuleList(ups)
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=eps)
        self.conv_out = nn.Conv2d(boc[0], cfg["out_channels"], 3, padding=1)
        self._pk = Packed()
        self._gradient_checkpointing = False

    # ------------------------------------------------------------------ diffusers-API shims
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        """No-op: the engine's attention always runs memory-efficiently (Marigold/run.py:284-287): the forward is the
        flash kernel, and the training backward recomputes P and dS on chip in the fused backward kernels, so neither
        pass stores a [heads, T, Tk] matrix."""

    def enable_gradient_checkpointing(self):
        self._gradient_checkpointing = True

    def register_to_config(self, **kw):
        """diffusers API used by the load hook (training/train.py:335): unknown keys are kept, not rejected."""
        self.config.update({k: v for k, v in kw.items() if k in _DEFAULTS})
        extra = {k: v for k, v in kw.items() if k not in _DEFAULTS and k != "_extra"}
        if extra:
            self.config.setdefault("_extra", {}).update(extra)

    def _resnets(self):
        for blk in self.down_blocks:
            yield from blk.resnets
        yield from self.mid_block.resnets
        for blk in self.up_blocks:
            yield from blk.resnets

    def _embed_packed(self):
        te, ce = self.time_embedding, self.class_embedding
        resnets = list(self._resnets())
        params = list(te.parameters()) + (list(ce.parameters()) if ce is not None else [])
        for r in resnets:
            params += [r.time_emb_proj.weight, r.time_emb_proj.bias]

        def build():
            d = dict(w1=_f16(te.linear_1.weight), b1=_f32(te.linear_1.bias),
                     w2=_f16(te.linear_2.weight), b2=_f32(te.linear_2.bias),
                     wall=_f16(torch.cat([r.time_emb_proj.weight for r in resnets], 0)),
                     ball=_f32(torch.cat([r.time_emb_proj.bias for r in resnets], 0)))
            if ce is not None:
                kin = ce.linear_1.weight.shape[1]
                kpad = (kin + 7) // 8 * 8
                w = torch.zeros(ce.linear_1.weight.shape[0], kpad, device=ce.linear_1.weight.device)
                w[:, :kin] = ce.linear_1.weight.detach()
                d.update(cw1=_f16(w), cb1=_f32(ce.linear_1.bias), cw2=_f16(ce.linear_2.weight),
                         cb2=_f32(ce.linear_2.bias), ckpad=kpad)
            offs, o = [], 0
            for r in resnets:
                offs.append(o)
                o += r.cout
            d["offs"] = offs
            return d
        return self._pk.get(params, build)

    # ------------------------------------------------------------------ forward
    # Exact single-step specialisations (SURVEY.md §8 f1) — pure wins on the reference's one-step path, all
    # parity-tested against the general path (tests/engine_checks.py:run_single_step_specialisations):
    #   * constant python-scalar timestep and no class labels (marigold_pipeline.py:452: `t` of the 1-step trailing
    #     schedule is always 999): temb and the 22 stacked `time_emb_proj` outputs are a function of the weights only
    #     -> computed once per weights version (unet_2d_condition.py:974-981), no embedding kernels per call;
    #   * zeros noise (marigold_pipeline.py:418-423): `sample` may carry only the leading channels, conv_in runs on
    #     those (the missing input channels are exact zeros);
    #   * one context shared by the batch (marigold_pipeline.py:428-432; detected without a device sync as a
    #     batch-broadcast view, `stride(0) == 0`, or batch 1): cross-attention collapses to two skinny GEMMs
    #     (modules.BasicTransformerBlock._packed_const_ctx).
    single_step_specialisations = True

    def _time_embedding(self, t, class_labels):
        """[B, sum(cout)] fp32: every resnet's time_emb_proj(silu(temb (+class_emb))) (unet_2d_condition.py:957-1000),
        and the intermediates its backward reads: (out, (e0, e1, e2, cl, c1, c))."""
        ep = self._embed_packed()
        e0 = ops.timestep_embedding(t, self.config["block_out_channels"][0])
        e1 = ops.linear(e0, ep["w1"], ep["b1"], act=ops.ACT_SILU)
        cl = c1 = c = None
        if self.class_embedding is not None:
            cl = torch.zeros((t.shape[0], ep["ckpad"]), dtype=F16, device=t.device)
            cl[:, :class_labels.shape[1]] = class_labels
            c1 = ops.linear(cl, ep["cw1"], ep["cb1"], act=ops.ACT_SILU)
            c = ops.linear(c1, ep["cw2"], ep["cb2"])
        e2 = ops.linear(e1, ep["w2"], ep["b2"], residual=c, act=ops.ACT_SILU)         # silu(temb (+ class_emb))
        return ops.linear(e2, ep["wall"], ep["ball"], out_dtype=F32), (e0, e1, e2, cl, c1, c)   # all 22 time_emb_proj

    def _walk(self, x, temb_of, forward_size, resnet, transformer, downsample, upsample):
        """Down / mid / up blocks from conv_in's output to conv_norm_out's input (unet_2d_condition.py:1005-1206).
        The four steps run one block each, as inference modules or as autograd Functions:
        resnet(block, x, temb, skip, f16_copy), transformer(block, x, f16_copy), downsample(block, x),
        upsample(block, x, out_hw)."""
        skips = [x]
        for blk in self.down_blocks:
            for i, r in enumerate(blk.resnets):
                last = (i == len(blk.resnets) - 1) and blk.downsamplers is not None    # feeds the stride-2 conv
                x = resnet(r, x, temb_of[id(r)], None, last and blk.attentions is None)
                if blk.attentions is not None:
                    x = transformer(blk.attentions[i], x, last)
                skips.append(x)
            if blk.downsamplers is not None:
                x = downsample(blk.downsamplers[0], x)
                skips.append(x)
        mb = self.mid_block
        x = resnet(mb.resnets[0], x, temb_of[id(mb.resnets[0])], None, False)
        x = transformer(mb.attentions[0], x, False)
        x = resnet(mb.resnets[1], x, temb_of[id(mb.resnets[1])], None, False)
        for blk in self.up_blocks:
            for i, r in enumerate(blk.resnets):
                skip = skips.pop()
                last = (i == len(blk.resnets) - 1) and blk.upsamplers is not None and not forward_size
                x = resnet(r, x, temb_of[id(r)], skip, last and blk.attentions is None)
                if blk.attentions is not None:
                    x = transformer(blk.attentions[i], x, last)
            if blk.upsamplers is not None:
                x = upsample(blk.upsamplers[0], x, tuple(skips[-1].shape[1:3]) if forward_size else None)
        return x

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, return_dict=True, **unused):
        """With grad enabled and a parameter or `sample` requiring grad, every block runs as its autograd Function
        (autograd_blocks.py), so `loss.backward()` fills `.grad` like the reference's training/train.py:563."""
        ops._need_cuda(sample)                                                      # sm_90a only, no CPU fallback
        train = torch.is_grad_enabled() and (sample.requires_grad or any(p.requires_grad for p in self.parameters()))
        cfg, sdt = self.config, self.stream_dtype
        if train and sdt != F32:
            raise NotImplementedError("training runs with the fp32 residual stream (stream_dtype=torch.float32)")
        if self.class_embedding is not None and class_labels is None:
            raise ValueError("class_labels should be provided when num_class_embeds > 0")
        B, _, H, W = sample.shape
        dev = sample.device
        n_up = len(cfg["block_out_channels"]) - 1
        forward_size = (H % (2 ** n_up) != 0) or (W % (2 ** n_up) != 0)      # unet_2d_condition.py:920-930
        spec = self.single_step_specialisations and not train
        if sample.shape[1] != cfg["in_channels"] and not (spec and sample.shape[1] < cfg["in_channels"]):
            raise ValueError(f"sample has {sample.shape[1]} channels, conv_in expects {cfg['in_channels']}")

        # ---- time / class embedding (unet_2d_condition.py:957-1000)
        ep = self._embed_packed()
        if spec and not torch.is_tensor(timestep) and self.class_embedding is None:
            cache = ep.setdefault("temb_cache", {})                 # lives and dies with the packed weights
            key = (float(timestep), B, str(dev))
            temb_all = cache.get(key)
            if temb_all is None:
                t = torch.full((B,), float(timestep), dtype=F32, device=dev)
                temb_all = cache[key] = self._time_embedding(t, None)[0]
                if dev.type == "cuda" and torch.cuda.is_current_stream_capturing():
                    cache.pop(key)                                   # graph-private memory must not outlive the capture
        else:
            if not torch.is_tensor(timestep):
                t = torch.full((B,), float(timestep), dtype=F32, device=dev)
            else:
                t = timestep.to(device=dev, dtype=F32).reshape(-1).expand(B).contiguous()
            temb_all = ab.embed(self, t, class_labels) if train else self._time_embedding(t, class_labels)[0]
        resnets = list(self._resnets())
        temb_of = {id(r): temb_all[:, o:o + r.cout] for r, o in zip(resnets, ep["offs"])}

        ehs = encoder_hidden_states.detach()
        const_ctx = None
        if spec and ehs.dim() == 3 and (ehs.shape[0] == 1 or ehs.stride(0) == 0):
            const_ctx = ehs[0]                                      # [S, Dctx] shared by every image
        ctx16 = ehs.to(F16).contiguous()

        if not hasattr(self, "_conv_in_run") or self._conv_in_run.conv is not self.conv_in:
            self._conv_in_run = ConvInSmall(self.conv_in)       # conv_in may be swapped (unet_prep.py:6-21)
        if not hasattr(self, "_conv_out_run") or self._conv_out_run.conv is not self.conv_out:
            self._conv_out_run = ConvOutSmall(self.conv_norm_out, self.conv_out)
        x_in = sample if sample.dtype in (F16, F32) else sample.float()
        if train:
            ck = bool(self._gradient_checkpointing)
            x = ab.conv_in(self._conv_in_run, x_in.detach())
            x = self._walk(x, temb_of, forward_size,
                           lambda r, x, temb, skip, f16_copy: ab.resnet(r, x, temb, skip, f16_copy, ckpt=ck),
                           lambda m, x, f16_copy: ab.transformer(m, x, ctx16, f16_copy, ckpt=ck),
                           ab.downsample, ab.upsample)
            out = ab.conv_out(self._conv_out_run, x)
        else:
            x = self._conv_in_run.run(x_in, sdt)
            x = self._walk(x, temb_of, forward_size,
                           lambda r, x, temb, skip, f16_copy: r.run(x, temb, skip, sdt, f16_copy),
                           lambda m, x, f16_copy: m.run(x, ctx16, sdt, f16_copy, const_ctx),
                           lambda m, x: m.run(x, sdt),
                           lambda m, x, out_hw: m.run(x, out_hw, sdt))
            out = self._conv_out_run.run(x)
        if out.dtype != sample.dtype:
            out = out.to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(out)
