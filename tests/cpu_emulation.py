"""TEST INFRASTRUCTURE ONLY — plain-torch restatements of the contracts of the CUDA kernels behind
`diffusion_e2e_ft_b200.ops` (include/b200_e2eft.h), installed over `ops` by CPU tests so the HOST-side logic that
sequences the kernels (module wiring, saved tensors, operand re-packing of the backward pass) can be exercised
without a GPU.  Never imported by the product; the kernels themselves are checked on the GPU (`-m gpu`)."""
import math

import torch
import torch.nn.functional as F

from diffusion_e2e_ft_b200 import ops

F16, F32 = torch.float16, torch.float32


def tap_conv(x_nhwc, wp, cout, taps, stride=1, out_hw=None, x2=None):
    """sum_t x[n, ho*s+dy_t, wo*s+dx_t, :] @ wp[:, t*Cin:(t+1)*Cin].T (+ x2 @ wp[:, T*Cin:].T); zero outside."""
    NB, H, W, Cin = x_nhwc.shape
    Ho, Wo = out_hw or (H, W)
    wpf = wp.float()
    res = torch.zeros(NB, Ho, Wo, cout)
    pad = 4
    xp = F.pad(x_nhwc.float().permute(0, 3, 1, 2), (pad, pad + stride * Wo, pad, pad + stride * Ho)).permute(0, 2, 3, 1)
    for t, (dy, dx) in enumerate(taps):
        ys = torch.arange(Ho) * stride + dy + pad
        xs = torch.arange(Wo) * stride + dx + pad
        res += xp[:, ys][:, :, xs] @ wpf[:, t * Cin:(t + 1) * Cin].T
    if x2 is not None:
        res += x2.float() @ wpf[:, len(taps) * Cin:].T
    return res


def _act(r, act):
    if act == ops.ACT_EXP2:
        return torch.exp2(r)
    if act == ops.ACT_SILU:
        return F.silu(r)
    if act == ops.ACT_GELU:
        return F.gelu(r)
    assert act == ops.ACT_NONE
    return r


def linear(a, w, bias=None, residual=None, out=None, out_dtype=F16, act=ops.ACT_NONE, alpha=1.0, bias_row=False,
           stats_rows_per_img=0, f16_copy=False, res_mul=False, a_t=False, w_t=False):
    assert a.stride(-1) == 1 and w.stride(-1) == 1 and a.dtype == F16 and w.dtype == F16
    assert a.stride(-2) % 8 == 0 and w.stride(-2) % 8 == 0, "TMA: 16-byte row pitch"
    assert a.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0, "TMA: 16-byte base"
    if a.dim() == 3:
        assert a.stride(0) % 8 == 0
    if w.dim() == 3:
        assert w.stride(0) % 8 == 0
    assert out is None or (out.data_ptr() % 16 == 0 and out.stride(-1) == 1 and out.stride(-2) % 4 == 0)
    af = a.float().transpose(-1, -2) if a_t else a.float()
    wf = w.float() if w_t else w.float().transpose(-1, -2)
    r = af @ wf * alpha
    if bias is not None:
        r = r + (bias.unsqueeze(-1) if bias_row else bias)
    if residual is not None:
        r = r * residual.float() if res_mul else r + residual.float()
    r = _act(r, act)
    if out is None:
        out = r.to(out_dtype)
    else:
        out.copy_(r.to(out.dtype))
    if f16_copy and out.dtype == F32:
        out._h16 = out.half()
    return out


def conv2d(x, wp, cout, bias=None, taps=ops.TAPS3, stride=1, out_hw=None, x2=None, rowvec=None, residual=None,
           out=None, out_dtype=F16, out_nchw=False, act=ops.ACT_NONE, out_mul=1, out_off=(0, 0), stats=None,
           f16_copy=False):
    assert x.dtype == F16 and x.is_contiguous() and wp.dtype == F16 and wp.is_contiguous()
    NB, H, W, Cin = x.shape
    Ho, Wo = out_hw if out_hw is not None else (H, W)
    C2 = x2.shape[3] if x2 is not None else 0
    assert wp.shape == (cout, len(taps) * Cin + C2), (wp.shape, cout, len(taps), Cin, C2)
    r = tap_conv(x, wp, cout, taps, stride, (Ho, Wo), x2)
    if bias is not None:
        r = r + bias
    if rowvec is not None:
        r = r + rowvec.float()[:, None, None, :]
    r = _act(r, act)
    if out is None:
        shape = (NB, cout, Ho * out_mul, Wo * out_mul) if out_nchw else (NB, Ho * out_mul, Wo * out_mul, cout)
        out = torch.zeros(shape, dtype=out_dtype)
    if out_nchw:
        assert out_mul == 1 and residual is None
        out.copy_(r.permute(0, 3, 1, 2).to(out.dtype))
        return out
    sl = (slice(None), slice(out_off[0], None, out_mul), slice(out_off[1], None, out_mul))
    if residual is not None:
        assert residual.shape == out.shape and residual.dtype == out.dtype
        r = r + residual[sl].float()
    out[sl] = r.to(out.dtype)
    if f16_copy and out.dtype == F32:
        out._h16 = out.half()
    return out


def group_norm(x1, gamma, beta, eps, groups=32, silu=True, x2=None, want_raw=False):
    x = x1 if x2 is None else torch.cat([x1, x2], dim=3)
    y = F.group_norm(x.float().permute(0, 3, 1, 2), groups, gamma, beta, eps)
    y = (F.silu(y) if silu else y).permute(0, 2, 3, 1).contiguous().half()
    return (y, x.half().contiguous()) if want_raw else y


def group_norm_mean_rstd(x1, eps, groups=32, x2=None):
    x = (x1 if x2 is None else torch.cat([x1, x2], dim=3)).float()
    NB, H, W, C = x.shape
    g = x.reshape(NB, H * W, groups, C // groups).permute(0, 2, 1, 3).reshape(NB, groups, -1)
    mean = g.mean(-1)
    var = g.var(-1, unbiased=False)
    return torch.stack([mean, 1.0 / torch.sqrt(var + eps)], dim=-1).contiguous()


def group_norm_bwd(xs, dy, mr, gamma, beta, groups=32, silu=True, adds=None, out_dtype=F32):
    assert dy.dtype == F16
    x = torch.cat([t.float() for t in xs], dim=3)
    NB, H, W, C = x.shape
    cpg = C // groups
    mean = mr[..., 0].repeat_interleave(cpg, dim=1)[:, None, None, :]
    rstd = mr[..., 1].repeat_interleave(cpg, dim=1)[:, None, None, :]
    xh = (x - mean) * rstd
    z = xh * gamma + beta
    d = dy.float()
    if silu:
        s = torch.sigmoid(z)
        d = d * s * (1 + z * (1 - s))
    dgamma = (d * xh).sum((0, 1, 2))
    dbeta = d.sum((0, 1, 2))
    dg = d * gamma

    def gmean(t):
        m = t.reshape(NB, H * W, groups, cpg).mean((1, 3))
        return m.repeat_interleave(cpg, dim=1)[:, None, None, :]
    dx = rstd * (dg - gmean(dg) - xh * gmean(dg * xh))
    outs, off = [], 0
    for i, t in enumerate(xs):
        part = dx[..., off:off + t.shape[3]]
        if adds is not None and adds[i] is not None:
            part = part + adds[i].float()
        outs.append(part.to(out_dtype).contiguous())
        off += t.shape[3]
    return outs, dgamma, dbeta


def layer_norm(x, gamma, beta, eps=1e-5):
    return F.layer_norm(x.float(), (x.shape[-1],), gamma, beta, eps).half()


def layer_norm_bwd(x, dy, gamma, eps=1e-5, add=None, out_dtype=F32, dgamma=None, dbeta=None):
    xr = x.float().detach().requires_grad_(True)
    g = gamma.detach().clone().requires_grad_(True)
    b = torch.zeros_like(gamma).requires_grad_(True)
    with torch.enable_grad():
        (F.layer_norm(xr, (x.shape[-1],), g, b, eps) * dy.float()).sum().backward()
    dx = xr.grad + (add.float() if add is not None else 0)
    dg = g.grad if dgamma is None else dgamma.add_(g.grad)
    db = b.grad if dbeta is None else dbeta.add_(b.grad)
    return dx.to(out_dtype), dg, db


def rowdot_heads(a, c, heads):
    B, L = a.shape[0], a.shape[1]
    return (a[..., :heads * 64].float() * c[..., :heads * 64].float()).view(B, L, heads, 64).sum(-1).permute(0, 2, 1).contiguous()


def attention_d64(q, k, v, heads, scale, kv_segments=1, out=None, want_lse=False):
    B, Lq = q.shape[0], q.shape[1]
    if kv_segments == 2:                                   # batch b sees the keys of b % (B/2) then b % (B/2) + B/2
        h = B // 2
        k = torch.cat([torch.cat([k[:h], k[h:]], dim=1)] * 2, dim=0)
        v = torch.cat([torch.cat([v[:h], v[h:]], dim=1)] * 2, dim=0)

    def split(t):
        return t.float().unflatten(-1, (heads, 64)).transpose(1, 2)
    k = k.expand(B, -1, -1) if k.shape[0] == 1 else k
    v = v.expand(B, -1, -1) if v.shape[0] == 1 else v
    logits = split(q) @ split(k).transpose(-1, -2) * scale
    o = torch.softmax(logits, dim=-1) @ split(v)
    o = o.transpose(1, 2).reshape(B, Lq, heads * 64).half()
    if out is not None:
        out.copy_(o)
        o = out
    if want_lse:
        return o, (torch.logsumexp(logits, dim=-1) * 1.4426950408889634).contiguous()      # log2 domain, [B, heads, Lq]
    return o


def softmax_rows(s, scale, cols=None):
    cols = cols or s.shape[-1]
    p = torch.zeros(s.shape, dtype=F16)
    p[..., :cols] = torch.softmax(s[..., :cols] * scale, dim=-1).half()
    return p


def softmax_groups(logits, heads, S, ld_out):
    rows = logits.shape[0]
    p = torch.zeros((rows, ld_out), dtype=F16)
    p[:, :heads * S] = torch.softmax(logits[:, :heads * S].view(rows, heads, S), dim=-1).reshape(rows, heads * S).half()
    return p


def softmax_bwd_rows(p, dp, scale, cols=None):
    cols = cols or p.shape[-1]
    pf, d = p[..., :cols].float(), dp[..., :cols]
    ds = torch.zeros(p.shape, dtype=F16)
    ds[..., :cols] = (scale * pf * (d - (pf * d).sum(-1, keepdim=True))).half()
    return ds


def gather_planar(x, out_hw=None, stride=1, up=1, off=(0, 0), out=None):
    NB, H, W, C = x.shape
    Ho, Wo = out_hw if out_hw is not None else (H, W)
    xu = x.float().permute(0, 3, 1, 2)
    if up == 2:
        xu = F.interpolate(xu, scale_factor=2.0, mode="nearest")
    pad = 4
    xp = F.pad(xu, (pad, pad + stride * Wo, pad, pad + stride * Ho))
    ys = torch.arange(Ho) * stride + off[0] + pad
    xs = torch.arange(Wo) * stride + off[1] + pad
    ref = xp[:, :, ys][:, :, :, xs].permute(1, 0, 2, 3).reshape(C, -1)
    P = NB * Ho * Wo
    if out is None:
        out = torch.zeros(C, ops._ru8(P), dtype=F16)
    else:
        assert out.shape[0] == C and out.stride(1) == 1 and out.stride(0) % 8 == 0
        out.zero_()
    out[:, :P] = ref.half()
    return out


def col_sum(x, out=None):
    r = x.float().sum(0)
    return r if out is None else out.add_(r)


def act_bwd(x, dy, act):
    xr = x.float().detach().requires_grad_(True)
    with torch.enable_grad():
        (_act(xr, act) * dy.float()).sum().backward()
    return xr.grad.half()


def geglu_bwd(hg, dy):
    r = hg.float().detach().requires_grad_(True)
    with torch.enable_grad():
        h, g = r.chunk(2, dim=-1)
        (h * F.gelu(g) * dy.float()).sum().backward()
    return r.grad.half()


def cast_f16(x):
    h = getattr(x, "_h16", None)
    return h if h is not None else x.half()


def im2col3x3(x_nchw, kpad):
    NB, C, H, W = x_nchw.shape
    cols = F.unfold(x_nchw.float(), 3, padding=1)                         # [NB, C*9, HW], (c, ky, kx) order
    cols = cols.view(NB, C, 9, H * W).permute(0, 3, 2, 1).reshape(NB * H * W, 9 * C)   # tap-major, channel-minor
    out = torch.zeros(NB * H * W, kpad, dtype=F16)
    out[:, :9 * C] = cols.half()
    return out


def conv3x3_small_cout(x, wq, bias, cout):
    c = x.shape[3]
    w = wq.float().permute(1, 3, 0, 2, 4).reshape(9, 8, c)[:, :cout]     # [tap][n][c]
    w = w.permute(1, 2, 0).reshape(cout, c, 3, 3)
    return F.conv2d(x.float().permute(0, 3, 1, 2), w, bias, padding=1)


def timestep_embedding(t, dim):
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F32) / half)
    a = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(a), torch.sin(a)], dim=-1).half()        # flip_sin_to_cos=True


def embed_tokens(ids, tok, pos):
    B, L = ids.shape
    return (tok.float()[ids] + pos.float()[:L][None]).reshape(B * L, -1).contiguous()


def nhwc_to_nchw_f32(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


def pointwise_nchw(in1, a1, wm, bias, in2=None, a2=0.0, cin=None):
    cin = cin or wm.shape[1]
    x = a1 * in1[:, :cin].float()
    if in2 is not None:
        x = x + a2 * in2[:, :cin].float()
    return torch.einsum("oc,nchw->nohw", wm[:, :cin].float(), x) + bias.float()[None, :, None, None]


def decode_post(x, normals=False, sign=1.0, training=False):
    if not normals:
        m = x.mean(1, keepdim=True).clamp(-1, 1)
        return m if training else (m + 1) / 2
    u = sign * x / (x.norm(dim=1, keepdim=True) + 1e-5)
    return u.clamp(-1, 1) if training else u


def _ssi(pred, target, mask):
    m = mask.reshape(pred.shape[0], -1).float()
    p, y = pred.reshape(pred.shape[0], -1).float(), target.reshape(pred.shape[0], -1).float()
    a00, a01, a11 = (m * p * p).sum(1), (m * p).sum(1), m.sum(1)
    b0, b1 = (m * p * y).sum(1), (m * y).sum(1)
    det = a00 * a11 - a01 * a01
    ok = det > 0
    safe = torch.where(ok, det, torch.ones_like(det))
    s = torch.where(ok, (a11 * b0 - a01 * b1) / safe, torch.zeros_like(det))
    t = torch.where(ok, (-a01 * b0 + a00 * b1) / safe, torch.zeros_like(det))
    r = (s[:, None] * p + t[:, None] - y).abs() * m
    return r.sum() / m.sum()


def _angular(pred, target, mask):
    d = (pred.float() * target.float()).sum(1).clamp(-1, 1)
    m = mask[:, 0].float()
    return (torch.acos(d) * m).sum() / m.sum()


def ssi_loss(pred, target, mask):
    return _ssi(pred, target, mask)


def angular_loss(pred, target, mask):
    return _angular(pred, target, mask)


def _loss_bwd(fn, pred, target, mask, grad_out):
    p = pred.detach().float().requires_grad_(True)
    with torch.enable_grad():
        (fn(p, target, mask) * grad_out.detach().float()).backward()
    return p.grad


def ssi_loss_bwd(pred, target, mask, grad_out):
    return _loss_bwd(_ssi, pred, target, mask, grad_out)


def angular_loss_bwd(pred, target, mask, grad_out):
    return _loss_bwd(_angular, pred, target, mask, grad_out)


def decode_post_bwd(x, dout, normals=False):
    xr = x.detach().requires_grad_(True)
    with torch.enable_grad():
        (decode_post(xr, normals=normals, training=True) * dout).sum().backward()
    return xr.grad


def grad_norm_sq(flat_grad):
    return flat_grad.double().pow(2).sum().reshape(1)


def adamw_step(param, grad, exp_avg, exp_avg_sq, step, lr=3e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
               grad_norm_sq_t=None, max_grad_norm=0.0, grad_unscale=1.0):
    clip = grad_unscale
    if grad_norm_sq_t is not None and max_grad_norm > 0:
        nrm = float(grad_norm_sq_t.sqrt()) * grad_unscale
        clip = grad_unscale * min(1.0, max_grad_norm / (nrm + 1e-6))
    g = grad * clip
    param.mul_(1 - lr * weight_decay)
    exp_avg.mul_(betas[0]).add_(g, alpha=1 - betas[0])
    exp_avg_sq.mul_(betas[1]).addcmul_(g, g, value=1 - betas[1])
    bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
    param.addcdiv_(exp_avg, exp_avg_sq.sqrt() / math.sqrt(bc2) + eps, value=-lr / bc1)


def adamw_step_state(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t, lr=3e-5, betas=(0.9, 0.999), eps=1e-8,
                     weight_decay=1e-2, max_grad_norm=0.0, inv_world=1.0, dynamic_scale=True, growth_interval=2000,
                     min_scale=1.0, max_scale=65536.0):
    """include/b200_e2eft.h b200_adamw_step_state: state = [scale, tracker, applied, skipped, skip flag, mult, bc1, bc2]."""
    nsq = float(grad_norm_sq_t)
    S = float(state[0])
    unscale = inv_world / S
    if not math.isfinite(nsq) or nsq == 0.0:
        state[3] += 1
        state[4] = 1
        if not math.isfinite(nsq) and dynamic_scale:
            state[0] = max(S * 0.5, min_scale)
            state[1] = 0
        return
    state[2] += 1
    state[4] = 0
    step = int(state[2])
    adamw_step(param, grad, exp_avg, exp_avg_sq, step, lr, betas, eps, weight_decay, grad_norm_sq_t, max_grad_norm, unscale)
    if dynamic_scale:
        state[1] += 1
        if float(state[1]) >= growth_interval:
            state[0] = min(S * 2.0, max_scale)
            state[1] = 0


def _nearest_index(n_in, n_out):
    return torch.clamp((torch.arange(n_out) * n_in) // n_out, max=n_in - 1)


def upsample_nearest(x, out_hw):
    OH, OW = out_hw
    ih, iw = _nearest_index(x.shape[1], OH), _nearest_index(x.shape[2], OW)
    return x[:, ih][:, :, iw].half().contiguous()


def upsample_nearest_bwd(dy, in_hw, add=None):
    H, W = in_hw
    NB, OH, OW, C = dy.shape
    ih, iw = _nearest_index(H, OH), _nearest_index(W, OW)
    dx = torch.zeros(NB, H, W, C)
    tmp = torch.zeros(NB, H, OW, C).index_add_(1, ih, dy.float())
    dx.index_add_(2, iw, tmp)
    return dx if add is None else dx + add


_EMULATED = dict(linear=linear, conv2d=conv2d, group_norm=group_norm, group_norm_mean_rstd=group_norm_mean_rstd,
                 group_norm_bwd=group_norm_bwd, layer_norm=layer_norm, layer_norm_bwd=layer_norm_bwd,
                 attention_d64=attention_d64, rowdot_heads=rowdot_heads, softmax_rows=softmax_rows, softmax_bwd_rows=softmax_bwd_rows,
                 gather_planar=gather_planar, col_sum=col_sum, act_bwd=act_bwd, geglu_bwd=geglu_bwd,
                 softmax_groups=softmax_groups, cast_f16=cast_f16, im2col3x3=im2col3x3, conv3x3_small_cout=conv3x3_small_cout,
                 timestep_embedding=timestep_embedding, embed_tokens=embed_tokens, nhwc_to_nchw_f32=nhwc_to_nchw_f32,
                 pointwise_nchw=pointwise_nchw, decode_post=decode_post, ssi_loss=ssi_loss, angular_loss=angular_loss,
                 ssi_loss_bwd=ssi_loss_bwd, angular_loss_bwd=angular_loss_bwd, decode_post_bwd=decode_post_bwd, grad_norm_sq=grad_norm_sq, adamw_step=adamw_step, adamw_step_state=adamw_step_state,
                 upsample_nearest=upsample_nearest, upsample_nearest_bwd=upsample_nearest_bwd)


def install(monkeypatch):
    for name, fn in _EMULATED.items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(ops, "_need_cuda", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
