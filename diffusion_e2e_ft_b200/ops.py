"""Torch-tensor wrappers over the C ABI (PyTorch tensors in, PyTorch tensors out).

PyTorch only owns memory and streams here: every arithmetic op is a kernel of libb200_e2eft.so
launched on `torch.cuda.current_stream()`.  Nothing in this module computes with torch ops, with two marked
exceptions that are O(channels) in size: dtype conversions of masks / loss inputs at the API boundary and the
final [NB, C, 2] -> [C, 2] fold of the GroupNorm-backward partial sums.
"""
from ctypes import c_float, c_int, c_void_p

import torch

from . import lib as _lib

ACT_NONE, ACT_SILU, ACT_GEGLU, ACT_GELU, ACT_EXP2 = 0, 1, 2, 3, 4
F16, F32 = torch.float16, torch.float32

TAPS3 = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]        # pad=1
TAPS3_PAD0 = [(ky, kx) for ky in range(3) for kx in range(3)]           # VAE downsample (0,1,0,1) pad


class Stats:
    """Launch / algorithmic-FLOP accounting (2*MAC, tensor-pipe ops only: SURVEY.md App. B rules) and
    optional CUDA-event timing of the implicit-GEMM conv launches (bench.py's roofline leg)."""

    def __init__(self):
        self.reset()
        self.time_kind = None          # e.g. "conv": bracket those launches with CUDA events

    def reset(self):
        self.launches = 0
        self.flops = {"conv": 0, "linear": 0, "attn": 0}
        self.count = {"conv": 0, "linear": 0, "attn": 0}
        self.events = []               # (start, end, flops)
        self.lin_events = []

    def add(self, kind=None, flops=0):
        self.launches += 1
        if kind is not None:
            self.flops[kind] += flops
            self.count[kind] += 1

    def timed(self, kind):
        return self.time_kind == kind or self.time_kind == "gemm"


STATS = Stats()
STATS.time_all = False
STATS.op_events = []           # (name, start, end) when time_all


def _timed(name):
    """Bracket an op with CUDA events when STATS.time_all (bench.py's per-op breakdown of an eager step)."""
    def deco(fn):
        def wrapper(*a, **k):
            if not STATS.time_all:
                return fn(*a, **k)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            STATS.op_events.append((name, e0, e1))
            return out
        wrapper.__name__ = fn.__name__
        wrapper.__doc__ = fn.__doc__
        return wrapper
    return deco


def _ck(rc, what):
    _lib.check(rc, what)
    STATS.add()


def _stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("diffusion_e2e_ft_b200 kernels need CUDA tensors (no CPU fallback)")


# ------------------------------------------------------------------------------ weight packing
def pack_conv(w, shortcut_w=None, taps=None):
    """[Cout,Cin,kh,kw] -> fp16 [Cout, taps*Cin (+Cin2)], tap-major / channel-minor (K contiguous)."""
    cout = w.shape[0]
    wp = w.detach().permute(0, 2, 3, 1).reshape(cout, -1)
    if shortcut_w is not None:
        wp = torch.cat([wp, shortcut_w.detach().reshape(cout, -1)], dim=1)
    return wp.to(F16).contiguous()


def pack_conv_small_cin(w, kpad):
    """conv_in weights for the im2col path: [Cout, 9*Cin] zero padded to kpad."""
    cout = w.shape[0]
    wp = w.detach().permute(0, 2, 3, 1).reshape(cout, -1)
    out = torch.zeros(cout, kpad, dtype=F16, device=w.device)
    out[:, :wp.shape[1]] = wp.to(F16)
    return out


def geglu_block_n(n):
    bn = _lib.load().b200_geglu_block_n(int(n))
    if bn == 0:
        raise RuntimeError(f"GEGLU width {n} is not tileable")
    return bn


def pack_geglu(w, b):
    """Interleave value/gate rows per output tile so the epilogue finds both halves in one tile."""
    n = w.shape[0]
    bn = geglu_block_n(n)
    h = bn // 2
    half = n // 2
    idx = []
    for t in range(n // bn):
        idx += list(range(t * h, (t + 1) * h)) + list(range(half + t * h, half + (t + 1) * h))
    idx = torch.tensor(idx, device=w.device)
    return w.detach()[idx].to(F16).contiguous(), b.detach()[idx].to(F32).contiguous()


# ------------------------------------------------------------------------------ GEMM
FUSE_GN_STATS = True     # GroupNorm statistics from the producing GEMM/conv epilogue (no gn_stats pass)


def _new_stats(nb, c, device):
    return torch.zeros((nb, c, 2), dtype=torch.float64, device=device)


@_timed("gemm_linear")
def linear(a, w, bias=None, residual=None, out=None, out_dtype=F16, act=ACT_NONE, alpha=1.0,
           bias_row=False, stats_rows_per_img=0, f16_copy=False, res_mul=False, a_t=False, w_t=False):
    """`stats_rows_per_img` > 0: also accumulate per-(image, channel) sum / sum-of-squares of the output
    (attached to the result as `._cs`) for a following GroupNorm.  `f16_copy`: an fp32 output also gets an
    fp16 twin (`._h16`) written by the same epilogue, so a following GEMM needs no cast pass."""
    """a: [M,K] or [B,M,K] fp16 (last dim contiguous); w: [N,K] or [B,N,K] fp16.
    `a_t` / `w_t`: the operand is given TRANSPOSED-AS-STORED — a: [K,M], w: [K,N] (row-major, last dim contiguous) —
    and is consumed MN-major by the tensor core: out = a.T @ w (a_t, w_t), a @ w (w_t), a.T @ w.T (a_t).  This is how
    the backward pass contracts over rows (weight gradients dY^T X, attention dS^T Q / P^T dO / dS K, data gradients
    dY W) without transposition kernels."""
    _need_cuda(a, w)
    assert a.dtype == F16 and w.dtype == F16 and a.stride(-1) == 1 and w.stride(-1) == 1
    batched = a.dim() == 3 or w.dim() == 3
    B = (a.shape[0] if a.dim() == 3 else w.shape[0]) if batched else 1
    M, K = (a.shape[-1], a.shape[-2]) if a_t else (a.shape[-2], a.shape[-1])
    N = w.shape[-1] if w_t else w.shape[-2]
    assert (w.shape[-2] if w_t else w.shape[-1]) == K, (a.shape, w.shape, a_t, w_t)
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty((B, M, n_out) if batched else (M, n_out), dtype=out_dtype, device=a.device)
    assert out.stride(-1) == 1
    if residual is not None:
        assert residual.dtype == out.dtype and residual.stride(-1) == 1
    cs = None
    if (FUSE_GN_STATS and stats_rows_per_img and not batched and stats_rows_per_img % 64 == 0
            and M % stats_rows_per_img == 0 and (N >= 128 or stats_rows_per_img % 128 == 0)):
        cs = _new_stats(M // stats_rows_per_img, n_out, a.device)
    h16 = torch.empty(out.shape, dtype=F16, device=out.device) if (f16_copy and out.dtype == F32 and out.is_contiguous()) else None
    ev = None
    if STATS.timed("linear"):
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    rc = _lib.load().b200_linear(
        _p(a), a.stride(-2), a.stride(0) if a.dim() == 3 else 0,
        _p(w), w.stride(-2), (w.stride(0) if w.dim() == 3 else 0),
        M, N, K, B, _p(bias), int(bias_row),
        _p(residual), residual.stride(-2) if residual is not None else 0,
        (residual.stride(0) if (residual is not None and batched) else 0),
        _p(out), out.stride(-2), out.stride(0) if batched else 0, int(out.dtype == F32),
        act, float(alpha), _p(cs), int(stats_rows_per_img) if cs is not None else 0, _p(h16), int(res_mul),
        int(a_t), int(w_t), (bias.stride(0) if (bias is not None and bias_row and bias.dim() == 2) else 0), _stream())
    _lib.check(rc, "b200_linear")
    STATS.add("linear", 2 * B * M * N * K)
    if ev is not None:
        ev[1].record()
        STATS.lin_events.append((ev[0], ev[1], 2 * B * M * N * K,
                                 (B, M, N, K, act, residual is not None, str(out.dtype)[6:])))
    if cs is not None:
        out._cs = cs
    if h16 is not None:
        out._h16 = h16
    return out


# ------------------------------------------------------------------------------ conv
@_timed("gemm_conv")
def conv2d(x, wp, cout, bias=None, taps=TAPS3, stride=1, out_hw=None, x2=None, rowvec=None,
           residual=None, out=None, out_dtype=F16, out_nchw=False, act=ACT_NONE,
           out_mul=1, out_off=(0, 0), stats=None, f16_copy=False):
    """`stats`: True -> allocate, or an existing [NB,Cout,2] fp32 tensor to accumulate into; the per-channel
    sums of the output are attached to the result as `._cs` for a following GroupNorm."""
    """x: NHWC fp16 [NB,H,W,Cin]; wp: packed fp16 [Cout, len(taps)*Cin (+C2)]."""
    _need_cuda(x, wp)
    assert x.dtype == F16 and x.is_contiguous() and wp.dtype == F16 and wp.is_contiguous()
    NB, H, W, Cin = x.shape
    Ho, Wo = out_hw if out_hw is not None else (H, W)
    C2 = 0
    if x2 is not None:
        assert x2.dtype == F16 and x2.is_contiguous() and tuple(x2.shape[:3]) == (NB, Ho, Wo)
        C2 = x2.shape[3]
    assert wp.shape == (cout, len(taps) * Cin + C2), (wp.shape, cout, len(taps), Cin, C2)
    if out is None:
        shape = (NB, cout, Ho * out_mul, Wo * out_mul) if out_nchw else (NB, Ho * out_mul, Wo * out_mul, cout)
        out = torch.empty(shape, dtype=out_dtype, device=x.device)
    if residual is not None:
        assert residual.dtype == out.dtype and residual.is_contiguous() and residual.shape == out.shape
    assert out.is_contiguous() and tuple(out.shape) == (
        (NB, cout, Ho * out_mul, Wo * out_mul) if out_nchw else (NB, Ho * out_mul, Wo * out_mul, cout)), out.shape
    cs = None
    if stats is not None and stats is not False and FUSE_GN_STATS and not out_nchw:
        cs = _new_stats(NB, cout, x.device) if stats is True else stats
    h16 = torch.empty(out.shape, dtype=F16, device=out.device) if (f16_copy and out.dtype == F32 and not out_nchw) else None
    dy = (c_int * len(taps))(*[t[0] for t in taps])
    dx = (c_int * len(taps))(*[t[1] for t in taps])
    fl = 2 * NB * Ho * Wo * cout * (len(taps) * Cin + C2)
    ev = None
    if STATS.timed("conv"):
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    rc = _lib.load().b200_conv2d_nhwc(
        _p(x), NB, H, W, Cin, _p(x2), C2, _p(wp), cout, len(taps), dy, dx, stride, Ho, Wo,
        out_mul, out_off[0], out_off[1], _p(bias), _p(rowvec),
        rowvec.stride(0) if rowvec is not None else 0, _p(residual), _p(out),
        int(out.dtype == F32), int(out_nchw), act, _p(cs), _p(h16), _stream())
    _lib.check(rc, "b200_conv2d_nhwc")
    if ev is not None:
        ev[1].record()
        STATS.events.append((ev[0], ev[1], fl, (NB, H, W, Cin, C2, cout, len(taps), stride, str(out.dtype)[6:])))
    STATS.add("conv", fl)
    if cs is not None:
        out._cs = cs
    if h16 is not None:
        out._h16 = h16
    return out


def pack_conv_small_cout(w):
    """[Cout<=8, C, 3, 3] -> fp16 [C/64][9][4][8][16]: per 64-channel chunk, tap, 16-channel k-step the B
    fragment rows (n = output channel, zero padded to 8) of mma.m16n8k16."""
    cout, c = w.shape[0], w.shape[1]
    assert cout <= 8 and c % 64 == 0
    wp = torch.zeros(8, c, 3, 3, dtype=F32, device=w.device)
    wp[:cout] = w.detach().float()
    wp = wp.permute(2, 3, 0, 1).reshape(9, 8, c // 64, 4, 16)        # [tap][n][chunk][ks][k]
    return wp.permute(2, 0, 3, 1, 4).contiguous().to(F16)             # [chunk][tap][ks][n][k]


@_timed("conv_small")
def conv3x3_small_cout(x, wq, bias, cout):
    """x NHWC fp16 -> NCHW fp32 [NB, cout, H, W]."""
    _need_cuda(x, wq)
    assert x.dtype == F16 and x.is_contiguous() and wq.dtype == F16 and wq.is_contiguous()
    NB, H, W, C = x.shape
    out = torch.empty((NB, cout, H, W), dtype=F32, device=x.device)
    _ck(_lib.load().b200_conv3x3_small_cout(_p(x), NB, H, W, C, _p(wq), _p(bias), cout, _p(out), _stream()),
        "b200_conv3x3_small_cout")
    STATS.flops["conv"] += 2 * NB * H * W * cout * 9 * C
    return out


@_timed("im2col")
def im2col3x3(x_nchw, kpad):
    _need_cuda(x_nchw)
    assert x_nchw.is_contiguous() and x_nchw.dtype in (F16, F32)
    NB, C, H, W = x_nchw.shape
    out = torch.empty((NB * H * W, kpad), dtype=F16, device=x_nchw.device)
    rc = _lib.load().b200_im2col3x3_nchw(_p(x_nchw), int(x_nchw.dtype == F32), NB, C, H, W, _p(out), kpad, _stream())
    _ck(rc, "b200_im2col3x3_nchw")
    return out


# ------------------------------------------------------------------------------ norms
@_timed("group_norm")
def group_norm(x1, gamma, beta, eps, groups=32, silu=True, x2=None, want_raw=False):
    """NHWC (fp16 or fp32) -> normalised fp16 NHWC of the channel-concat [x1 | x2]."""
    _need_cuda(x1, x2)
    assert x1.is_contiguous() and (x2 is None or (x2.is_contiguous() and x2.dtype == x1.dtype))
    NB, H, W, C1 = x1.shape
    C2 = x2.shape[3] if x2 is not None else 0
    C = C1 + C2
    f32 = int(x1.dtype == F32)
    L = _lib.load()
    y = torch.empty((NB, H, W, C), dtype=F16, device=x1.device)
    raw = torch.empty_like(y) if want_raw else None
    cs1 = getattr(x1, "_cs", None)
    cs2 = getattr(x2, "_cs", None) if x2 is not None else None
    if FUSE_GN_STATS and cs1 is not None and (x2 is None or cs2 is not None):
        _ck(L.b200_group_norm_apply_cs(_p(x1), C1, _p(cs1), _p(x2), C2, _p(cs2), f32, NB, H * W, groups, _p(gamma),
                                       _p(beta), float(eps), int(silu), _p(y), _p(raw), _stream()),
            "b200_group_norm_apply_cs")
        return (y, raw) if want_raw else y
    sums = torch.zeros((NB, groups, 2), dtype=torch.float64, device=x1.device)
    _ck(L.b200_group_norm_stats(_p(x1), C1, _p(x2), C2, f32, NB, H * W, groups, _p(sums), _stream()),
        "b200_group_norm_stats")
    _ck(L.b200_group_norm_apply(_p(x1), C1, _p(x2), C2, f32, NB, H * W, groups, _p(sums), _p(gamma),
                                _p(beta), float(eps), int(silu), _p(y), _p(raw), _stream()),
        "b200_group_norm_apply")
    return (y, raw) if want_raw else y


@_timed("layer_norm")
def layer_norm(x, gamma, beta, eps=1e-5):
    _need_cuda(x)
    assert x.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    y = torch.empty(x.shape, dtype=F16, device=x.device)
    _ck(_lib.load().b200_layer_norm(_p(x), int(x.dtype == F32), rows, C, _p(gamma), _p(beta), float(eps),
                                           _p(y), _stream()), "b200_layer_norm")
    return y


# ------------------------------------------------------------------------------ attention
HEAD_DIMS = (40, 64, 80, 160)          # head widths the flash kernel is instantiated for


def attention(q, k, v, heads, scale, kv_segments=1, out=None, want_lse=False):
    """Multi-head flash attention with head width D = C / heads, C = q.shape[-1], D in HEAD_DIMS.
    q: [B,Lq,C] view, k/v: [B,Lk,C] views (fp16, last dim contiguous, e.g. column blocks of one fused QKV buffer)
    -> [B,Lq,C].  `kv_segments` = 2: joint attention (batch b attends to the keys of b % (B/2) and b % (B/2) + B/2).
    `want_lse`: also return the log2-domain log-sum-exp of the scaled scores, fp32 [B, heads, Lq]
    (P_ij = exp2(scale * log2(e) * S_ij - lse_i)) for the backward pass.  Width 64 (SD-2) is `attention_d64`."""
    C = q.shape[-1]
    if C % heads or C // heads not in HEAD_DIMS:
        raise ValueError(f"attention: {C} channels over {heads} heads is head width {C / heads:g}, "
                         f"the kernel supports {HEAD_DIMS}")
    if C // heads == 64:
        return attention_d64(q, k, v, heads, scale, kv_segments, out, want_lse)
    return _attention(q, k, v, heads, C // heads, scale, kv_segments, out, want_lse)


def attention_d64(q, k, v, heads, scale, kv_segments=1, out=None, want_lse=False):
    """q: [B,Lq,>=heads*64] view, k/v: [B,Lk,...] views (fp16, last dim contiguous) -> [B,Lq,heads*64].
    `want_lse`: also return the log2-domain log-sum-exp of the scaled scores, fp32 [B, heads, Lq]
    (P_ij = exp2(scale * log2(e) * S_ij - lse_i)) for the backward pass."""
    return _attention(q, k, v, heads, 64, scale, kv_segments, out, want_lse)


@_timed("attention")
def _attention(q, k, v, heads, D, scale, kv_segments, out, want_lse):
    _need_cuda(q, k, v)
    assert q.dtype == F16 and k.dtype == F16 and v.dtype == F16
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    B, Lq = q.shape[0], q.shape[1]
    Lk = k.shape[1]
    if out is None:
        out = torch.empty((B, Lq, heads * D), dtype=F16, device=q.device)
    kb = k.stride(0) if k.shape[0] > 1 else k.stride(1) * Lk
    vb = v.stride(0) if v.shape[0] > 1 else v.stride(1) * Lk
    qb = q.stride(0) if B > 1 else q.stride(1) * Lq
    lse = torch.empty((B, heads, Lq), dtype=F32, device=q.device) if want_lse else None
    rc = _lib.load().b200_attention(_p(q), qb, q.stride(1), _p(k), kb, k.stride(1), _p(v), vb, v.stride(1),
                                    _p(out), out.stride(0) if B > 1 else out.stride(1) * Lq, out.stride(1),
                                    B, heads, D, Lq, Lk, kv_segments, float(scale), _p(lse), _stream())
    _lib.check(rc, "b200_attention")
    STATS.add("attn", 4 * B * heads * Lq * Lk * kv_segments * D)
    return (out, lse) if want_lse else out


def _bstride(t, L):
    """Batch stride of a [B, L, C] view as the kernels take it (a single batch element may have any stride(0))."""
    return t.stride(0) if t.shape[0] > 1 else t.stride(1) * L


@_timed("attention_bwd")
def attention_bwd(q, k, v, do, lse, delta, dq, dk, dv, heads, scale, kv_segments=1):
    """Fused flash attention backward (b200_attention_bwd): q / do / dq [B,Lq,C], k / v / dk / dv [B,Lk,C] fp16 views
    (last dim contiguous, e.g. column blocks of fused QKV / d(QKV) buffers), lse / delta fp32 [B, heads, Lq] from
    `attention(..., want_lse=True)` and `rowdot_heads_d(do, out, ...)`.  Writes dq, dk, dv; P and dS stay on chip."""
    _need_cuda(q, k, v, do, dq, dk, dv)
    C = q.shape[-1]
    D = C // heads
    B, Lq, Lk = q.shape[0], q.shape[1], k.shape[1]
    for t in (q, k, v, do, dq, dk, dv):
        assert t.dtype == F16 and t.stride(-1) == 1 and t.shape[-1] == C, (t.dtype, t.shape, t.stride())
    assert lse.dtype == F32 and delta.dtype == F32 and lse.is_contiguous() and delta.is_contiguous()
    assert tuple(lse.shape) == (B, heads, Lq) and tuple(delta.shape) == (B, heads, Lq)
    rc = _lib.load().b200_attention_bwd(
        _p(q), _bstride(q, Lq), q.stride(1), _p(k), _bstride(k, Lk), k.stride(1), _p(v), _bstride(v, Lk), v.stride(1),
        _p(do), _bstride(do, Lq), do.stride(1), _p(lse), _p(delta), _p(dq), _bstride(dq, Lq), dq.stride(1),
        _p(dk), _bstride(dk, Lk), dk.stride(1), _p(dv), _bstride(dv, Lk), dv.stride(1),
        B, heads, D, Lq, Lk, kv_segments, float(scale), _stream())
    _lib.check(rc, "b200_attention_bwd")
    STATS.add("attn", 10 * B * heads * Lq * Lk * kv_segments * D)       # the 5 products of the backward
    return dq, dk, dv


@_timed("attention")
def attention_d512(q, k, v, scale, out=None, want_lse=False):
    """One head of width 512 (VAE mid-block): q [B,Lq,512], k/v [B,Lk,512] fp16 views (last dim contiguous, e.g.
    slices of one fused [B, L, 1536] projection) -> fp16 [B,Lq,512].  Flash kernel: no L x L buffer.
    `want_lse`: also return the log2-domain log-sum-exp of the scaled scores, fp32 [B, Lq] (P_ij = exp2(scale *
    log2(e) * S_ij - lse_i)) for `attention_d512_bwd`; the output has the same bits either way."""
    _need_cuda(q, k, v)
    assert q.dtype == F16 and k.dtype == F16 and v.dtype == F16
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    assert q.shape[-1] == 512 and k.shape[-1] == 512 and v.shape[-1] == 512
    B, Lq = q.shape[0], q.shape[1]
    Lk = k.shape[1]
    assert k.shape[0] == B and v.shape[:2] == k.shape[:2]
    if out is None:
        out = torch.empty((B, Lq, 512), dtype=F16, device=q.device)
    assert out.dtype == F16 and out.stride(-1) == 1 and tuple(out.shape) == (B, Lq, 512)
    qb = q.stride(0) if B > 1 else q.stride(1) * Lq
    kb = k.stride(0) if B > 1 else k.stride(1) * Lk
    vb = v.stride(0) if B > 1 else v.stride(1) * Lk
    ob = out.stride(0) if B > 1 else out.stride(1) * Lq
    args = (_p(q), qb, q.stride(1), _p(k), kb, k.stride(1), _p(v), vb, v.stride(1), _p(out), ob, out.stride(1),
            B, Lq, Lk, float(scale))
    if want_lse:
        lse = torch.empty((B, Lq), dtype=F32, device=q.device)
        _lib.check(_lib.load().b200_attention_d512_lse(*args, _p(lse), _stream()), "b200_attention_d512_lse")
    else:
        _lib.check(_lib.load().b200_attention_d512(*args, _stream()), "b200_attention_d512")
    STATS.add("attn", 4 * B * Lq * Lk * 512)
    return (out, lse) if want_lse else out


@_timed("bwd_misc")
def rowdot_d512(a, c):
    """delta[b, l] = sum_d a[b, l, d] * c[b, l, d] over 512 columns; a, c fp16 [B, L, 512] views (last dim
    contiguous) -> fp32 [B, L]: the delta = rowsum(dO * O) of `attention_d512_bwd`."""
    _need_cuda(a, c)
    assert a.dtype == F16 and c.dtype == F16 and a.stride(-1) == 1 and c.stride(-1) == 1
    assert a.shape[-1] == 512 and c.shape == a.shape
    B, L = a.shape[0], a.shape[1]
    out = torch.empty((B, L), dtype=F32, device=a.device)
    _ck(_lib.load().b200_rowdot_d512(_p(a), _bstride(a, L), a.stride(1), _p(c), _bstride(c, L), c.stride(1), B, L,
                                     _p(out), _stream()), "b200_rowdot_d512")
    return out


@_timed("attention_bwd")
def attention_d512_bwd(q, k, v, do, lse, delta, dq, dk, dv, scale):
    """Fused flash attention backward of `attention_d512` (b200_attention_d512_bwd): q / do / dq [B,Lq,512],
    k / v / dk / dv [B,Lk,512] fp16 views (last dim contiguous, e.g. column blocks of fused QKV / d(QKV) buffers),
    lse fp32 [B, Lq] from `attention_d512(..., want_lse=True)`, delta fp32 [B, Lq] from `rowdot_d512(do, out)`.
    Writes dq, dk, dv; P and dS stay on chip."""
    _need_cuda(q, k, v, do, dq, dk, dv)
    B, Lq, Lk = q.shape[0], q.shape[1], k.shape[1]
    for t, L in ((q, Lq), (k, Lk), (v, Lk), (do, Lq), (dq, Lq), (dk, Lk), (dv, Lk)):
        assert t.dtype == F16 and t.stride(-1) == 1 and tuple(t.shape) == (B, L, 512), (t.dtype, t.shape, t.stride())
    assert lse.dtype == F32 and delta.dtype == F32 and lse.is_contiguous() and delta.is_contiguous()
    assert tuple(lse.shape) == (B, Lq) and tuple(delta.shape) == (B, Lq)
    rc = _lib.load().b200_attention_d512_bwd(
        _p(q), _bstride(q, Lq), q.stride(1), _p(k), _bstride(k, Lk), k.stride(1), _p(v), _bstride(v, Lk), v.stride(1),
        _p(do), _bstride(do, Lq), do.stride(1), _p(lse), _p(delta), _p(dq), _bstride(dq, Lq), dq.stride(1),
        _p(dk), _bstride(dk, Lk), dk.stride(1), _p(dv), _bstride(dv, Lk), dv.stride(1), B, Lq, Lk, float(scale),
        _stream())
    _lib.check(rc, "b200_attention_d512_bwd")
    STATS.add("attn", 10 * B * Lq * Lk * 512)       # the 5 products of the backward
    return dq, dk, dv


def rowdot_heads(a, c, heads):
    """delta[b, h, t] = sum_d a[b, t, h*64+d] * c[b, t, h*64+d]; a, c fp16 [B, L, >=heads*64] views -> fp32 [B, heads, L]."""
    return _rowdot_heads(a, c, heads, 64)


def rowdot_heads_d(a, c, heads, head_dim):
    """delta[b, h, t] = sum_d a[b, t, h*D+d] * c[b, t, h*D+d] with D = head_dim in HEAD_DIMS; a, c fp16
    [B, L, >=heads*D] views -> fp32 [B, heads, L].  Width 64 is `rowdot_heads`."""
    if head_dim == 64:
        return rowdot_heads(a, c, heads)
    return _rowdot_heads(a, c, heads, head_dim)


@_timed("bwd_misc")
def _rowdot_heads(a, c, heads, head_dim):
    _need_cuda(a, c)
    assert a.dtype == F16 and c.dtype == F16 and a.stride(-1) == 1 and c.stride(-1) == 1 and a.shape[:2] == c.shape[:2]
    B, L = a.shape[0], a.shape[1]
    out = torch.empty((B, heads, L), dtype=F32, device=a.device)
    _ck(_lib.load().b200_rowdot_heads_d(_p(a), a.stride(0), a.stride(1), _p(c), c.stride(0), c.stride(1), B, L, heads,
                                        int(head_dim), _p(out), _stream()), "b200_rowdot_heads_d")
    return out


@_timed("softmax_rows")
def softmax_rows(s, scale, cols=None):
    """softmax(scale*s) over the last dim -> fp16, same (possibly padded) layout.  `cols` = valid
    columns when the last dim is padded (row stride = s.shape[-1])."""
    _need_cuda(s)
    assert s.dtype == F32 and s.is_contiguous()
    ld = s.shape[-1]
    cols = cols or ld
    rows = s.numel() // ld
    p = (torch.zeros if cols != ld else torch.empty)(s.shape, dtype=F16, device=s.device)   # padding stays 0
    _ck(_lib.load().b200_softmax_rows(_p(s), ld, _p(p), ld, rows, cols, float(scale), _stream()),
               "b200_softmax_rows")
    return p


@_timed("softmax_rows")
def softmax_groups(logits, heads, S, ld_out):
    """logits fp32 [rows, ld_in] (column head*S+s) -> per-head softmax over the S keys, fp16 [rows, ld_out] with the
    padding columns zeroed (constant-context cross-attention, SURVEY.md §8 f1)."""
    _need_cuda(logits)
    assert logits.dtype == F32 and logits.is_contiguous() and logits.dim() == 2
    rows, ld_in = logits.shape
    p = torch.empty((rows, ld_out), dtype=F16, device=logits.device)
    _ck(_lib.load().b200_softmax_groups(_p(logits), ld_in, rows, heads, S, _p(p), ld_out, _stream()),
        "b200_softmax_groups")
    return p


# ------------------------------------------------------------------------------ elementwise
@_timed("upsample")
def upsample_nearest(x, out_hw):
    _need_cuda(x)
    assert x.is_contiguous()
    NB, H, W, C = x.shape
    OH, OW = out_hw
    y = torch.empty((NB, OH, OW, C), dtype=F16, device=x.device)
    _ck(_lib.load().b200_upsample_nearest_nhwc(_p(x), int(x.dtype == F32), NB, H, W, C, OH, OW, _p(y),
                                                      _stream()), "b200_upsample_nearest_nhwc")
    return y


@_timed("misc")
def timestep_embedding(t, dim):
    _need_cuda(t)
    assert t.dtype == F32 and t.is_contiguous()
    out = torch.empty((t.shape[0], dim), dtype=F16, device=t.device)
    _ck(_lib.load().b200_timestep_embedding(_p(t), t.shape[0], dim, _p(out), _stream()),
               "b200_timestep_embedding")
    return out


@_timed("misc")
def embed_tokens(ids, tok, pos):
    """CLIP text embeddings: ids [B, L] int64, tables [vocab, C] / [max_pos, C] (fp16 or fp32) -> fp32 [B*L, C]."""
    _need_cuda(ids, tok, pos)
    assert ids.dtype == torch.long and ids.is_contiguous() and tok.dtype == pos.dtype and tok.dtype in (F16, F32)
    B, L = ids.shape
    C = tok.shape[1]
    tok, pos = tok.detach().contiguous(), pos.detach().contiguous()
    out = torch.empty((B * L, C), dtype=F32, device=ids.device)
    _ck(_lib.load().b200_embed_tokens(_p(ids), _p(tok), _p(pos), int(tok.dtype == F32), B * L, L, C, tok.shape[0],
                                      _p(out), _stream()), "b200_embed_tokens")
    return out


def pointwise_nchw(in1, a1, wm, bias, in2=None, a2=0.0, cin=None):
    """out[n,co] = sum_ci wm[co,ci]*(a1*in1[n,ci] + a2*in2[n,ci]) + bias[co]; fp32 NCHW, C<=8."""
    _need_cuda(in1)
    assert in1.dtype == F32 and in1.is_contiguous() and (in2 is None or (in2.dtype == F32 and in2.is_contiguous()))
    NB, Cs, H, W = in1.shape
    cout, cin_ = wm.shape
    cin = cin or cin_
    out = torch.empty((NB, cout, H, W), dtype=F32, device=in1.device)
    _ck(_lib.load().b200_pointwise_nchw(_p(in1), float(a1), _p(in2), float(a2), Cs, _p(wm), _p(bias), NB,
                                               cin, cout, H * W, _p(out), _stream()), "b200_pointwise_nchw")
    return out


PREDICTION_TYPES = {"epsilon": 0, "v_prediction": 1, "sample": 2}      # B200_PRED_* of include/b200_e2eft.h


def _nchw_inner_contiguous(t):
    _, C, H, W = t.shape
    return t.stride(3) == 1 and t.stride(2) == W and t.stride(1) == H * W


@_timed("misc")
def ddim_step(model_out, sample, alpha_prod_t, alpha_prod_t_prev, prediction_type="v_prediction", out=None,
              want_x0=False, unet_in=None):
    """DDIM update with eta = 0 (diffusers DDIMScheduler.step) -> (prev_sample fp32, pred_original_sample fp32 or None).
    model_out [B,C,H,W] fp16/fp32 and sample (fp32, None = exact zeros) may be batch-strided; `out` (fp32, contiguous)
    may be `sample` itself.  `unet_in`: a [B,C,H,W] fp16/fp32 view (e.g. channels 4..7 of the next UNet input) that
    also receives prev_sample cast to its dtype."""
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type {prediction_type!r} is not one of {sorted(PREDICTION_TYPES)}")
    _need_cuda(model_out, sample, out, unet_in)
    assert model_out.dim() == 4 and model_out.dtype in (F16, F32) and _nchw_inner_contiguous(model_out)
    B, C, H, W = model_out.shape
    if sample is not None:
        assert sample.shape == model_out.shape and sample.dtype == F32 and _nchw_inner_contiguous(sample)
    if out is None:
        out = torch.empty((B, C, H, W), dtype=F32, device=model_out.device)
    assert out.shape == model_out.shape and out.dtype == F32 and out.is_contiguous()
    x0 = torch.empty((B, C, H, W), dtype=F32, device=model_out.device) if want_x0 else None
    if unet_in is not None:
        assert unet_in.shape == model_out.shape and unet_in.dtype in (F16, F32) and _nchw_inner_contiguous(unet_in)
    _ck(_lib.load().b200_ddim_step(_p(model_out), int(model_out.dtype == F16), model_out.stride(0), _p(sample),
                                   sample.stride(0) if sample is not None else 0, B, C, H * W,
                                   PREDICTION_TYPES[prediction_type], float(alpha_prod_t), float(alpha_prod_t_prev),
                                   _p(out), _p(x0), _p(unet_in), int(unet_in is not None and unet_in.dtype == F16),
                                   unet_in.stride(0) if unet_in is not None else 0, _stream()), "b200_ddim_step")
    return out, x0


@_timed("misc")
def decode_post(x, normals=False, sign=1.0, training=False):
    """`training`: the train.py:532-540 variants (no (x+1)/2 map for depth; clamp after normalising)."""
    _need_cuda(x)
    assert x.dtype == F32 and x.is_contiguous() and x.shape[1] == 3
    NB, _, H, W = x.shape
    out = torch.empty((NB, 3 if normals else 1, H, W), dtype=F32, device=x.device)
    mode = int(normals) + (2 if training else 0)
    _ck(_lib.load().b200_decode_post(_p(x), NB, H * W, mode, float(sign), _p(out), _stream()),
        "b200_decode_post")
    return out


@_timed("loss")
def ssi_loss(pred, target, mask):
    """ScaleAndShiftInvariantLoss forward (training/util/loss.py:13-47): pred/target [B,1,H,W] fp32, mask bool."""
    _need_cuda(pred, target, mask)
    B = pred.shape[0]
    hw = pred.numel() // B
    p, t = pred.float().contiguous(), target.float().contiguous()
    m = mask.reshape(B, -1).to(torch.uint8).contiguous()
    ws = torch.zeros(5 * B + 2, dtype=torch.float64, device=pred.device)
    out = torch.empty(1, dtype=F32, device=pred.device)
    _ck(_lib.load().b200_ssi_loss(_p(p), _p(t), _p(m), B, hw, _p(ws), _p(out), _stream()), "b200_ssi_loss")
    return out[0]


@_timed("loss")
def angular_loss(pred, target, mask):
    """AngularLoss forward (training/util/loss.py:51-67): pred/target [B,3,H,W] fp32, mask [B,1,H,W] bool."""
    _need_cuda(pred, target, mask)
    B = pred.shape[0]
    hw = pred.numel() // (3 * B)
    p, t = pred.float().contiguous(), target.float().contiguous()
    m = mask.reshape(B, -1).to(torch.uint8).contiguous()
    ws = torch.zeros(2, dtype=torch.float64, device=pred.device)
    out = torch.empty(1, dtype=F32, device=pred.device)
    _ck(_lib.load().b200_angular_loss(_p(p), _p(t), _p(m), B, hw, _p(ws), _p(out), _stream()), "b200_angular_loss")
    return out[0]


@_timed("optim")
def grad_norm_sq(flat_grad):
    """Sum of squares of a flat fp32 gradient buffer -> 0-d float64 device tensor (no host sync)."""
    _need_cuda(flat_grad)
    assert flat_grad.dtype == F32 and flat_grad.is_contiguous()
    out = torch.zeros(1, dtype=torch.float64, device=flat_grad.device)
    _ck(_lib.load().b200_sumsq(_p(flat_grad), flat_grad.numel(), _p(out), _stream()), "b200_sumsq")
    return out


@_timed("optim")
def adamw_step(param, grad, exp_avg, exp_avg_sq, step, lr=3e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
               grad_norm_sq_t=None, max_grad_norm=0.0, grad_unscale=1.0):
    """Fused clip_grad_norm_ + AdamW on flat fp32 buffers, in place (training/train.py:346-353,564-566).
    `grad_unscale` = 1 / loss scale when `grad` (and `grad_norm_sq_t`) hold loss-scaled gradients."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq)
    for t in (param, grad, exp_avg, exp_avg_sq):
        assert t.dtype == F32 and t.is_contiguous() and t.numel() == param.numel()
    _ck(_lib.load().b200_adamw_step_scaled(_p(param), _p(grad), _p(exp_avg), _p(exp_avg_sq), param.numel(), float(lr),
                                           float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step),
                                           _p(grad_norm_sq_t), float(max_grad_norm), float(grad_unscale), _stream()),
        "b200_adamw_step_scaled")


@_timed("optim")
def adamw_step_state(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t, lr=3e-5, betas=(0.9, 0.999), eps=1e-8,
                     weight_decay=1e-2, max_grad_norm=0.0, inv_world=1.0, dynamic_scale=True, growth_interval=2000,
                     min_scale=1.0, max_scale=65536.0):
    """Fused clip + AdamW driven by the device-side `state` block (fp32[8], see include/b200_e2eft.h): skipped steps
    (non-finite / all-zero gradient) and dynamic loss scaling without a host sync."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t)
    for t in (param, grad, exp_avg, exp_avg_sq):
        assert t.dtype == F32 and t.is_contiguous() and t.numel() == param.numel()
    assert state.dtype == F32 and state.numel() == 8 and state.is_contiguous()
    _ck(_lib.load().b200_adamw_step_state(_p(param), _p(grad), _p(exp_avg), _p(exp_avg_sq), param.numel(), float(lr),
                                          float(betas[0]), float(betas[1]), float(eps), float(weight_decay),
                                          _p(grad_norm_sq_t), float(max_grad_norm), float(inv_world), _p(state),
                                          int(dynamic_scale), float(growth_interval), float(min_scale), float(max_scale),
                                          _stream()), "b200_adamw_step_state")


ADAMW_MAX_GROUPS, ADAMW_MAX_RUNS = 16, 1024            # B200_ADAMW_MAX_GROUPS / B200_ADAMW_MAX_RUNS


def adamw_run_table(starts, groups, n, n_groups, device):
    """Check a run table on the host and put it on the device: run r covers [starts[r], starts[r+1]) of a flat
    buffer of n elements and belongs to group groups[r].  Returns (run_start int64, run_group int32) device tensors."""
    starts, groups = [int(s) for s in starts], [int(k) for k in groups]
    if not 1 <= len(starts) <= ADAMW_MAX_RUNS or len(groups) != len(starts):
        raise ValueError(f"a run table has 1..{ADAMW_MAX_RUNS} runs with one group each, got {len(starts)} starts and "
                         f"{len(groups)} groups")
    if not 1 <= n_groups <= ADAMW_MAX_GROUPS:
        raise ValueError(f"1..{ADAMW_MAX_GROUPS} parameter groups, got {n_groups}")
    if starts[0] != 0 or any(b <= a for a, b in zip(starts, starts[1:])) or starts[-1] >= n or any(s % 4 for s in starts):
        raise ValueError("run starts must begin at 0, increase, stay below the buffer size and be multiples of 4")
    if any(not 0 <= k < n_groups for k in groups):
        raise ValueError(f"run groups must lie in [0, {n_groups})")
    return (torch.tensor(starts, dtype=torch.int64).to(device), torch.tensor(groups, dtype=torch.int32).to(device))


@_timed("optim")
def adamw_step_state_groups(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t, run_start, run_group, group_lr,
                            group_wd, betas=(0.9, 0.999), eps=1e-8, max_grad_norm=0.0, inv_world=1.0, dynamic_scale=True,
                            growth_interval=2000, min_scale=1.0, max_scale=65536.0):
    """`adamw_step_state` with per-group learning rate and weight decay (torch.optim.AdamW parameter groups,
    train_depth_normal.py:428-444): `run_start` / `run_group` from `adamw_run_table`, `group_lr` / `group_wd` one
    float per group.  One skip decision, loss scale and bias correction for all groups, as in torch."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t, run_start, run_group)
    for t in (param, grad, exp_avg, exp_avg_sq):
        assert t.dtype == F32 and t.is_contiguous() and t.numel() == param.numel()
    assert state.dtype == F32 and state.numel() == 8 and state.is_contiguous()
    assert run_start.dtype == torch.int64 and run_group.dtype == torch.int32 and run_start.is_contiguous() \
        and run_group.is_contiguous() and run_start.numel() == run_group.numel()
    n_groups = len(group_lr)
    if len(group_wd) != n_groups or not 1 <= n_groups <= ADAMW_MAX_GROUPS:
        raise ValueError(f"one lr and one weight_decay per group, 1..{ADAMW_MAX_GROUPS} groups")
    lr_h, wd_h = (c_float * n_groups)(*map(float, group_lr)), (c_float * n_groups)(*map(float, group_wd))
    _ck(_lib.load().b200_adamw_step_state_groups(_p(param), _p(grad), _p(exp_avg), _p(exp_avg_sq), param.numel(),
                                                 _p(run_start), _p(run_group), run_start.numel(), lr_h, wd_h, n_groups,
                                                 float(betas[0]), float(betas[1]), float(eps), _p(grad_norm_sq_t),
                                                 float(max_grad_norm), float(inv_world), _p(state), int(dynamic_scale),
                                                 float(growth_interval), float(min_scale), float(max_scale), _stream()),
        "b200_adamw_step_state_groups")


@_timed("cast")
def cast_f16(x):
    h = getattr(x, "_h16", None)
    if h is not None:                      # the producing epilogue already wrote the fp16 twin
        return h
    _need_cuda(x)
    assert x.dtype == F32 and x.is_contiguous()
    y = torch.empty(x.shape, dtype=F16, device=x.device)
    _ck(_lib.load().b200_cast_f32_to_f16(_p(x), _p(y), x.numel(), _stream()), "b200_cast_f32_to_f16")
    return y


@_timed("misc")
def nhwc_to_nchw_f32(x):
    _need_cuda(x)
    assert x.is_contiguous()
    NB, H, W, C = x.shape
    y = torch.empty((NB, C, H, W), dtype=F32, device=x.device)
    _ck(_lib.load().b200_nhwc_to_nchw_f32(_p(x), int(x.dtype == F32), NB, C, H * W, _p(y), _stream()),
               "b200_nhwc_to_nchw_f32")
    return y


# ------------------------------------------------------------------------------ backward-pass kernels (row a10)
def _ru8(n):
    return (n + 7) // 8 * 8


@_timed("bwd_gather")
def gather_planar(x, out_hw=None, stride=1, up=1, off=(0, 0), out=None):
    """x: [NB,H,W,C] fp16/fp32 whose last dim is contiguous and whose pixels are uniformly strided (a channel
    slice of an NHWC tensor is fine) -> fp16 [C, ru8(NB*Ho*Wo)] with
    out[c][(n*Ho+o)*Wo+p] = x[n, (stride*o+off_y)//up, (stride*p+off_x)//up, c] (zero outside / in the padding)."""
    _need_cuda(x)
    NB, H, W, C = x.shape
    assert x.stride(3) == 1 and x.stride(1) == W * x.stride(2) and (NB == 1 or x.stride(0) == H * x.stride(1)), x.stride()
    Ho, Wo = out_hw if out_hw is not None else (H, W)
    P = NB * Ho * Wo
    if out is None:
        out = torch.empty((C, _ru8(P)), dtype=F16, device=x.device)
    assert out.dtype == F16 and out.shape[0] == C and out.shape[1] >= P and out.is_contiguous() and out.shape[1] % 8 == 0
    _ck(_lib.load().b200_gather_planar(_p(x), int(x.dtype == F32), x.stride(2), NB, H, W, C, Ho, Wo, stride, up,
                                       off[0], off[1], _p(out), out.stride(0), _stream()), "b200_gather_planar")
    return out


def transpose_rows(a):
    """[R, C] (row-strided view allowed) -> fp16 [C, ru8(R)], zero padded."""
    assert a.dim() == 2
    R, ld = a.shape[0], a.stride(0)
    return gather_planar(a.as_strided((1, 1, R, a.shape[1]), (R * ld, R * ld, ld, 1), a.storage_offset()))


@_timed("bwd_misc")
def col_sum(x, out=None):
    """sum over rows of a [rows, C] (row-strided) fp16/fp32 matrix -> fp32 [C] (accumulated into `out`)."""
    _need_cuda(x)
    assert x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.zeros((x.shape[1],), dtype=F32, device=x.device)
    _ck(_lib.load().b200_col_sum(_p(x), int(x.dtype == F32), x.shape[0], x.shape[1], x.stride(0), _p(out), _stream()),
        "b200_col_sum")
    return out


def group_norm_mean_rstd(x1, eps, groups=32, x2=None):
    """(mean, rstd) [NB, groups, 2] fp32 of the channel-concat [x1 | x2], from the per-channel sums attached by
    the producing kernels when present, else by a statistics pass."""
    _need_cuda(x1, x2)
    NB, H, W, C1 = x1.shape
    C2 = x2.shape[3] if x2 is not None else 0
    L = _lib.load()
    mr = torch.empty((NB, groups, 2), dtype=F32, device=x1.device)
    cs1 = getattr(x1, "_cs", None)
    cs2 = getattr(x2, "_cs", None) if x2 is not None else None
    if FUSE_GN_STATS and cs1 is not None and (x2 is None or cs2 is not None):
        _ck(L.b200_group_norm_mean_rstd(None, _p(cs1), C1, _p(cs2), C2, NB, H * W, groups, float(eps), _p(mr), _stream()),
            "b200_group_norm_mean_rstd")
        return mr
    sums = torch.zeros((NB, groups, 2), dtype=torch.float64, device=x1.device)
    _ck(L.b200_group_norm_stats(_p(x1), C1, _p(x2), C2, int(x1.dtype == F32), NB, H * W, groups, _p(sums), _stream()),
        "b200_group_norm_stats")
    _ck(L.b200_group_norm_mean_rstd(_p(sums), None, C1, None, C2, NB, H * W, groups, float(eps), _p(mr), _stream()),
        "b200_group_norm_mean_rstd")
    return mr


@_timed("bwd_group_norm")
def group_norm_bwd(xs, dy, mr, gamma, beta, groups=32, silu=True, adds=None, out_dtype=F32):
    """Backward of group_norm over the channel-concat of `xs` (list of 1 or 2 NHWC tensors).  dy: fp16
    [NB,H,W,sum C].  Returns ([dx per input], dgamma, dbeta); `adds[i]` (same shape/dtype as dx_i) is added."""
    _need_cuda(dy, *xs)
    assert dy.dtype == F16 and dy.is_contiguous()
    NB, H, W, Ctot = dy.shape
    assert sum(x.shape[3] for x in xs) == Ctot
    L = _lib.load()
    S = torch.zeros((NB, Ctot, 2), dtype=F32, device=dy.device)
    off = 0
    for x in xs:
        assert x.is_contiguous() and x.shape[:3] == dy.shape[:3]
        _ck(L.b200_group_norm_bwd_sums(_p(x), int(x.dtype == F32), x.shape[3], off, Ctot, _p(dy), NB, H * W, groups,
                                       _p(mr), _p(gamma), _p(beta), int(silu), _p(S), _stream()),
            "b200_group_norm_bwd_sums")
        off += x.shape[3]
    dxs, off = [], 0
    for i, x in enumerate(xs):
        add = adds[i] if adds is not None else None
        dx = torch.empty(x.shape, dtype=out_dtype, device=x.device)
        if add is not None:
            assert add.dtype == out_dtype and add.is_contiguous() and add.shape == x.shape
        _ck(L.b200_group_norm_bwd_apply(_p(x), int(x.dtype == F32), x.shape[3], off, Ctot, _p(dy), NB, H * W, groups,
                                        _p(mr), _p(gamma), _p(beta), int(silu), _p(S), _p(add), _p(dx),
                                        int(out_dtype == F32), _stream()), "b200_group_norm_bwd_apply")
        dxs.append(dx)
        off += x.shape[3]
    dparam = S.sum(0)                       # [Ctot, 2]: (d_beta, d_gamma) — a [NB, C, 2] reduction, host plumbing
    return dxs, dparam[:, 1].contiguous(), dparam[:, 0].contiguous()


@_timed("bwd_layer_norm")
def layer_norm_bwd(x, dy, gamma, eps=1e-5, add=None, out_dtype=F32, dgamma=None, dbeta=None):
    _need_cuda(x, dy)
    assert x.is_contiguous() and dy.is_contiguous() and dy.dtype == F16 and dy.shape == x.shape
    C = x.shape[-1]
    rows = x.numel() // C
    dx = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    if add is not None:
        assert add.dtype == out_dtype and add.is_contiguous() and add.shape == x.shape
    dgamma = torch.zeros((C,), dtype=F32, device=x.device) if dgamma is None else dgamma
    dbeta = torch.zeros((C,), dtype=F32, device=x.device) if dbeta is None else dbeta
    _ck(_lib.load().b200_layer_norm_bwd(_p(x), int(x.dtype == F32), rows, C, _p(gamma), _p(dy), float(eps), _p(add),
                                        _p(dx), int(out_dtype == F32), _p(dgamma), _p(dbeta), _stream()),
        "b200_layer_norm_bwd")
    return dx, dgamma, dbeta


@_timed("bwd_softmax")
def softmax_bwd_rows(p, dp, scale, cols=None):
    """p: fp16 [..., ld] probabilities, dp: fp32 same layout -> dS fp16 (padding columns zero)."""
    _need_cuda(p, dp)
    assert p.dtype == F16 and dp.dtype == F32 and p.is_contiguous() and dp.is_contiguous() and p.shape == dp.shape
    ld = p.shape[-1]
    cols = cols or ld
    ds = (torch.zeros if cols != ld else torch.empty)(p.shape, dtype=F16, device=p.device)
    _ck(_lib.load().b200_softmax_bwd_rows(_p(p), ld, _p(dp), ld, _p(ds), p.numel() // ld, cols, float(scale), _stream()),
        "b200_softmax_bwd_rows")
    return ds


@_timed("bwd_misc")
def act_bwd(x, dy, act):
    _need_cuda(x, dy)
    assert x.dtype == F16 and dy.dtype == F16 and x.is_contiguous() and dy.is_contiguous() and x.shape == dy.shape
    dx = torch.empty_like(x)
    _ck(_lib.load().b200_act_bwd(_p(x), _p(dy), x.numel(), act, _p(dx), _stream()), "b200_act_bwd")
    return dx


@_timed("bwd_misc")
def geglu_bwd(hg, dy):
    """hg: fp16 [rows, 2*inner] = [value | gate] pre-activations of the GEGLU projection; dy: [rows, inner].
    Returns d(hg) [rows, 2*inner] fp16."""
    _need_cuda(hg, dy)
    assert hg.dtype == F16 and dy.dtype == F16 and hg.is_contiguous() and dy.is_contiguous()
    rows, inner = dy.shape
    assert hg.shape == (rows, 2 * inner)
    d = torch.empty_like(hg)
    _ck(_lib.load().b200_geglu_bwd(_p(hg), _p(hg[:, inner:]), 2 * inner, _p(dy), rows, inner, _p(d), _p(d[:, inner:]),
                                   2 * inner, _stream()), "b200_geglu_bwd")
    return d


@_timed("loss")
def ssi_loss_bwd(pred, target, mask, grad_out):
    """d ssi_loss / d pred * grad_out (0-d fp32 device tensor) -> fp32, shape of pred."""
    _need_cuda(pred, target, mask, grad_out)
    B = pred.shape[0]
    hw = pred.numel() // B
    p, t = pred.float().contiguous(), target.float().contiguous()
    m = mask.reshape(B, -1).to(torch.uint8).contiguous()
    ws = torch.zeros(7 * B, dtype=torch.float64, device=pred.device)
    out = torch.empty(p.shape, dtype=F32, device=pred.device)
    go = grad_out.detach().to(F32).reshape(1).contiguous()
    _ck(_lib.load().b200_ssi_loss_bwd(_p(p), _p(t), _p(m), B, hw, _p(ws), _p(go), _p(out), _stream()), "b200_ssi_loss_bwd")
    return out


@_timed("loss")
def angular_loss_bwd(pred, target, mask, grad_out):
    _need_cuda(pred, target, mask, grad_out)
    B = pred.shape[0]
    hw = pred.numel() // (3 * B)
    p, t = pred.float().contiguous(), target.float().contiguous()
    m = mask.reshape(B, -1).to(torch.uint8).contiguous()
    ws = torch.zeros(1, dtype=torch.float64, device=pred.device)
    out = torch.empty(p.shape, dtype=F32, device=pred.device)
    go = grad_out.detach().to(F32).reshape(1).contiguous()
    _ck(_lib.load().b200_angular_loss_bwd(_p(p), _p(t), _p(m), B, hw, _p(ws), _p(go), _p(out), _stream()),
        "b200_angular_loss_bwd")
    return out


@_timed("misc")
def decode_post_bwd(x, dout, normals=False):
    """Backward of decode_post(..., training=True): x [NB,3,H,W] fp32 decoder output, dout the gradient of the
    estimate ([NB,1,H,W] depth / [NB,3,H,W] normals)."""
    _need_cuda(x, dout)
    assert x.dtype == F32 and x.is_contiguous() and dout.dtype == F32 and dout.is_contiguous()
    NB, _, H, W = x.shape
    dx = torch.empty_like(x)
    _ck(_lib.load().b200_decode_post_bwd(_p(x), _p(dout), NB, H * W, 3 if normals else 2, _p(dx), _stream()),
        "b200_decode_post_bwd")
    return dx


@_timed("bwd_misc")
def upsample_nearest_bwd(dy, in_hw, add=None):
    """dy: fp32 [NB,OH,OW,C] -> fp32 [NB,H,W,C] (+ add): backward of upsample_nearest."""
    _need_cuda(dy, add)
    assert dy.dtype == F32 and dy.is_contiguous()
    NB, OH, OW, C = dy.shape
    H, W = in_hw
    dx = torch.empty((NB, H, W, C), dtype=F32, device=dy.device)
    if add is not None:
        assert add.dtype == F32 and add.is_contiguous() and add.shape == dx.shape
    _ck(_lib.load().b200_upsample_nearest_bwd(_p(dy), NB, H, W, C, OH, OW, _p(add), _p(dx), _stream()),
        "b200_upsample_nearest_bwd")
    return dx


# ------------------------------------------------------------------------------ diffusion objective + EMA (ABI 10)
DIFFUSION_PREDICTION_TYPES = ("epsilon", "v_prediction")     # train_depth_normal.py:677-682


@_timed("misc")
def diffusion_inputs(rgb_latents, x0, noise, timesteps, alphas_cumprod, prediction_type, timesteps_host=None):
    """DDPM add_noise + get_velocity + the UNet-input concatenation (train_depth_normal.py:666-705) in one kernel.
    rgb_latents [B,C,h,w], x0 / noise [2B,C,h,w] fp32 (noise None = zeros), timesteps int64 [2B] on the device,
    alphas_cumprod fp32 [T] on the device.  `timesteps_host`: the host copy of the timesteps for the range check (read
    back from the device when omitted, a sync).  Returns (unet_in [2B,2C,h,w], target [2B,C,h,w]), both fp32."""
    if prediction_type not in DIFFUSION_PREDICTION_TYPES:
        raise ValueError(f"Unknown prediction type {prediction_type}")
    _need_cuda(rgb_latents, x0, noise, timesteps, alphas_cumprod)
    B, C, h, w = rgb_latents.shape
    if tuple(x0.shape) != (2 * B, C, h, w) or (noise is not None and noise.shape != x0.shape):
        raise ValueError(f"x0 / noise must be [2B, C, h, w] = {[2 * B, C, h, w]}, got {list(x0.shape)}"
                         f"{'' if noise is None else ' / ' + str(list(noise.shape))}")
    T = alphas_cumprod.numel()
    th = [int(v) for v in (timesteps_host if timesteps_host is not None else timesteps.cpu()).reshape(-1).tolist()]
    if len(th) != 2 * B or timesteps.numel() != 2 * B:
        raise ValueError(f"timesteps must hold 2B = {2 * B} entries")
    if not all(0 <= v < T for v in th):
        raise ValueError(f"timesteps {th} outside [0, {T})")
    for t in (rgb_latents, x0, noise, alphas_cumprod):
        assert t is None or (t.dtype == F32 and t.is_contiguous())
    assert timesteps.dtype == torch.long and timesteps.is_contiguous()
    unet_in = torch.empty((2 * B, 2 * C, h, w), dtype=F32, device=x0.device)
    target = torch.empty_like(x0)
    _ck(_lib.load().b200_diffusion_inputs(_p(rgb_latents), _p(x0), _p(noise), _p(timesteps), _p(alphas_cumprod), B, C,
                                          h * w, PREDICTION_TYPES[prediction_type], _p(unet_in), _p(target), _stream()),
        "b200_diffusion_inputs")
    return unet_in, target


def latent_mask_shape(val_mask, pred):
    """Checks that ~max_pool2d(~val_mask, 8, 8) has pred's spatial size and one image per pair of halves: the
    reference's `noise_pred[latent_mask]` fails otherwise.  Returns (B, C, H, W, h, w)."""
    if val_mask.dim() != 4 or val_mask.shape[1] != 1:
        raise ValueError(f"val_mask must be [B, 1, H, W], got {list(val_mask.shape)}")
    B, _, H, W = val_mask.shape
    n, C, h, w = pred.shape
    if n != 2 * B or (h, w) != (H // 8, W // 8):
        raise ValueError(f"latent mask [{2 * B}, {C}, {H // 8}, {W // 8}] (max_pool2d 8x8 of val_mask {list(val_mask.shape)}) "
                         f"does not match the prediction {list(pred.shape)}")
    return B, C, H, W, h, w


@_timed("loss")
def masked_latent_mse(pred, target, val_mask):
    """F.mse_loss(pred[latent_mask], target[latent_mask]) with latent_mask = ~max_pool2d(~val_mask, 8, 8) repeated over
    both halves and all channels (train_depth_normal.py:607-609,712-714).  pred [2B,C,h,w] fp32/fp16, target fp32,
    val_mask [B,1,H,W] bool.  Returns (loss 0-d fp32 device tensor, 0 for an empty mask; latent_mask [B,h,w] uint8;
    workspace fp64 [2] = (sum, count)) — the last two feed masked_latent_mse_bwd."""
    _need_cuda(pred, target, val_mask)
    B, C, H, W, h, w = latent_mask_shape(val_mask, pred)
    assert pred.dtype in (F16, F32) and pred.is_contiguous() and target.dtype == F32 and target.is_contiguous()
    assert target.shape == pred.shape
    vm = val_mask if val_mask.dtype in (torch.bool, torch.uint8) else val_mask.to(torch.bool)
    vm = vm.contiguous()
    lm = torch.empty((B, h, w), dtype=torch.uint8, device=pred.device)
    ws = torch.zeros(2, dtype=torch.float64, device=pred.device)
    out = torch.empty(1, dtype=F32, device=pred.device)
    _ck(_lib.load().b200_masked_latent_mse(_p(pred), int(pred.dtype == F16), _p(target), _p(vm), B, C, H, W, h, w,
                                           _p(lm), _p(ws), _p(out), _stream()), "b200_masked_latent_mse")
    return out[0], lm, ws


@_timed("loss")
def masked_latent_mse_bwd(pred, target, latent_mask, workspace, grad_out):
    """d masked_latent_mse / d pred * grad_out (0-d fp32 device tensor) -> pred's dtype and shape."""
    _need_cuda(pred, target, latent_mask, workspace, grad_out)
    assert pred.is_contiguous() and target.is_contiguous() and latent_mask.is_contiguous()
    n, C, h, w = pred.shape
    go = grad_out.detach().to(F32).reshape(1).contiguous()
    grad = torch.empty_like(pred)
    _ck(_lib.load().b200_masked_latent_mse_bwd(_p(pred), int(pred.dtype == F16), _p(target), _p(latent_mask),
                                               _p(workspace), _p(go), n // 2, C, h * w, _p(grad), _stream()),
        "b200_masked_latent_mse_bwd")
    return grad


@_timed("optim")
def ema_update(ema, param, one_minus_decay):
    """ema <- ema - one_minus_decay * (ema - param) over flat fp32 buffers, in place (diffusers EMAModel.step);
    `one_minus_decay` is a host float, so there is no sync."""
    _need_cuda(ema, param)
    assert ema.dtype == F32 and param.dtype == F32 and ema.is_contiguous() and param.is_contiguous()
    assert ema.numel() == param.numel()
    _ck(_lib.load().b200_ema_update(_p(ema), _p(param), ema.numel(), float(one_minus_decay), _stream()),
        "b200_ema_update")
