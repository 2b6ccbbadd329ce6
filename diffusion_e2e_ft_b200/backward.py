"""Backward-pass operators of the fine-tuning step (SURVEY.md §8 row a10; reference training/train.py:545-566,
`accelerator.backward(loss)`), composed from the wgmma GEMM / implicit-GEMM conv kernels with transposed or
re-packed operands plus the streaming kernels in csrc/backward.cu.  Every function here is checked against
torch.autograd on the GPU (tests/kernel_checks.py, `bwd_*`).

Conventions: activations / incoming gradients that feed a GEMM are fp16 (the training step multiplies the loss
by a static loss scale so they stay in range), parameter gradients are fp32, the gradient of the residual stream
is fp32 unless stated.  Weight-gradient GEMMs contract over pixels (K = NB*H*W): both operands are brought into
K-major form by `ops.gather_planar` (one pass each; a later version reads them MN-major straight from the
NHWC tensors through the wgmma descriptor, like V in the attention kernel).
"""
import torch

from . import ops
from .backward_packing import pack_conv_dgrad_s1, pack_conv_dgrad_s2, pack_upsample_conv_dgrad
from .ops import F16, F32, TAPS3


# ------------------------------------------------------------------------------------------------ linear
def linear_bwd(a, w, dy, need_da=True, da_dtype=F16, da_add=None, need_dw=True, bias=True):
    """y = a @ w.T (+ b).  a [M,K] fp16, w [N,K] fp16, dy [M,N] fp16 (row-strided views allowed).
    Returns (da [M,K] | None, dw fp32 [N,K] | None, db fp32 [N] | None)."""
    M, K = a.shape
    N = w.shape[0]
    assert dy.shape == (M, N) and N % 8 == 0 and K % 8 == 0
    da = dw = db = None
    if need_da:
        # da = dy @ w: w [N, K] IS the [contraction, out-column] matrix -> MN-major B operand, no W^T copy
        da = ops.linear(dy, w, residual=da_add, out_dtype=da_dtype, w_t=True)
    if need_dw:
        # dw = dy^T @ a: both operands are stored [contraction = M rows][columns] -> MN-major A and B, no transposes.
        # An [N x K] output is only a handful of 128 x 256 tiles: split the row contraction over `S` batches (views of
        # the same buffers) so the GEMM fills the 132 SMs, then fold the partial sums.
        S = _row_splits(M, N, K)
        if S > 1 and dy.stride(1) == 1 and a.stride(1) == 1:
            mc = M // S
            dy3 = dy.as_strided((S, mc, N), (mc * dy.stride(0), dy.stride(0), 1), dy.storage_offset())
            a3 = a.as_strided((S, mc, K), (mc * a.stride(0), a.stride(0), 1), a.storage_offset())
            part = ops.linear(dy3, a3, out_dtype=F32, a_t=True, w_t=True)            # [S, N, K]
            dw = ops.col_sum(part.view(S, N * K)).view(N, K)
        else:
            dw = ops.linear(dy, a, out_dtype=F32, a_t=True, w_t=True)
        if bias:
            db = ops.col_sum(dy)
    return da, dw, db


def _row_splits(M, N, K, target_ctas=264, min_rows=512):
    """Number of equal row chunks (a divisor of M / 64) for a split-K weight-gradient GEMM of an [N x K] output."""
    if M % 64 != 0:
        return 1
    tiles = ((N + 127) // 128) * ((K + 255) // 256)
    want = max(1, min(target_ctas // max(tiles, 1), M // min_rows))
    kb = M // 64
    best = 1
    for s in range(1, want + 1):
        if kb % s == 0:
            best = s
    return best


# -------------------------------------------------------------------------------------------------- conv
# Weight-gradient GEMM variants (GPU-verified: tests/test_engine_gpu.py::test_wgrad_variants; overridable with
# B200_WGRAD_PADDED / B200_WGRAD_SPLIT_K):
#   WGRAD_PADDED  stride-1 3x3 convs: one zero-padded planar copy of X and three column-shifted copies of dY instead
#                 of nine shifted copies of X; a kernel row (ky) is a 16-byte-aligned pointer offset of ky*Wp into X.
#   WGRAD_SPLIT_K split the pixel contraction over `batch` so a Cout x Cin weight-gradient GEMM fills the 132 SMs;
#                 value = target number of CTAs (0 = no split, default two waves of 132); partial sums are reduced by
#                 `col_sum`.
import os as _os
WGRAD_PADDED = _os.environ.get("B200_WGRAD_PADDED", "1") == "1"
WGRAD_SPLIT_K = int(_os.environ.get("B200_WGRAD_SPLIT_K", "264"))
WGRAD_MIN_KBLOCKS = 8        # at least this many 64-wide k-blocks per split


def _split_plan(K, cout, cin):
    """(S, Kc): number of K chunks and chunk length (multiple of 64) for a [cout x cin] GEMM over K."""
    kb = (K + 63) // 64
    if WGRAD_SPLIT_K <= 0:
        return 1, kb * 64
    tiles = ((cout + 127) // 128) * ((cin + 159) // 160)
    S = max(1, min(WGRAD_SPLIT_K // max(tiles, 1), kb // WGRAD_MIN_KBLOCKS))
    kc = (kb + S - 1) // S
    return (kb + kc - 1) // kc, kc * 64


def _wgrad_taps(x, dy, taps, stride, up):
    """Validated path: one K-major copy of dY, one shifted K-major copy of X per tap, one GEMM per tap."""
    NB, Ho, Wo, Cout = dy.shape
    Cin = x.shape[3]
    P = NB * Ho * Wo
    S, Kc = _split_plan(P, Cout, Cin)
    if S == 1:
        dyt = ops.gather_planar(dy)                                          # [Cout, P8]
        dwp = torch.empty((Cout, len(taps) * Cin), dtype=F32, device=x.device)
        for t, (ty, tx) in enumerate(taps):
            xt = ops.gather_planar(x, out_hw=(Ho, Wo), stride=stride, up=up, off=(ty, tx))   # [Cin, P8]
            ops.linear(dyt, xt, out=dwp[:, t * Cin:(t + 1) * Cin], out_dtype=F32)
        return dwp
    ld = S * Kc
    dyt = ops.gather_planar(dy, out=torch.empty((Cout, ld), dtype=F16, device=x.device))
    part = torch.empty((S, Cout, len(taps) * Cin), dtype=F32, device=x.device)
    xt = torch.empty((Cin, ld), dtype=F16, device=x.device)
    a3 = dyt.as_strided((S, Cout, Kc), (Kc, ld, 1))
    w3 = xt.as_strided((S, Cin, Kc), (Kc, ld, 1))
    for t, (ty, tx) in enumerate(taps):
        ops.gather_planar(x, out_hw=(Ho, Wo), stride=stride, up=up, off=(ty, tx), out=xt)
        ops.linear(a3, w3, out=part[:, :, t * Cin:(t + 1) * Cin], out_dtype=F32)
    return ops.col_sum(part.view(S, -1)).view(Cout, len(taps) * Cin)


def _wgrad_padded(x, dy):
    """3x3 / stride 1 / pad 1.  Planar geometry (Hp, Wp) = (H + 2, ru8(W + 2)), flat index f = (n*Hp + i)*Wp + j:
         Xp[ci][f]     = X[n, i-1, j-1, ci]                 (zero border)
         dYk[kx][co][f] = dY[n, i, j-kx, co]                (rows i >= H and columns outside the image zero)
       => dW[co][ky][kx][ci] = sum_f dYk[kx][co][f] * Xp[ci][f + ky*Wp]."""
    NB, H, W, Cout = dy.shape
    Cin = x.shape[3]
    Hp, Wp = H + 2, ops._ru8(W + 2)
    K = NB * Hp * Wp
    S, Kc = _split_plan(K, Cout, Cin)
    ld = S * Kc                                                              # >= K, multiple of 64, zero tail
    dev = x.device
    xp = torch.zeros((Cin + 1, ld), dtype=F16, device=dev)                   # +1 row: reads at f + 2*Wp stay inside
    ops.gather_planar(x, out_hw=(Hp, Wp), off=(-1, -1), out=xp[:Cin])
    part = torch.empty((S, Cout, 9 * Cin), dtype=F32, device=dev)
    dyk = torch.empty((Cout, ld), dtype=F16, device=dev)
    a3 = dyk.as_strided((S, Cout, Kc), (Kc, ld, 1))
    for kx in range(3):
        ops.gather_planar(dy, out_hw=(Hp, Wp), off=(0, -kx), out=dyk)
        for ky in range(3):
            w3 = xp.as_strided((S, Cin, Kc), (Kc, ld, 1), ky * Wp)
            t = ky * 3 + kx
            ops.linear(a3, w3, out=part[:, :, t * Cin:(t + 1) * Cin], out_dtype=F32)
    if S == 1:
        return part[0]
    return ops.col_sum(part.view(S, -1)).view(Cout, 9 * Cin)


def conv_wgrad(x, dy, taps=TAPS3, stride=1, up=1, bias=True):
    """Weight gradient of out[n,o,p,:] = sum_t Wp[:, t*Cin:(t+1)*Cin] @ x_up[n, stride*o+ty, stride*p+tx, :]
    (x_up = nearest-`up`x of x).  x [NB,H,W,Cin], dy [NB,Ho,Wo,Cout] fp16 NHWC.
    Returns (dWp fp32 [Cout, T*Cin] in the packed forward layout, db fp32 [Cout] | None)."""
    Cout = dy.shape[3]
    if WGRAD_PADDED and stride == 1 and up == 1 and list(taps) == list(TAPS3) and x.shape[:3] == dy.shape[:3]:
        dwp = _wgrad_padded(x, dy)
    else:
        dwp = _wgrad_taps(x, dy, taps, stride, up)
    db = ops.col_sum(dy.reshape(-1, Cout)) if bias else None
    return dwp, db


def unpack_conv_grad(dwp, cin, kh=3, kw=3):
    """packed [Cout, kh*kw*Cin] -> parameter layout [Cout, Cin, kh, kw] (host-side re-layout of a gradient)."""
    return dwp.view(dwp.shape[0], kh, kw, cin).permute(0, 3, 1, 2).contiguous()


def conv_dgrad(dy, w, cin, kind="s1", out_dtype=F32, add=None, packed=None, in_hw=None):
    """Data gradient of the path's convolutions on the forward conv kernel.
    kind: "s1" (3x3 pad 1), "s2" (stride 2 pad 1), "s2_vae" (stride 2, pad (0,1,0,1)), "up" (nearest-2x + 3x3),
    "1x1".  dy NHWC fp16; returns dx NHWC (`add`, same shape/dtype, is accumulated)."""
    NB, Ho, Wo, Cout = dy.shape
    if kind == "1x1":
        wt = packed if packed is not None else ops.transpose_rows(w.reshape(w.shape[0], -1).to(F16))
        return ops.conv2d(dy, wt, cin, taps=[(0, 0)], residual=add, out_dtype=out_dtype)
    if kind == "s1":
        wp, taps = packed if packed is not None else pack_conv_dgrad_s1(w)
        return ops.conv2d(dy, wp, cin, taps=taps, residual=add, out_dtype=out_dtype)
    if kind in ("s2", "s2_vae"):
        ph = packed if packed is not None else pack_conv_dgrad_s2(w, 1 if kind == "s2" else 0)
        H, W = in_hw if in_hw is not None else (2 * Ho, 2 * Wo)
        even = (H, W) == (2 * Ho, 2 * Wo)
        assert even or (kind == "s2" and 2 * Ho - H in (0, 1) and 2 * Wo - W in (0, 1)), (H, W, Ho, Wo)
        out = torch.empty((NB, 2 * Ho, 2 * Wo, cin), dtype=out_dtype, device=dy.device)
        for (py, px), (wp, taps) in ph.items():
            ops.conv2d(dy, wp, cin, taps=taps, out_hw=(Ho, Wo), out=out, out_mul=2, out_off=(py, px),
                       residual=add if even else None)
        if even:
            return out
        # odd input size (pad-1 stride-2 conv): the extra row/column of the even-sized buffer is the forward's
        # zero padding; crop it (host-side re-layout, only on sizes that are not multiples of 2)
        out = out[:, :H, :W].contiguous()
        return out if add is None else out.add_(add)
    if kind == "up":
        acc = add
        for (py, px), (wp, taps) in (packed if packed is not None else pack_upsample_conv_dgrad(w)).items():
            taps2 = [(2 * ty + py, 2 * tx + px) for ty, tx in taps]
            acc = ops.conv2d(dy, wp, cin, taps=taps2, stride=2, out_hw=(Ho // 2, Wo // 2), residual=acc,
                             out_dtype=out_dtype)
        return acc
    raise ValueError(kind)


# --------------------------------------------------------------------------------------------- attention
def attention_bwd(q, k, v, do, heads, scale, outs=None, kv_segments=1):
    """Backward of softmax(scale * q k^T) v per head of width D = C / heads in ops.HEAD_DIMS.  q/do [B,T,C],
    k/v [B,Tk,C] fp16 views (last dim contiguous).  Returns fp16 (dq, dk, dv) — written into `outs` (row-strided
    views, e.g. the three column blocks of a fused d(qkv) buffer) when given.  `kv_segments` = 2: GeoWizard's joint
    attention (batch b attends to the keys of b % (B/2) and b % (B/2) + B/2, as in ops.attention).

    The flash kernel is re-run for (O, log-sum-exp) and delta_t = sum_d dO_td O_td (`rowdot_heads_d`); then, per head,
        P  = exp2(c * Q K^T - lse),  dS = scale * P o (dO V^T - delta)
        dQ = dS K,  dK = dS^T Q,  dV = P^T dO
    in the fused kernels (ops.attention_bwd): P and dS never leave the SM, so memory is O(B T C) at any length.
    Tensors the engine's kernels cannot take (not on a CUDA device) go to `_attention_bwd_gemm` instead, the per-image
    composition of GEMM launches that the fused kernels replaced: its ops raise for such tensors as every op does,
    and the CPU tests that restate each kernel in plain torch (tests/cpu_emulation.py) check this host algebra
    through it."""
    B, T, C = q.shape
    Tk = k.shape[1]
    D = C // heads
    assert C == heads * D and D in ops.HEAD_DIMS, (C, heads)
    assert kv_segments in (1, 2) and (kv_segments == 1 or B % 2 == 0), (kv_segments, B)
    dev = q.device
    if outs is not None:
        dq, dk, dv = outs
        assert dq.shape == (B, T, C) and dk.shape == (B, Tk, C) and dv.shape == (B, Tk, C)
    else:
        dq = torch.empty((B, T, C), dtype=F16, device=dev)
        dk = torch.empty((B, Tk, C), dtype=F16, device=dev)
        dv = torch.empty((B, Tk, C), dtype=F16, device=dev)

    if Tk == 1 and kv_segments == 1:
        # One key (GeoWizard's single image-embedding token): the softmax is constant, P = 1, so dS = P o (dP - delta)
        # is exactly zero, as torch.autograd finds it in the reference.  dQ = dK = 0 and dV = the sum of dO over the
        # queries.  The general path would form dP - delta from two differently ordered fp32 sums and leave rounding
        # noise in gradients that are exactly zero.
        dq.zero_()
        dk.zero_()
        for b in range(B):
            dv[b, 0].copy_(ops.cast_f16(ops.col_sum(do[b])))
        return dq, dk, dv

    o, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)   # lse: log2 domain
    delta = ops.rowdot_heads_d(do, o, heads, D)                                           # [B,heads,T]
    if q.is_cuda:
        ops.attention_bwd(q, k, v, do, lse, delta, dq, dk, dv, heads, scale, kv_segments)
    else:
        _attention_bwd_gemm(q, k, v, do, heads, scale, lse, delta, dq, dk, dv, kv_segments)
    return dq, dk, dv


def _attention_bwd_gemm(q, k, v, do, heads, scale, lse, delta, dq, dk, dv, kv_segments=1):
    """The backward as GEMM launches per image, batched over heads, with P and dS stored ([heads, T, Tk] fp16):
        P  = exp2(c * Q K^T - lse)                     exp2 epilogue with the row bias -lse
        dS = scale * P o (dO V^T - delta)              row bias -scale * delta, P as multiplicative operand
        dQ = dS K,  dK = dS^T Q,  dV = P^T dO          row contractions, operands consumed MN-major as stored.
    Joint attention (kv_segments = 2): the images i and i + B/2 of a pair form one problem of 2T queries over 2Tk keys
    whose dK / dV rows are the two images' own gradients."""
    B, T, C = q.shape
    Tk = k.shape[1]
    D = C // heads
    if kv_segments == 2:
        h = B // 2
        for i in range(h):
            pair = lambda t: torch.cat([t[i], t[i + h]], 0).unsqueeze(0)                    # host re-layout
            g = [torch.empty((1, 2 * L, C), dtype=F16, device=q.device) for L in (T, Tk, Tk)]
            _attention_bwd_gemm(pair(q), pair(k), pair(v), pair(do), heads, scale, pair(lse.transpose(1, 2)).transpose(
                1, 2).contiguous(), pair(delta.transpose(1, 2)).transpose(1, 2).contiguous(), *g)
            for out, gp, L in ((dq, g[0], T), (dk, g[1], Tk), (dv, g[2], Tk)):
                out[i].copy_(gp[0, :L])
                out[i + h].copy_(gp[0, L:])
        return
    Tkp = ops._ru8(Tk)

    def heads_view(t2d):                      # [L, heads*D] -> [heads, L, D] strided view
        return t2d.unflatten(-1, (heads, D)).permute(1, 0, 2)

    neg_lse = _scaled(lse, -1.0)
    neg_delta = _scaled(delta, -float(scale))
    c = float(scale) * 1.4426950408889634
    for b in range(B):
        qh, kh, vh, doh = heads_view(q[b]), heads_view(k[b]), heads_view(v[b]), heads_view(do[b])
        p = torch.empty((heads, T, Tkp), dtype=F16, device=q.device)
        ops.linear(qh, kh, bias=neg_lse[b], bias_row=True, act=ops.ACT_EXP2, alpha=c, out=p[:, :, :Tk])
        ds = torch.empty((heads, T, Tkp), dtype=F16, device=q.device)
        ops.linear(doh, vh, bias=neg_delta[b], bias_row=True, alpha=float(scale), residual=p[:, :, :Tk], res_mul=True,
                   out=ds[:, :, :Tk])
        # dQ[h] = dS[h] @ K[h]            (K [Tk, D] = [contraction, columns])
        ops.linear(ds[:, :, :Tk], kh, out=heads_view(dq[b]), w_t=True)
        # dK[h] = dS[h]^T @ Q[h], dV[h] = P[h]^T @ dO[h]   (contraction over the T query rows of both operands)
        ops.linear(ds[:, :, :Tk], qh, out=heads_view(dk[b]), a_t=True, w_t=True)
        ops.linear(p[:, :, :Tk], doh, out=heads_view(dv[b]), a_t=True, w_t=True)


def _scaled(t, f):
    """f * t for a small fp32 per-row vector ([B, heads, T] softmax statistics): host-level plumbing, O(rows)."""
    return (t * f).contiguous()
