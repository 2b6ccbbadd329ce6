"""Kernel-level parity checks (CUDA kernel through the C ABI vs a plain PyTorch fp32 reference of
the same op on the same seeded inputs).  Used by tests/test_kernels_gpu.py (pytest -m gpu) and by
tools/gpu_kernel_check.py (one subprocess per check, so one broken kernel cannot hide the others).

Tolerances: operands are fp16-rounded before BOTH paths, accumulation is fp32 on both, so the
residual error is summation order + fp16 output rounding: rel-L2 <= 2e-3 (fp16 out) / 2e-5-ish
(fp32 out).  Written per check below.
"""
import math

import torch
import torch.nn.functional as F

from diffusion_e2e_ft_b200 import ops

DEV = "cuda"
import os as _os
if _os.environ.get("B200_DEBUG_FLAGS"):            # perf / bring-up experiments (tools/): never set in the test suite
    ops._lib.load().b200_debug_set_flags(int(_os.environ["B200_DEBUG_FLAGS"]))


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _rand(*shape, seed=0, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


# ----------------------------------------------------------------------------------- GEMM
def check_linear(M=300, N=320, K=320, bias=True, residual=False, out_f32=False, act=0, batch=0, seed=0,
                 tol=None):
    bs = (batch,) if batch else ()
    a = _rand(*bs, M, K, seed=seed, scale=1.0)
    w = _rand(*bs, N, K, seed=seed + 1, scale=1.0 / math.sqrt(K))
    b = _rand(N, seed=seed + 2, dtype=torch.float32) if bias else None
    odt = torch.float32 if out_f32 else torch.float16
    n_out = N // 2 if act == ops.ACT_GEGLU else N
    r = _rand(*bs, M, n_out, seed=seed + 3, dtype=odt) if residual else None
    ref = torch.matmul(a.float(), w.float().transpose(-1, -2))
    if b is not None:
        ref = ref + b
    if act == ops.ACT_GEGLU:
        h, g = ref.chunk(2, dim=-1)
        ref = h * F.gelu(g)
        wp, bp = ops.pack_geglu(w, b)
    else:
        wp, bp = w, b
    if r is not None:
        ref = ref + r.float()
    if act == ops.ACT_SILU:
        ref = F.silu(ref)
    out = ops.linear(a, wp, bp, residual=r, out_dtype=odt, act=act)
    torch.cuda.synchronize()
    err = rel_l2(out, ref)
    tol = tol or (3e-5 if out_f32 else 1e-3)
    return err, tol


def check_linear_mn(M=1000, N=320, K=200, a_t=False, w_t=False, batch=0, out_f32=True, swap=1, seed=81):
    """MN-major operands: a given as [K, M] and / or w as [K, N] (row-major, as the backward pass finds them) are
    consumed by the tensor core as stored — out = a^T w, a w, a^T w^T — against torch on the same fp16 values.
    Row pitches are padded (row-strided views), M / N / K ragged against the 64-row atoms."""
    bs = (batch,) if batch else ()
    ar = _rand(*bs, M, K, seed=seed)                    # logical a [M, K]
    wr = _rand(*bs, N, K, seed=seed + 1, scale=1.0 / math.sqrt(K))
    ref = torch.matmul(ar.float(), wr.float().transpose(-1, -2))

    def stored(t, transposed):
        t = t.transpose(-1, -2).contiguous() if transposed else t
        pad = torch.zeros(*t.shape[:-1], (t.shape[-1] + 15) // 8 * 8, dtype=t.dtype, device=t.device)   # padded row pitch
        pad[..., :t.shape[-1]] = t
        return pad[..., :t.shape[-1]]
    a, w = stored(ar, a_t), stored(wr, w_t)
    L = ops._lib.load()
    L.b200_debug_set_swap(swap)
    try:
        out = ops.linear(a, w, out_dtype=torch.float32 if out_f32 else torch.float16, a_t=a_t, w_t=w_t)
        torch.cuda.synchronize()
    finally:
        L.b200_debug_set_swap(1)
    return rel_l2(out, ref), (3e-5 if out_f32 else 1e-3)


def check_geglu_two_gemm(M=300, C=320, seed=17):
    """GEGLU as gate GEMM (erf-GELU epilogue) + value GEMM with a multiplicative residual operand."""
    a = _rand(M, C, seed=seed)
    w = _rand(8 * C, C, seed=seed + 1, scale=1 / math.sqrt(C))
    b = _rand(8 * C, seed=seed + 2, dtype=torch.float32)
    gate = ops.linear(a, w[4 * C:].contiguous(), b[4 * C:].contiguous(), act=ops.ACT_GELU)
    out = ops.linear(a, w[:4 * C].contiguous(), b[:4 * C].contiguous(), residual=gate, res_mul=True)
    torch.cuda.synchronize()
    h, g = (a.float() @ w.float().t() + b).chunk(2, dim=-1)
    return rel_l2(out, h * F.gelu(g)), 1.5e-3


def check_linear_bias_row(seed=5):
    """D[m,n] = W[m,:]·h[n,:] + bias[m]  (V^T projection of the VAE attention)."""
    M, N, K = 512, 700, 512
    a = _rand(M, K, seed=seed, scale=1 / math.sqrt(K))
    w = _rand(N, K, seed=seed + 1)
    b = _rand(M, seed=seed + 2, dtype=torch.float32)
    ref = a.float() @ w.float().t() + b[:, None]
    out = ops.linear(a, w, b, bias_row=True)
    torch.cuda.synchronize()
    return rel_l2(out, ref), 1e-3


# ----------------------------------------------------------------------------------- conv
def _conv_ref(x_nhwc, w, b, stride, pad_mode):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    if pad_mode == "vae_down":
        x = F.pad(x, (0, 1, 0, 1))
        return F.conv2d(x, w.float(), b, stride=stride, padding=0)
    return F.conv2d(x, w.float(), b, stride=stride, padding=1)


def check_conv(NB=2, H=24, W=24, Cin=128, Cout=192, stride=1, pad_mode="same", shortcut=0, rowvec=False,
               residual=False, out_f32=False, out_nchw=False, seed=0, tol=None):
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    ref = _conv_ref(x, w, b, stride, pad_mode)
    Ho, Wo = ref.shape[2], ref.shape[3]
    x2 = ws = None
    if shortcut:
        x2 = _rand(NB, Ho, Wo, shortcut, seed=seed + 4)
        ws = _rand(Cout, shortcut, 1, 1, seed=seed + 5, scale=1.0 / math.sqrt(shortcut))
        ref = ref + F.conv2d(x2.float().permute(0, 3, 1, 2), ws.float())
    rv = None
    if rowvec:
        rv = _rand(NB, Cout, seed=seed + 6, dtype=torch.float32)
        ref = ref + rv[:, :, None, None]
    odt = torch.float32 if out_f32 else torch.float16
    res = None
    if residual:
        res = _rand(NB, Ho, Wo, Cout, seed=seed + 7, dtype=odt)
        ref = ref + res.float().permute(0, 3, 1, 2)
    wp = ops.pack_conv(w, ws)
    taps = ops.TAPS3_PAD0 if pad_mode == "vae_down" else ops.TAPS3
    out = ops.conv2d(x, wp, Cout, bias=b, taps=taps, stride=stride, out_hw=(Ho, Wo), x2=x2, rowvec=rv,
                     residual=res, out_dtype=odt, out_nchw=out_nchw)
    torch.cuda.synchronize()
    got = out if out_nchw else out.permute(0, 3, 1, 2)
    err = rel_l2(got, ref)
    return err, tol or (3e-5 if out_f32 else 1e-3)


def check_swap_epilogue_twins(seed=51):
    """Vectorised swapped epilogue: fp32 output + fp16 twin + fused per-channel statistics + SiLU + fp32 residual on a
    ragged conv (odd pixel count, Cout = 320 = 2.5 channel tiles), and a fp16-output linear with a multiplicative
    fp16 residual operand and N = 960.  Output, twin and statistics against torch."""
    NB, H, W, Cin, Cout = 2, 15, 21, 64, 320
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    res = _rand(NB, H, W, Cout, seed=seed + 3, dtype=torch.float32)
    L = ops._lib.load()
    L.b200_debug_force_block_n(256)          # 256-wide candidates only: the cost model then takes the swapped orientation
    try:
        out = ops.conv2d(x, ops.pack_conv(w), Cout, bias=b, residual=res, out_dtype=torch.float32, act=ops.ACT_SILU,
                         stats=True, f16_copy=True)
        torch.cuda.synchronize()
    finally:
        L.b200_debug_force_block_n(0)
    ref = F.silu(_conv_ref(x, w, b, 1, "same").permute(0, 2, 3, 1) + res)
    e1 = rel_l2(out, ref)
    e2 = rel_l2(out._h16, out.half())
    cs = out._cs.float()                                                   # [NB, Cout, 2] (sum, sum of squares)
    want = torch.stack([out.double().sum((1, 2)), (out.double() ** 2).sum((1, 2))], -1).float()
    e3 = rel_l2(cs, want)
    M, N, K = 1000, 960, 320
    a = _rand(M, K, seed=seed + 4)
    w2 = _rand(N, K, seed=seed + 5, scale=1.0 / math.sqrt(K))
    b2 = _rand(N, seed=seed + 6, dtype=torch.float32)
    gate = _rand(M, N, seed=seed + 7)
    L.b200_debug_force_block_n(128)
    try:
        o2 = ops.linear(a, w2, b2, residual=gate, res_mul=True)
        torch.cuda.synchronize()
    finally:
        L.b200_debug_force_block_n(0)
    ref2 = (a.float() @ w2.float().t() + b2) * gate.float()
    e4 = rel_l2(o2, ref2)
    return max(e1 / 3e-5, e2 / 1e-7 if e2 > 0 else 0.0, e3 / 1e-5, e4 / 1e-3) * 1e-3, 1e-3


def check_conv_halo(NB=2, H=40, W=64, Cin=128, Cout=128, shortcut=0, residual=False, out_f32=False, rowvec=False,
                    stats=False, seed=71):
    """Halo-resident stride-1 3x3 conv (one patch load per 64-channel block, nine taps as row-shifted wgmma views) vs
    torch AND vs the per-tap-box path of the same kernel; asserts that the halo path was really taken."""
    L = ops._lib.load()
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    ref = _conv_ref(x, w, b, 1, "same")
    x2 = ws = None
    if shortcut:
        x2 = _rand(NB, H, W, shortcut, seed=seed + 4)
        ws = _rand(Cout, shortcut, 1, 1, seed=seed + 5, scale=1.0 / math.sqrt(shortcut))
        ref = ref + F.conv2d(x2.float().permute(0, 3, 1, 2), ws.float())
    rv = None
    if rowvec:
        rv = _rand(NB, Cout, seed=seed + 6, dtype=torch.float32)
        ref = ref + rv[:, :, None, None]
    odt = torch.float32 if out_f32 else torch.float16
    res = None
    if residual:
        res = _rand(NB, H, W, Cout, seed=seed + 7, dtype=odt)
        ref = ref + res.float().permute(0, 3, 1, 2)
    wp = ops.pack_conv(w, ws)
    outs = []
    for halo in (2, 0):                                    # 2 = halo even where the dispatcher would call it epilogue-bound
        L.b200_debug_set_halo(halo)
        try:
            o = ops.conv2d(x, wp, Cout, bias=b, x2=x2, rowvec=rv, residual=res, out_dtype=odt, stats=True if stats else None)
            torch.cuda.synchronize()
            assert L.b200_debug_last_path() == (1 if halo else 0), f"expected conv path {halo}, kernel took {L.b200_debug_last_path()}"
        finally:
            L.b200_debug_set_halo(1)
        outs.append(o)
    e_ref = rel_l2(outs[0].permute(0, 3, 1, 2), ref)
    e_tap = rel_l2(outs[0], outs[1])                       # same products, different summation order: fp32 / fp16 rounding
    tol = 3e-5 if out_f32 else 1e-3
    worst = max(e_ref, e_tap)
    if stats:
        worst = max(worst, rel_l2(outs[0]._cs.float(), outs[1]._cs.float()) * (tol / 1e-5))
    return worst, tol


def check_conv_halo_taps(seed=91):
    """Halo path with other tap sets: the flipped-tap data gradient of a 3x3 conv and the 2x2 phases of the 4-phase
    upsample conv (out_mul = 2), each against the per-tap-box path."""
    L = ops._lib.load()
    NB, H, W, Cin, Cout = 2, 24, 48, 128, 128
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    from diffusion_e2e_ft_b200.backward_packing import pack_conv_dgrad_s1
    wp, taps = pack_conv_dgrad_s1(w)
    worst = 0.0
    outs = []
    for halo in (2, 0):
        L.b200_debug_set_halo(halo)
        try:
            outs.append(ops.conv2d(x, wp, Cin, taps=taps, out_dtype=torch.float32))
            torch.cuda.synchronize()
            assert L.b200_debug_last_path() == (1 if halo else 0)
        finally:
            L.b200_debug_set_halo(1)
    worst = max(worst, rel_l2(outs[0], outs[1]))
    from diffusion_e2e_ft_b200.modules import Upsample2D
    m = Upsample2D(Cin).to(DEV)
    xs = _rand(NB, H, W, Cin, seed=seed + 2, dtype=torch.float32)
    ys = []
    with torch.no_grad():
        for halo in (2, 0):
            L.b200_debug_set_halo(halo)
            try:
                ys.append(m.run(xs, None, torch.float32))
                torch.cuda.synchronize()
                assert L.b200_debug_last_path() == (1 if halo else 0)
            finally:
                L.b200_debug_set_halo(1)
    worst = max(worst, rel_l2(ys[0], ys[1]))
    return worst, 3e-5


def check_attention_lse_and_rowdot(B=2, heads=5, Lq=300, Lk=200, seed=95, fused=False):
    """Flash kernel's log2-domain log-sum-exp output and the rowdot kernel (the two row statistics of the attention
    backward) against torch; then P recomputed by the exp2-epilogue GEMM against softmax.  fused=True takes q from one
    projection output and k, v as strided views of another."""
    C = heads * 64
    if fused:
        q = _rand(B, Lq, 2 * C, seed=seed)[..., :C]
        kv = _rand(B, Lk, 2 * C, seed=seed + 1)
        k, v = kv[..., :C], kv[..., C:]
    else:
        q, k, v = _rand(B, Lq, C, seed=seed), _rand(B, Lk, C, seed=seed + 1), _rand(B, Lk, C, seed=seed + 2)
    scale = 64 ** -0.5
    o, lse = ops.attention_d64(q, k, v, heads, scale, want_lse=True)
    def split(t):
        return t.float().view(t.shape[0], t.shape[1], heads, 64).permute(0, 2, 1, 3)
    logits = split(q) @ split(k).transpose(-1, -2) * scale
    lse_ref = torch.logsumexp(logits, -1) * 1.4426950408889634
    e1 = (lse - lse_ref).abs().max().item() / lse_ref.abs().max().item()
    do = _rand(B, Lq, C, seed=seed + 3)
    d = ops.rowdot_heads(do, o, heads)
    d_ref = (split(do) * split(o)).sum(-1)
    e2 = rel_l2(d, d_ref)
    b = 1
    qh = q[b].unflatten(-1, (heads, 64)).permute(1, 0, 2)
    kh = k[b].unflatten(-1, (heads, 64)).permute(1, 0, 2)
    p = torch.empty((heads, Lq, (Lk + 7) // 8 * 8), dtype=torch.float16, device=DEV)
    ops.linear(qh, kh, bias=(-lse[b]).contiguous(), bias_row=True, act=ops.ACT_EXP2, alpha=scale * 1.4426950408889634,
               out=p[:, :, :Lk])
    torch.cuda.synchronize()
    e3 = rel_l2(p[:, :, :Lk], torch.softmax(logits[b], -1))
    return max(e1 / 1e-5, e2 / 1e-5, e3 / 1e-3) * 1e-3, 1e-3


def check_upsample_conv_phases(NB=2, H=12, W=10, C=128, seed=21):
    """Upsample2D: nearest x2 + conv3x3 computed as four 2x2 convs on the low-res input."""
    from diffusion_e2e_ft_b200.modules import Upsample2D
    m = Upsample2D(C).to(DEV)
    g = torch.Generator(device="cpu").manual_seed(seed)
    with torch.no_grad():
        m.conv.weight.copy_((torch.randn(C, C, 3, 3, generator=g) / math.sqrt(9 * C)).half().float())
        m.conv.bias.copy_(torch.randn(C, generator=g) * 0.1)
    x = _rand(NB, H, W, C, seed=seed + 1, dtype=torch.float32)
    with torch.no_grad():
        y = m.run(x, None, torch.float32)
        torch.cuda.synchronize()
        up = F.interpolate(x.half().float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
        ref = F.conv2d(up, m.conv.weight, m.conv.bias, padding=1).permute(0, 2, 3, 1)
    return rel_l2(y, ref), 1e-3


def check_conv_small_cout(NB=2, H=37, W=50, C=128, Cout=3, seed=41):
    x = _rand(NB, H, W, C, seed=seed)
    w = _rand(Cout, C, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * C))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    out = ops.conv3x3_small_cout(x, ops.pack_conv_small_cout(w), b, Cout)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1)
    return rel_l2(out, ref), 3e-5


def check_conv_in(NB=2, C=8, H=20, W=24, Cout=320, seed=3):
    """small-Cin conv = im2col kernel + GEMM, NCHW fp32 input straight from the caller."""
    x = _rand(NB, C, H, W, seed=seed, dtype=torch.float32)
    w = _rand(Cout, C, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * C))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    kpad = (9 * C + 7) // 8 * 8
    patches = ops.im2col3x3(x, kpad)
    out = ops.linear(patches, ops.pack_conv_small_cin(w, kpad), b)
    torch.cuda.synchronize()
    ref = F.conv2d(x.half().float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    return rel_l2(out, ref), 1e-3


# ----------------------------------------------------------------------------------- norms
def check_group_norm(NB=2, H=17, W=24, C1=320, C2=0, in_f32=False, silu=True, seed=0):
    dt = torch.float32 if in_f32 else torch.float16
    x1 = _rand(NB, H, W, C1, seed=seed, dtype=dt) + 0.5
    x2 = (_rand(NB, H, W, C2, seed=seed + 1, dtype=dt) * 2.0) if C2 else None
    C = C1 + C2
    g = _rand(C, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    b = _rand(C, seed=seed + 3, dtype=torch.float32) * 0.2
    y, raw = ops.group_norm(x1, g, b, 1e-5, 32, silu, x2=x2, want_raw=True)
    torch.cuda.synchronize()
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=-1)
    ref = F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    e1 = rel_l2(y, ref)
    e2 = rel_l2(raw, xc)
    return max(e1, e2), 6e-4


def check_gn_fused_stats(swap=True, seed=31):
    """GroupNorm whose statistics come from the producing conv / linear epilogues (no gn_stats pass),
    on a channel concat of a conv output (fp32) and a linear output viewed NHWC."""
    NB, H, W, Cin = 2, 16, 24, 64
    C1, C2 = (128, 128) if swap else (192, 64)
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(C1, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(C1, seed=seed + 2, dtype=torch.float32)
    y1 = ops.conv2d(x, ops.pack_conv(w), C1, bias=b, out_dtype=torch.float32, stats=True)
    a = _rand(NB * H * W, 128, seed=seed + 3)
    w2 = _rand(C2, 128, seed=seed + 4, scale=1 / math.sqrt(128))
    y2 = ops.linear(a, w2, None, out_dtype=torch.float32, stats_rows_per_img=H * W)
    y2v = y2.view(NB, H, W, C2)
    y2v._cs = y2._cs
    assert getattr(y1, "_cs", None) is not None and getattr(y2, "_cs", None) is not None
    C = C1 + C2
    g = _rand(C, seed=seed + 5, dtype=torch.float32) * 0.2 + 1.0
    bt = _rand(C, seed=seed + 6, dtype=torch.float32) * 0.2
    out = ops.group_norm(y1, g, bt, 1e-5, 32, True, x2=y2v)
    torch.cuda.synchronize()
    xc = torch.cat([y1, y2v], dim=-1)
    ref = F.silu(F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, bt, 1e-5)).permute(0, 2, 3, 1)
    return rel_l2(out, ref), 6e-4


def check_gn_stress(fused=False, NB=1, H=768, W=768, C=128, mean=50.0, std=1.0, seed=41):
    """VERDICT r1 weak #3: per-channel |mean| >> std (mean 50, std 1, 128 ch x 768^2) against an fp64 GroupNorm.
    A single-pass fp32 sum / sum-of-squares loses the variance to cancellation here (E[x^2] ~ 2501 vs var 1); the
    kernels accumulate SHIFTED partial sums per thread and merge them in fp64.
    fused=False: standalone gn_stats pass on an fp32 tensor.  fused=True: statistics from the epilogue of the
    producing GEMM (a linear layer whose bias carries the large per-channel mean), both tile orientations."""
    g = _rand(C, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    b = _rand(C, seed=seed + 3, dtype=torch.float32) * 0.2
    cmean = (mean * (1.0 + 0.2 * torch.arange(C, device=DEV) / C)).float()                # 50 .. 60 per channel
    if not fused:
        x = _rand(NB, H, W, C, seed=seed, dtype=torch.float32) * std + cmean
        y = ops.group_norm(x, g, b, 1e-5, 32, True)
        xs = [x]
    else:
        K = 64
        a = _rand(NB * H * W, K, seed=seed)
        w = _rand(C, K, seed=seed + 1, scale=std / math.sqrt(K))
        xs, ys = [], []
        for swap in (1, 0):
            ops._lib.load().b200_debug_set_swap(swap)
            try:
                x = ops.linear(a, w, cmean.contiguous(), out_dtype=torch.float32, stats_rows_per_img=H * W)
            finally:
                ops._lib.load().b200_debug_set_swap(1)
            assert getattr(x, "_cs", None) is not None
            xv = x.view(NB, H, W, C)
            xv._cs = x._cs
            ys.append(ops.group_norm(xv, g, b, 1e-5, 32, True))
            xs.append(xv)
    torch.cuda.synchronize()
    worst = 0.0
    for x, yy in zip(xs, [y] if not fused else ys):
        ref = F.silu(F.group_norm(x.double().permute(0, 3, 1, 2), 32, g.double(), b.double(), 1e-5)).permute(0, 2, 3, 1)
        worst = max(worst, ((yy.double() - ref).norm() / ref.norm()).item())
    return worst, 6e-4          # fp16 output rounding only (2.8e-4 rms); a cancelled variance shows up as >= 1e-2


def check_layer_norm(rows=1000, C=640, in_f32=True, seed=0):
    dt = torch.float32 if in_f32 else torch.float16
    x = _rand(rows, C, seed=seed, dtype=dt) * 2 + 0.3
    g = _rand(C, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    b = _rand(C, seed=seed + 3, dtype=torch.float32) * 0.2
    y = ops.layer_norm(x, g, b, 1e-5)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5)
    return rel_l2(y, ref), 6e-4


def check_softmax_rows(rows=300, cols=1152, seed=0):
    s = _rand(rows, cols, seed=seed, dtype=torch.float32) * 20
    p = ops.softmax_rows(s, 0.125)
    torch.cuda.synchronize()
    return rel_l2(p, torch.softmax(s * 0.125, dim=-1)), 6e-4


# ----------------------------------------------------------------------------------- attention
def check_attention(B=2, heads=5, Lq=576, Lk=None, joint=False, gain=3.0, seed=0, ramp=None, separate=False):
    """Flash kernel vs fp32 torch.  q, k, v are strided views of one fused projection output (the engine's layout);
    separate=True passes them as three contiguous tensors instead (row strides C, not 3C / 2C)."""
    Lk = Lk or Lq
    C = heads * 64
    qkv = _rand(B, Lq, 3 * C, seed=seed)
    if separate:
        q = qkv[..., :C].contiguous()
        kv = qkv if Lk == Lq else _rand(B, Lk, 2 * C, seed=seed + 1)
        k, v = kv[..., -2 * C:-C].contiguous(), kv[..., -C:].contiguous()
    elif Lk == Lq:
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:
        q = qkv[..., :C]
        kv = _rand(B, Lk, 2 * C, seed=seed + 1)
        k, v = kv[..., :C], kv[..., C:]
    if ramp is not None:
        # key magnitude grows (ramp > 0) or shrinks (< 0) along the sequence: the running row maximum keeps moving tile
        # after tile, so the online-softmax rescale of O and of the row sum is exercised
        r = torch.linspace(0.05, abs(ramp), Lk, device=DEV)
        r = r if ramp > 0 else r.flip(0)
        k = (k.float() * r[None, :, None]).half()
    q = q * gain if False else q
    scale = 64 ** -0.5 * gain
    out = ops.attention_d64(q, k, v, heads, scale, kv_segments=2 if joint else 1)
    torch.cuda.synchronize()
    qf = q.float().view(B, Lq, heads, 64).transpose(1, 2)
    kf = k.float().reshape(B, Lk, heads, 64).transpose(1, 2)
    vf = v.float().reshape(B, Lk, heads, 64).transpose(1, 2)
    if joint:
        k0, k1 = kf.chunk(2, 0)
        v0, v1 = vf.chunk(2, 0)
        kf = torch.cat([torch.cat([k0, k1], 2)] * 2, 0)
        vf = torch.cat([torch.cat([v0, v1], 2)] * 2, 0)
    p = torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1)
    ref = (p @ vf).transpose(1, 2).reshape(B, Lq, C)
    return rel_l2(out, ref), 2e-3


# ----------------------------------------------------------------------------------- elementwise
def check_losses(seed=51):
    """SSI / angular loss kernels against the oracle restatement of training/util/loss.py."""
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import pipeline as OP
    pred = _rand(3, 1, 40, 56, seed=seed, dtype=torch.float32).clamp(-1, 1)
    gt = (_rand(3, 1, 40, 56, seed=seed + 1, dtype=torch.float32).abs() * 3 + 0.1)
    mask = _rand(3, 1, 40, 56, seed=seed + 2, dtype=torch.float32) > -0.5
    e1 = abs(ops.ssi_loss(pred, gt, mask).item() - OP.ssi_loss(pred.cpu(), gt.cpu(), mask.cpu()).item())
    n1 = F.normalize(_rand(3, 3, 40, 56, seed=seed + 3, dtype=torch.float32), dim=1)
    n2 = F.normalize(_rand(3, 3, 40, 56, seed=seed + 4, dtype=torch.float32), dim=1)
    e2 = abs(ops.angular_loss(n1, n2, mask).item() - OP.angular_loss(n1.cpu(), n2.cpu(), mask.cpu()).item())
    d = _rand(2, 3, 9, 7, seed=seed + 5, dtype=torch.float32)
    e3 = rel_l2(ops.decode_post(d, training=True), d.mean(1, keepdim=True).clamp(-1, 1))
    e4 = rel_l2(ops.decode_post(d, normals=True, training=True), (d / (d.norm(dim=1, keepdim=True) + 1e-5)).clamp(-1, 1))
    torch.cuda.synchronize()
    return max(e1, e2, e3, e4), 2e-5


def check_adamw(seed=61, n=100003):
    """Fused clip + AdamW over a flat buffer vs torch.optim.AdamW + clip_grad_norm_ (training/train.py:346-353,564-566)."""
    p0 = _rand(n, seed=seed, dtype=torch.float32)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=3e-3, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    p = p0.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    worst = 0.0
    for step in range(1, 4):
        g = _rand(n, seed=seed + step, dtype=torch.float32) * (3.0 if step == 2 else 0.001)
        ref_p.grad = g.clone()
        torch.nn.utils.clip_grad_norm_([ref_p], 1.0)
        opt.step()
        nsq = ops.grad_norm_sq(g)
        ops.adamw_step(p, g, m, v, step, lr=3e-3, grad_norm_sq_t=nsq, max_grad_norm=1.0)
        torch.cuda.synchronize()
        worst = max(worst, rel_l2(p, ref_p.data), abs(nsq.item() - float((g.double() ** 2).sum())) / nsq.item())
    return worst, 2e-6


def check_adamw_state(seed=67, n=100003):
    """State-driven fused clip + AdamW (device-side skip decision + dynamic loss scale, no host sync) vs
    torch.optim.AdamW + clip_grad_norm_: three good steps with a loss-scaled, world-summed gradient buffer, then a
    non-finite gradient (step skipped, scale halved), an all-zero gradient (skipped, scale kept), another good step
    (bias correction continues from the APPLIED step count), and scale growth after `growth_interval` good steps."""
    p0 = _rand(n, seed=seed, dtype=torch.float32)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=3e-3, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    p = p0.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    state = torch.zeros(8, dtype=torch.float32, device=DEV)
    state[0] = 1024.0
    world = 4
    worst = 0.0

    def engine_step(g_true):
        S = float(state[0])
        g = g_true * (S * world)
        nsq = ops.grad_norm_sq(g)
        ops.adamw_step_state(p, g, m, v, state, nsq, lr=3e-3, max_grad_norm=1.0, inv_world=1.0 / world,
                             dynamic_scale=True, growth_interval=3)
        torch.cuda.synchronize()

    def ref_step(g_true):
        ref_p.grad = g_true.clone()
        torch.nn.utils.clip_grad_norm_([ref_p], 1.0)
        opt.step()

    for step in range(1, 3):
        g = _rand(n, seed=seed + step, dtype=torch.float32) * (3.0 if step == 2 else 0.001)
        ref_step(g); engine_step(g)
        worst = max(worst, rel_l2(p, ref_p.data))
    assert state.tolist()[:5] == [1024.0, 2.0, 2.0, 0.0, 0.0], state.tolist()
    keep = (p.clone(), m.clone(), v.clone())
    bad = _rand(n, seed=seed + 9, dtype=torch.float32)
    bad[5] = float("inf")
    engine_step(bad)                                                   # overflow: skipped, scale halves, tracker resets
    assert all(torch.equal(a, b) for a, b in zip(keep, (p, m, v))) and state.tolist()[:5] == [512.0, 0.0, 2.0, 1.0, 1.0]
    engine_step(torch.zeros(n, device=DEV))                            # empty masks: skipped, scale kept
    assert all(torch.equal(a, b) for a, b in zip(keep, (p, m, v))) and state.tolist()[:5] == [512.0, 0.0, 2.0, 2.0, 1.0]
    for step in range(3, 6):                                           # 3 good steps -> scale doubles once
        g = _rand(n, seed=seed + step, dtype=torch.float32) * 0.01
        ref_step(g); engine_step(g)
        worst = max(worst, rel_l2(p, ref_p.data))
    assert state.tolist()[:5] == [1024.0, 0.0, 5.0, 2.0, 0.0], state.tolist()
    return worst, 2e-6


def check_upsample(in_f32=False, out_hw=None):
    dt = torch.float32 if in_f32 else torch.float16
    x = _rand(2, 7, 9, 64, dtype=dt)
    ohw = out_hw or (14, 18)
    y = ops.upsample_nearest(x, ohw)
    torch.cuda.synchronize()
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), size=ohw, mode="nearest").permute(0, 2, 3, 1)
    return rel_l2(y, ref.half()), 1e-6


def check_timestep_embedding():
    t = torch.tensor([999.0, 1.0, 500.0], device=DEV)
    out = ops.timestep_embedding(t, 320)
    torch.cuda.synchronize()
    half = 160
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=DEV) / half)
    e = t[:, None] * f[None]
    ref = torch.cat([torch.cos(e), torch.sin(e)], -1)
    return (out.float() - ref).abs().max().item(), 2e-3


def check_pointwise_and_post():
    x = _rand(2, 8, 6, 10, dtype=torch.float32)
    z = _rand(2, 8, 6, 10, seed=9, dtype=torch.float32)
    wm = _rand(4, 8, seed=3, dtype=torch.float32)
    b = _rand(4, seed=4, dtype=torch.float32)
    out = ops.pointwise_nchw(x, 0.5, wm, b, in2=z, a2=-2.0)
    ref = torch.einsum("oc,nchw->nohw", wm, 0.5 * x - 2.0 * z) + b[None, :, None, None]
    e1 = rel_l2(out, ref)
    d = _rand(2, 3, 5, 7, seed=11, dtype=torch.float32)
    dep = ops.decode_post(d, normals=False)
    e2 = rel_l2(dep, (d.mean(1, keepdim=True).clip(-1, 1) + 1) / 2)
    nrm = ops.decode_post(d, normals=True, sign=-1.0)
    e3 = rel_l2(nrm, -d / (d.norm(dim=1, keepdim=True) + 1e-5))
    y = _rand(2, 5, 6, 24, seed=12)
    e4 = rel_l2(ops.nhwc_to_nchw_f32(y), y.float().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    return max(e1, e2, e3, e4), 1e-5


def _noswap(fn):
    """run a check with the swapped-operand mode disabled (exercises the transposed-epilogue path)."""
    def run():
        from diffusion_e2e_ft_b200 import lib
        L = lib.load()
        L.b200_debug_set_swap(0)
        try:
            return fn()
        finally:
            L.b200_debug_set_swap(1)
    return run


# ------------------------------------------------------------------ backward (data-gradient) convs, row a10
def _autograd_dx(fwd, x_nchw, dy_nchw):
    x = x_nchw.clone().requires_grad_(True)
    (fwd(x) * dy_nchw).sum().backward()
    return x.grad.permute(0, 2, 3, 1)


def check_conv_dgrad_s1(NB=2, H=20, W=24, Cin=128, Cout=192, seed=61):
    from diffusion_e2e_ft_b200.backward_packing import pack_conv_dgrad_s1
    w = _rand(Cout, Cin, 3, 3, seed=seed, scale=1.0 / math.sqrt(9 * Cin))
    dy = _rand(NB, H, W, Cout, seed=seed + 1)
    x = _rand(NB, Cin, H, W, seed=seed + 2, dtype=torch.float32)
    wp, taps = pack_conv_dgrad_s1(w)
    got = ops.conv2d(dy, wp, Cin, taps=taps, out_dtype=torch.float32)
    torch.cuda.synchronize()
    ref = _autograd_dx(lambda t: F.conv2d(t, w.float(), padding=1), x, dy.float().permute(0, 3, 1, 2))
    return rel_l2(got, ref), 3e-5


def check_conv_dgrad_s2(pad_lo=1, NB=2, H=20, W=24, Cin=128, Cout=128, seed=63):
    from diffusion_e2e_ft_b200.backward_packing import pack_conv_dgrad_s2
    w = _rand(Cout, Cin, 3, 3, seed=seed, scale=1.0 / math.sqrt(9 * Cin))
    x = _rand(NB, Cin, H, W, seed=seed + 2, dtype=torch.float32)
    if pad_lo:
        fwd = lambda t: F.conv2d(t, w.float(), stride=2, padding=1)
    else:
        fwd = lambda t: F.conv2d(F.pad(t, (0, 1, 0, 1)), w.float(), stride=2)
    dy = _rand(NB, H // 2, W // 2, Cout, seed=seed + 1)
    got = torch.empty((NB, H, W, Cin), dtype=torch.float32, device=DEV)
    for (py, px), (wp, taps) in pack_conv_dgrad_s2(w, pad_lo).items():
        ops.conv2d(dy, wp, Cin, taps=taps, out_hw=(H // 2, W // 2), out=got, out_mul=2, out_off=(py, px))
    torch.cuda.synchronize()
    ref = _autograd_dx(fwd, x, dy.float().permute(0, 3, 1, 2))
    return rel_l2(got, ref), 3e-5


def check_upsample_conv_dgrad(NB=2, H=12, W=10, C=128, seed=65):
    """dX of (nearest x2 -> conv3x3): four stride-2 tap convs over the full-resolution dY, accumulated through
    the fp32 residual operand (phase (py,px) reads dY[2a + py - 2dy, 2b + px - 2dx])."""
    from diffusion_e2e_ft_b200.backward_packing import pack_upsample_conv_dgrad
    from diffusion_e2e_ft_b200.modules import Upsample2D
    m = Upsample2D(C).to(DEV)
    g = torch.Generator(device="cpu").manual_seed(seed)
    with torch.no_grad():
        m.conv.weight.copy_((torch.randn(C, C, 3, 3, generator=g) / math.sqrt(9 * C)).half().float())
    w = m.conv.weight.detach()
    dy = _rand(NB, 2 * H, 2 * W, C, seed=seed + 1)
    x = _rand(NB, C, H, W, seed=seed + 2, dtype=torch.float32)
    acc = None
    for (py, px), (wp, taps) in pack_upsample_conv_dgrad(m._pack_phases()).items():
        taps2 = [(2 * ty + py, 2 * tx + px) for ty, tx in taps]
        acc = ops.conv2d(dy, wp.to(DEV), C, taps=taps2, stride=2, out_hw=(H, W), residual=acc,
                         out_dtype=torch.float32)
    torch.cuda.synchronize()
    fwd = lambda t: F.conv2d(F.interpolate(t, scale_factor=2.0, mode="nearest"), w, padding=1)
    ref = _autograd_dx(fwd, x, dy.float().permute(0, 3, 1, 2))
    return rel_l2(acc, ref), 1e-3      # phase weights are sums of fp16 weights re-rounded to fp16


CHECKS = {
    "conv_dgrad_s1": check_conv_dgrad_s1,
    "conv_dgrad_s2_pad1": lambda: check_conv_dgrad_s2(1),
    "conv_dgrad_s2_vae_pad": lambda: check_conv_dgrad_s2(0),
    "upsample_conv_dgrad": check_upsample_conv_dgrad,
    "linear_basic": lambda: check_linear(),
    "linear_small_m": lambda: check_linear(M=8, N=1280, K=320),
    "linear_bn256": lambda: check_linear(M=2000, N=1280, K=1280, seed=2),
    "linear_ragged_k": lambda: check_linear(M=130, N=64, K=72, seed=3),
    "linear_f32_residual": lambda: check_linear(M=1000, N=640, K=2560, residual=True, out_f32=True),
    "linear_f16_residual_silu": lambda: check_linear(M=257, N=1280, K=1280, residual=True, act=ops.ACT_SILU),
    "linear_geglu": lambda: check_linear(M=300, N=2560, K=320, act=ops.ACT_GEGLU),
    "linear_geglu_small": lambda: check_linear(M=100, N=512, K=64, act=ops.ACT_GEGLU),
    "linear_batched": lambda: check_linear(M=200, N=300 // 4 * 4 + 4, K=512, batch=3, bias=False),
    "linear_bias_row": check_linear_bias_row,
    "geglu_two_gemm": check_geglu_two_gemm,
    "geglu_two_gemm_64": lambda: check_geglu_two_gemm(M=100, C=64),
    "linear_unaligned_ldo": lambda: check_linear(M=130, N=700, K=128, residual=True, seed=7),
    "conv_s1": lambda: check_conv(),
    "conv_s1_96": lambda: check_conv(NB=1, H=96, W=96, Cin=64, Cout=320),
    "conv_s1_odd": lambda: check_conv(NB=1, H=15, W=20, Cin=64, Cout=64),
    "conv_s1_12": lambda: check_conv(NB=3, H=12, W=12, Cin=256, Cout=256),
    "conv_fused_shortcut_temb_res_f32": lambda: check_conv(shortcut=64, rowvec=True, residual=True, out_f32=True),
    "conv_res_f16": lambda: check_conv(residual=True),
    "conv_s2_pad1": lambda: check_conv(stride=2),
    "conv_s2_pad1_odd": lambda: check_conv(H=15, W=30, stride=2, Cin=64, Cout=64),
    "conv_s2_vae": lambda: check_conv(stride=2, pad_mode="vae_down", H=32, W=48),
    "conv_out_nchw": lambda: check_conv(Cin=128, Cout=3, out_f32=True, out_nchw=True, H=40, W=56),
    "conv_out4_nchw": lambda: check_conv(Cin=64, Cout=4, out_f32=True, out_nchw=True),
    "conv_in_im2col": check_conv_in,
    "conv_small_cout_3": check_conv_small_cout,
    "conv_small_cout_4_320": lambda: check_conv_small_cout(NB=1, H=96, W=96, C=320, Cout=4),
    "conv_small_cout_8_512": lambda: check_conv_small_cout(NB=2, H=12, W=20, C=512, Cout=8),
    "upsample_conv_4phase": check_upsample_conv_phases,
    "conv_swap_128_res_temb_f32": lambda: check_conv(H=40, W=40, Cin=128, Cout=128, rowvec=True, residual=True, out_f32=True),
    "conv_swap_256_shortcut": lambda: check_conv(H=24, W=24, Cin=128, Cout=256, shortcut=128),
    "conv_swap_s2": lambda: check_conv(H=32, W=32, Cin=64, Cout=128, stride=2),
    "conv_swap_s2_vae": lambda: check_conv(H=32, W=48, Cin=128, Cout=128, stride=2, pad_mode="vae_down"),
    "conv_swap_odd": lambda: check_conv(NB=1, H=15, W=20, Cin=64, Cout=128, residual=True),
    "conv_swap_768": lambda: check_conv(NB=1, H=96, W=768, Cin=128, Cout=128, seed=9),
    "conv_swap_1280_12": lambda: check_conv(NB=2, H=12, W=12, Cin=256, Cout=1280),
    "swap_epilogue_twins_stats": check_swap_epilogue_twins,
    "conv_halo_128": lambda: check_conv_halo(),
    "conv_halo_dgrad_and_upsample_taps": check_conv_halo_taps,
    "conv_halo_res_f32_stats": lambda: check_conv_halo(H=48, W=96, Cin=64, Cout=256, residual=True, out_f32=True, rowvec=True, stats=True),
    "conv_halo_shortcut_320": lambda: check_conv_halo(NB=1, H=48, W=48, Cin=192, Cout=320, shortcut=128, out_f32=True),
    "conv_halo_edges_768": lambda: check_conv_halo(NB=1, H=35, W=768, Cin=64, Cout=128, seed=73),
    "conv_halo_ragged": lambda: check_conv_halo(NB=2, H=21, W=120, Cin=64, Cout=128, residual=True, seed=75),
    "conv_noswap_256": _noswap(lambda: check_conv(H=24, W=24, Cin=128, Cout=256, residual=True, out_f32=True)),
    "linear_noswap_1280": _noswap(lambda: check_linear(M=2000, N=1280, K=1280, residual=True, seed=2)),
    "linear_swap_small_m": lambda: check_linear(M=8, N=1280, K=1280, act=ops.ACT_SILU),
    "linear_swap_ragged": lambda: check_linear(M=777, N=384, K=200, residual=True, out_f32=True),
    "linear_mn_w": lambda: check_linear_mn(w_t=True),                                        # dX = dY W
    "linear_mn_w_noswap": lambda: check_linear_mn(w_t=True, swap=0, N=64, K=1000, M=333),    # dQ = dS K (N = 64)
    "linear_mn_aw": lambda: check_linear_mn(M=320, N=640, K=2304, a_t=True, w_t=True),       # dW = dY^T X
    "linear_mn_aw_noswap": lambda: check_linear_mn(M=77, N=64, K=1000, a_t=True, w_t=True, swap=0),   # dK = dS^T Q, 77 keys
    "linear_mn_a": lambda: check_linear_mn(M=200, N=256, K=520, a_t=True, out_f32=False),
    "linear_mn_aw_batched": lambda: check_linear_mn(M=576, N=64, K=576, a_t=True, w_t=True, batch=5, swap=0),
    "gn_f16": lambda: check_group_norm(),
    "gn_f32_concat": lambda: check_group_norm(C1=1280, C2=640, in_f32=True),
    "gn_concat_f16_nosilu": lambda: check_group_norm(C1=640, C2=320, silu=False),
    "gn_128": lambda: check_group_norm(C1=128, H=64, W=64),
    "gn_fused_stats_swap": lambda: check_gn_fused_stats(True),
    "gn_fused_stats_normal": lambda: check_gn_fused_stats(False),
    "gn_stress_mean50_standalone": lambda: check_gn_stress(False),
    "gn_stress_mean50_fused": lambda: check_gn_stress(True),
    "ln_f32": lambda: check_layer_norm(),
    "ln_f16_1280": lambda: check_layer_norm(C=1280, in_f32=False),
    "ln_320": lambda: check_layer_norm(C=320),
    "softmax_rows": check_softmax_rows,
    "softmax_rows_persistent_9216": lambda: check_softmax_rows(rows=2100, cols=9216, seed=1),   # ~7 rows per CTA, 2-deep ring
    "softmax_rows_persistent_1024": lambda: check_softmax_rows(rows=9001, cols=1024, seed=2),
    "softmax_rows_single_row": lambda: check_softmax_rows(rows=1, cols=64, seed=3),
    "softmax_rows_16384": lambda: check_softmax_rows(rows=333, cols=16384, seed=4),
    "softmax_rows_unaligned_cols": lambda: check_softmax_rows(rows=50, cols=77, seed=5),         # scalar fallback kernel
    "ln_8": lambda: check_layer_norm(rows=77, C=8),
    "ln_1024": lambda: check_layer_norm(rows=514, C=1024),
    "ln_2048_f16": lambda: check_layer_norm(rows=300, C=2048, in_f32=False),
    "ln_1536": lambda: check_layer_norm(rows=300, C=1536),
    "attn_self_576": lambda: check_attention(),
    "attn_self_2304": lambda: check_attention(B=1, heads=10, Lq=2304),
    "attn_ragged_144": lambda: check_attention(B=2, heads=20, Lq=144),
    "attn_cross_2": lambda: check_attention(Lq=576, Lk=2),
    "attn_cross_77": lambda: check_attention(Lq=300, Lk=77),
    "attn_joint": lambda: check_attention(B=4, heads=5, Lq=576, joint=True),
    "attn_lse_rowdot_exp2_gemm": check_attention_lse_and_rowdot,
    "attn_ramp_up": lambda: check_attention(B=1, heads=3, Lq=700, Lk=1500, ramp=6.0),
    "attn_ramp_down": lambda: check_attention(B=1, heads=3, Lq=700, Lk=1500, ramp=-6.0),
    # attn_v2_*: the same shapes with the other operand layout (separate contiguous q / k / v; for the LSE check, strided
    # views).  The name is kept from an earlier kernel variant of the same checks.
    "attn_v2_self_576": lambda: check_attention(separate=True),
    "attn_v2_self_2304": lambda: check_attention(B=1, heads=10, Lq=2304, separate=True),
    "attn_v2_ragged_144": lambda: check_attention(B=2, heads=20, Lq=144, separate=True),
    "attn_v2_cross_2": lambda: check_attention(Lq=576, Lk=2, separate=True),
    "attn_v2_cross_77": lambda: check_attention(Lq=300, Lk=77, separate=True),
    "attn_v2_joint": lambda: check_attention(B=4, heads=5, Lq=576, joint=True, separate=True),
    "attn_v2_lse_rowdot_exp2_gemm": lambda: check_attention_lse_and_rowdot(fused=True),
    "attn_v2_ramp_up": lambda: check_attention(B=1, heads=3, Lq=700, Lk=1500, ramp=6.0, separate=True),
    "attn_v2_ramp_down": lambda: check_attention(B=1, heads=3, Lq=700, Lk=1500, ramp=-6.0, separate=True),
    "attn_v2_single_query": lambda: check_attention(B=2, heads=4, Lq=1, Lk=9, separate=True),
    "upsample_2x": check_upsample,
    "upsample_size_f32": lambda: check_upsample(True, (15, 20)),
    "timestep_embedding": check_timestep_embedding,
    "pointwise_post": check_pointwise_and_post,
    "losses_ssi_angular": check_losses,
    "adamw_clip_fused": check_adamw,
    "adamw_state_skip_dynamic_scale": check_adamw_state,
}


# backward-pass operators (row a10): tests/bwd_checks.py
from bwd_checks import BWD_CHECKS  # noqa: E402

CHECKS.update(BWD_CHECKS)
