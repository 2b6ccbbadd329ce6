"""The attention, softmax and normalisation kernels against fp64 references, element by element, under the bounds
derived in tests/numerics_bounds.py.  Each case asserts max(|got - ref| / bound) <= 1 and prints that ratio.  The case
lists follow the kernels' tiling constants: key tiles of 128 (D = 40, 64), 64 (D = 80, 160) and 32 (d512) keys, query
tiles of 192 (D <= 80), 128 (D = 160) and 64 (d512) rows, and each boundary is covered once per kernel."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import numerics_bounds as NB  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, F32 = torch.float16, torch.float32


def _check(what, got, ref, bound):
    r = NB.bound_ratio(got, ref, bound)
    print(f"{what}: max err / bound {r:.3f}")
    assert r <= 1.0, f"{what}: max err / bound {r:.3g}"
    return r


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ flash forward
def _flash_cases():
    cases = []
    for D in (40, 64, 80, 160):
        bk, bq = NB.ATT_BK[D], NB.ATT_BQ[D]
        cases += [(D, 65, Lk, "gauss", 1) for Lk in (1, bk - 1, bk, bk + 1, 3 * bk + 1, 2304)]
        cases += [(D, Lq, bk + 1, "gauss", 1) for Lq in (1, 63, 64, bq - 1, bq, bq + 1)]
        cases += [(D, bq + 1, 3 * bk + 1, "ramp_up", 1), (D, bq - 1, 3 * bk + 1, "ramp_down", 1),
                  (D, bq + 1, bk + 1, "jump", 2), (D, 64, bk - 1, "gauss", 2),
                  (D, 65, 2304, "peaked", 1), (D, 65, 3 * bk + 1, "uniform", 1)]
    return cases


@pytest.mark.parametrize("D,Lq,Lk,regime,kv_segments", _flash_cases())
def test_flash_forward_and_lse_within_bound(D, Lq, Lk, regime, kv_segments):
    """Q / K / V are head slices of fused [B, L, 3C] buffers whose other columns are non-zero; 8 heads."""
    from diffusion_e2e_ft_b200 import ops
    B, heads = 2, 8
    q, k, v, scale = NB.attention_inputs(B, heads, D, Lq, Lk, regime, seed=D + Lq + Lk, device=DEV,
                                         kv_segments=kv_segments)
    out, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)
    torch.cuda.synchronize()
    ref, bound, lse_ref, lse_b = NB.attention_ref_bound(NB.split_heads(q, heads), NB.split_heads(k, heads, kv_segments),
                                                        NB.split_heads(v, heads, kv_segments), scale, NB.ATT_BK[D])
    got = NB.split_heads(out, heads)
    tag = f"flash D={D} Lq={Lq} Lk={Lk} {regime} seg={kv_segments}"
    _check(tag + " out", got, ref, bound)
    _check(tag + " lse", lse.flatten(0, 1), lse_ref, lse_b)


# ------------------------------------------------------------------------------------------------ d512
@pytest.mark.parametrize("Lq,Lk,regime", [(65, 33, "ramp_up"), (64, 32, "ramp_down"), (63, 31, "peaked"),
                                          (1, 97, "ramp_up"), (129, 1, "gauss"), (65, 65, "peaked"),
                                          (127, 95, "uniform")])
def test_attention_d512_within_bound(Lq, Lk, regime):
    from diffusion_e2e_ft_b200 import ops
    q, k, v, scale = NB.attention_inputs(2, 1, 512, Lq, Lk, regime, seed=Lq + Lk, device=DEV)
    out = ops.attention_d512(q, k, v, scale)
    torch.cuda.synchronize()
    ref, bound, _, _ = NB.attention_ref_bound(q, k, v, scale, NB.ATT_BK[512])
    _check(f"d512 Lq={Lq} Lk={Lk} {regime}", out, ref, bound)


def test_attention_d512_large_lk_subnormal_p_within_bound():
    """50,000 keys with logits of std ~3: most weights, relative to the row maximum, fall below the fp16 normal range
    (P subnormal in the P V product).  Checked on 768 sampled query rows."""
    from diffusion_e2e_ft_b200 import ops
    L = 50000
    q, k, v, scale = NB.attention_inputs(1, 1, 512, L, L, "gauss", seed=5, device=DEV)
    scale *= 1.5
    out = ops.attention_d512(q, k, v, scale)
    torch.cuda.synchronize()
    g = torch.Generator().manual_seed(0)
    rows = torch.cat([torch.arange(256), torch.randint(256, L - 256, (256,), generator=g),
                      torch.arange(L - 256, L)]).to(DEV)
    ref, bound, _, _ = NB.attention_ref_bound(q, k, v, scale, NB.ATT_BK[512], rows=rows)
    s = q[:, rows[:64]].double() @ k.double().transpose(-1, -2) * scale
    sub = (torch.exp(s - s.amax(-1, keepdim=True)) < NB.F16_MIN_NORMAL).double().mean().item()
    print(f"d512 L={L}: {sub:.1%} of the sampled weights are below the fp16 normal range")
    assert sub > 0.5
    _check(f"d512 L={L} sampled rows", out[:, rows], ref, bound)


# ------------------------------------------------------------------------------------------------ attention bwd
def _bwd_inputs(B, T, Tk, heads, D, fused, seed):
    C = heads * D
    g = torch.Generator().manual_seed(seed)
    if fused:
        qkv = torch.randn(B, T, 3 * C, generator=g).half().to(DEV)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:
        q = torch.randn(B, T, C, generator=g).half().to(DEV)
        kv = torch.randn(B, Tk, 2 * C, generator=g).half().to(DEV)
        k, v = kv[..., :C], kv[..., C:]
    do = torch.randn(B, T, C, generator=g).half().to(DEV)
    return q, k, v, do


def _check_bwd(tag, q, k, v, do, heads, scale, dq, dk, dv):
    worst = {}
    qh, kh, vh, doh, dqh, dkh, dvh = (NB.split_heads(t, heads) for t in (q, k, v, do, dq, dk, dv))
    for n in range(qh.shape[0]):
        res = NB.attention_bwd_ref_bound(qh[n], kh[n], vh[n], doh[n], scale)
        for name, got in (("dq", dqh[n]), ("dk", dkh[n]), ("dv", dvh[n])):
            worst[name] = max(worst.get(name, 0.0), NB.bound_ratio(got, *res[name]))
        del res
    print(f"{tag}: max err / bound {', '.join(f'{k_} {v_:.3f}' for k_, v_ in worst.items())}")
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("D", [40, 64, 80, 160])
@pytest.mark.parametrize("T,Tk,fused", [(192, 192, True), (300, 300, True), (256, 77, False), (4, 77, False)])
def test_attention_bwd_within_bound(D, T, Tk, fused):
    from diffusion_e2e_ft_b200 import backward as bw
    B, heads, scale = 2, 8, D ** -0.5
    q, k, v, do = _bwd_inputs(B, T, Tk, heads, D, fused, seed=D + T)
    dq, dk, dv = bw.attention_bwd(q, k, v, do, heads, scale)
    torch.cuda.synchronize()
    _check_bwd(f"attention bwd D={D} T={T} Tk={Tk}", q, k, v, do, heads, scale, dq, dk, dv)


@pytest.mark.parametrize("D", [40, 64, 80, 160])
def test_attention_bwd_single_key(D):
    """Tk = 1: dQ and dK exactly zero, dV = the fp32 column sum of dO stored as fp16."""
    from diffusion_e2e_ft_b200 import backward as bw
    B, T, heads = 2, 129, 8
    q, k, v, do = _bwd_inputs(B, T, 1, heads, D, False, seed=D)
    dq, dk, dv = bw.attention_bwd(q, k, v, do, heads, D ** -0.5)
    torch.cuda.synchronize()
    assert not dq.any() and not dk.any()
    ref = do.double().sum(1, keepdim=True)
    bound = (T + 4) * NB.U32 * do.double().abs().sum(1, keepdim=True) * (1 + NB.U16) + NB.U16 * ref.abs() + NB.SUB16
    _check(f"attention bwd D={D} Tk=1 dv", dv, ref, bound)


@pytest.mark.parametrize("D,heads", [(64, 5), (40, 8)])
def test_attention_bwd_training_length_within_bound(D, heads):
    """T = Tk = 4800: the first attention level of a 480 x 640 training image (Hypersim)."""
    from diffusion_e2e_ft_b200 import backward as bw
    T, scale = 4800, D ** -0.5
    q, k, v, do = _bwd_inputs(1, T, T, heads, D, True, seed=D)
    dq, dk, dv = bw.attention_bwd(q, k, v, do, heads, scale)
    torch.cuda.synchronize()
    _check_bwd(f"attention bwd D={D} heads={heads} T=Tk={T}", q, k, v, do, heads, scale, dq, dk, dv)


# ------------------------------------------------------------------------------------------------ softmax
@pytest.mark.parametrize("rows,cols,peaked", [(50, 77, False), (300, 1024, False), (210, 9216, False),
                                              (33, 16384, True), (17, 20480, False), (1, 64, False)])
def test_softmax_rows_within_bound(rows, cols, peaked):
    """cols = 77: scalar kernel; <= 16384 and % 4: persistent shared-memory kernel; 20480: vectorised kernel."""
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(cols)
    s = torch.randn(rows, cols, generator=g) * 20
    if peaked:
        s[torch.arange(rows), (torch.arange(rows) * 977) % cols] += 400.0
    s = s.to(DEV)
    p = ops.softmax_rows(s, 0.125)
    torch.cuda.synchronize()
    _check(f"softmax_rows {rows}x{cols}{' peaked' if peaked else ''}", p, *NB.softmax_rows_ref_bound(s, 0.125))


@pytest.mark.parametrize("heads,S,ld_out", [(8, 77, 640), (5, 1, 8), (20, 257, 5144)])
def test_softmax_groups_within_bound(heads, S, ld_out):
    from diffusion_e2e_ft_b200 import ops
    x = (torch.randn(300, heads * S + 13, generator=torch.Generator().manual_seed(S)) * 6).to(DEV)
    p = ops.softmax_groups(x, heads, S, ld_out)
    torch.cuda.synchronize()
    assert torch.equal(p[:, heads * S:], torch.zeros_like(p[:, heads * S:]))
    _check(f"softmax_groups heads={heads} S={S}", p[:, :heads * S], *NB.softmax_groups_ref_bound(x, heads, S))


@pytest.mark.parametrize("rows,cols", [(300, 77), (64, 4801), (16, 16384)])
def test_softmax_bwd_rows_within_bound(rows, cols):
    from diffusion_e2e_ft_b200 import ops
    ld = (cols + 7) // 8 * 8
    g = torch.Generator().manual_seed(cols)
    p = torch.zeros(rows, ld, dtype=F16)
    p[:, :cols] = torch.softmax(torch.randn(rows, cols, generator=g) * 4, -1).half()
    dp = torch.zeros(rows, ld)
    dp[:, :cols] = torch.randn(rows, cols, generator=g)
    p, dp = p.to(DEV), dp.to(DEV)
    ds = ops.softmax_bwd_rows(p, dp, 0.125, cols=cols)
    torch.cuda.synchronize()
    assert not ds[:, cols:].any()             # the padding columns: zero-filled by ops.softmax_bwd_rows, not the kernel
    _check(f"softmax_bwd_rows {rows}x{cols}", ds[:, :cols], *NB.softmax_bwd_ref_bound(p[:, :cols], dp[:, :cols], 0.125))


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("C", [8, 256, 264, 512, 520, 768, 776, 1024, 1032, 1280, 1288, 1536, 1544, 1792, 1800, 2048])
@pytest.mark.parametrize("in_f32", [True, False])
def test_layer_norm_within_bound(C, in_f32):
    """(C + 255) / 256 picks the NV instantiation: one C on each side of every boundary."""
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(301, C, generator=g) * 2 + 0.3).to(F32 if in_f32 else F16).to(DEV)
    gamma = (torch.randn(C, generator=g) * 0.2 + 1.0).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.2).to(DEV)
    y = ops.layer_norm(x, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    _check(f"layer_norm C={C} {'f32' if in_f32 else 'f16'}", y, *NB.layer_norm_ref_bound(x, gamma, beta, 1e-5))


# ------------------------------------------------------------------------------------------------ GroupNorm
# (C1, C2): the channel concatenations of the UNet's up-block ResnetBlock2Ds (skip connections); groups of
# (C1 + C2) / 32 channels straddle C1 for (1280, 640) and (640, 320).  The VAE builds no concatenation.
GN_CONCATS = [(1280, 1280), (1280, 640), (640, 640), (640, 320), (320, 320)]


def _gn_inputs(NBt, H, W, C1, C2, in_f32, seed):
    g = torch.Generator().manual_seed(seed)
    dt = F32 if in_f32 else F16
    x1 = (torch.randn(NBt, H, W, C1, generator=g) + 0.5).to(dt).to(DEV)
    x2 = (torch.randn(NBt, H, W, C2, generator=g) * 2.0).to(dt).to(DEV) if C2 else None
    C = C1 + C2
    gamma = (torch.randn(C, generator=g) * 0.2 + 1.0).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.2).to(DEV)
    return x1, x2, gamma, beta


def _cs(x):
    """Exact per-channel [sum, sum of squares] in fp64, the layout the producing epilogues attach as `_cs`."""
    xd = x.double().flatten(1, 2)
    return torch.stack([xd.sum(1), (xd * xd).sum(1)], -1).contiguous()


def _gn_unrolled_hw(NBt, C, sms):
    """A pixel count per image for which every CTA of the GroupNorm kernels gets ppc = 8 rpb + 3 pixels: each thread
    runs the 8-pixel unrolled loop of gn_apply_kernel once and then the scalar tail (norm.cu gn_chunks)."""
    _, rpb = NB.gn_pixels_per_cta(NBt, 1, C, sms)
    target = (sms * 8 + NBt - 1) // NBt
    HW = target * (8 * rpb + 3) - 5
    ppc, _ = NB.gn_pixels_per_cta(NBt, HW, C, sms)
    assert ppc == 8 * rpb + 3 and ppc % (8 * rpb)
    return HW


@pytest.mark.parametrize("C1,C2", GN_CONCATS + [(320, 0)])
@pytest.mark.parametrize("in_f32,silu", [(False, True), (True, False)])
@pytest.mark.parametrize("fused", [False, True])
def test_group_norm_within_bound(C1, C2, in_f32, silu, fused):
    """HW from _gn_unrolled_hw: the unrolled loop and the tail both run.  fused: statistics from per-channel sums
    (`apply_cs`), here exact fp64 sums, so only the apply pass and its channel-to-group indexing are under test."""
    from diffusion_e2e_ft_b200 import ops
    NBt = 2
    HW = _gn_unrolled_hw(NBt, C1 + C2, _sms())
    x1, x2, gamma, beta = _gn_inputs(NBt, HW, 1, C1, C2, in_f32, seed=C1 + C2)
    if fused:
        x1._cs = _cs(x1)
        if x2 is not None:
            x2._cs = _cs(x2)
    y, raw = ops.group_norm(x1, gamma, beta, 1e-5, 32, silu, x2=x2, want_raw=True)
    torch.cuda.synchronize()
    xc = x1 if x2 is None else torch.cat([x1, x2], -1)
    assert torch.equal(raw, xc.half())
    cnt = 0 if fused else NB.gn_thread_count(NBt, HW, C1 + C2, _sms())
    _check(f"group_norm ({C1}, {C2}) HW={HW} {'f32' if in_f32 else 'f16'} silu={silu} "
           f"{'apply_cs' if fused else 'stats'}", y, *NB.group_norm_ref_bound(xc, gamma, beta, 1e-5, 32, silu, cnt))


@pytest.mark.parametrize("swap", [1, 0])
def test_group_norm_epilogue_statistics_within_bound(swap):
    """GroupNorm of a conv output (fp32, 192 channels) concatenated with a linear output (64 channels), both with the
    per-channel statistics their epilogues accumulate (shifted fp32 partial sums of at most HW stored values each, so
    cnt = HW), in both tile orientations.  A group straddles the two (256 / 32 = 8 channels, 192 / 8 = 24)."""
    import math
    from diffusion_e2e_ft_b200 import ops
    NBt, H, W, Cin, C1, C2 = 2, 16, 24, 64, 192, 64
    g = torch.Generator().manual_seed(31)
    x = torch.randn(NBt, H, W, Cin, generator=g).half().to(DEV)
    w = (torch.randn(C1, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)).half().to(DEV)
    b = torch.randn(C1, generator=g).to(DEV)
    a = torch.randn(NBt * H * W, 128, generator=g).half().to(DEV)
    w2 = (torch.randn(C2, 128, generator=g) / math.sqrt(128)).half().to(DEV)
    gamma = (torch.randn(C1 + C2, generator=g) * 0.2 + 1.0).to(DEV)
    beta = (torch.randn(C1 + C2, generator=g) * 0.2).to(DEV)
    L = ops._lib.load()
    L.b200_debug_set_swap(swap)
    try:
        y1 = ops.conv2d(x, ops.pack_conv(w), C1, bias=b, out_dtype=F32, stats=True)
        y2 = ops.linear(a, w2, None, out_dtype=F32, stats_rows_per_img=H * W)
    finally:
        L.b200_debug_set_swap(1)
    y2v = y2.view(NBt, H, W, C2)
    y2v._cs = y2._cs
    assert getattr(y1, "_cs", None) is not None and getattr(y2, "_cs", None) is not None
    out = ops.group_norm(y1, gamma, beta, 1e-5, 32, True, x2=y2v)
    torch.cuda.synchronize()
    xc = torch.cat([y1, y2v], -1)
    _check(f"group_norm epilogue statistics swap={swap}", out,
           *NB.group_norm_ref_bound(xc, gamma, beta, 1e-5, 32, True, H * W))


@pytest.mark.parametrize("C1,C2", GN_CONCATS + [(320, 0)])
@pytest.mark.parametrize("in_f32,silu,add,out_f32", [(False, True, True, True), (True, False, False, False),
                                                     (True, True, True, False)])
def test_group_norm_bwd_within_bound(C1, C2, in_f32, silu, add, out_f32):
    """dx (per concatenated input, with and without `add`, fp32 and fp16), dgamma and dbeta of ops.group_norm_bwd."""
    from diffusion_e2e_ft_b200 import ops
    NBt, H, W = 2, 7, 9
    x1, x2, gamma, beta = _gn_inputs(NBt, H, W, C1, C2, in_f32, seed=C1 + C2 + 1)
    xs = [x1] if x2 is None else [x1, x2]
    C = C1 + C2
    g = torch.Generator().manual_seed(C)
    dy = torch.randn(NBt, H, W, C, generator=g).half().to(DEV)
    odt = F32 if out_f32 else F16
    adds = [torch.randn(*t.shape, generator=g).to(odt).to(DEV) for t in xs] if add else None
    mr = ops.group_norm_mean_rstd(x1, 1e-5, 32, x2)
    dxs, dg, db = ops.group_norm_bwd(xs, dy, mr, gamma, beta, 32, silu, adds, odt)
    torch.cuda.synchronize()
    xc = torch.cat(xs, -1)
    res = NB.group_norm_bwd_ref_bound(xc, dy, gamma, beta, 1e-5, 32, silu, NB.gn_thread_count(NBt, H * W, C, _sms()),
                                      torch.cat(adds, -1) if add else None, out_f32)
    tag = f"group_norm_bwd ({C1}, {C2}) {'f32' if in_f32 else 'f16'} silu={silu} add={add} out {'f32' if out_f32 else 'f16'}"
    _check(tag + " dx", torch.cat(dxs, -1), *res["dx"])
    _check(tag + " dgamma", dg, *res["dgamma"])
    _check(tag + " dbeta", db, *res["dbeta"])


@pytest.mark.parametrize("C,in_f32,add,out_f32", [(8, True, True, True), (264, False, False, True),
                                                  (320, True, True, False), (640, False, True, False),
                                                  (1280, True, False, True), (1288, False, True, True),
                                                  (2048, True, True, False), (2048, False, False, True)])
def test_layer_norm_bwd_within_bound(C, in_f32, add, out_f32):
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator().manual_seed(C + 2)
    rows = 777
    x = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(F32 if in_f32 else F16).to(DEV)
    dy = torch.randn(rows, C, generator=g).half().to(DEV)
    gamma = (torch.randn(C, generator=g) * 0.3 + 1.0).to(DEV)
    odt = F32 if out_f32 else F16
    addt = torch.randn(rows, C, generator=g).to(odt).to(DEV) if add else None
    dx, dg, db = ops.layer_norm_bwd(x, dy, gamma, 1e-5, addt, out_dtype=odt)
    torch.cuda.synchronize()
    res = NB.layer_norm_bwd_ref_bound(x, dy, gamma, 1e-5, addt, out_f32)
    tag = f"layer_norm_bwd C={C} {'f32' if in_f32 else 'f16'} add={add} out {'f32' if out_f32 else 'f16'}"
    _check(tag + " dx", dx, *res["dx"])
    _check(tag + " dgamma", dg, *res["dgamma"])
    _check(tag + " dbeta", db, *res["dbeta"])


def test_group_norm_mean50_stress_within_bound():
    """Per-channel |mean| >> std (mean 50 .. 60, std 1, 128 channels x 768^2 pixels), standalone statistics pass."""
    from diffusion_e2e_ft_b200 import ops
    C, H, W = 128, 768, 768
    g = torch.Generator().manual_seed(41)
    gamma = (torch.randn(C, generator=g) * 0.2 + 1.0).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.2).to(DEV)
    x = (torch.randn(1, H, W, C, generator=g) + 50.0 * (1.0 + 0.2 * torch.arange(C) / C)).to(DEV)
    y = ops.group_norm(x, gamma, beta, 1e-5, 32, True)
    torch.cuda.synchronize()
    _check("group_norm mean-50 stress", y,
           *NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, True, NB.gn_thread_count(1, H * W, C, _sms())))
