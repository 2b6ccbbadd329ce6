"""The per-element bounds of tests/numerics_bounds.py, checked without a GPU:
* not too tight: a CPU emulation of each kernel's rounding schedule stays at or below half its bound.  An elementwise
  fp16 result (softmax, the norms) can spend the whole U16 |ref| store term by itself, so for those the emulated fp32
  value before the store is held to the bound without the store term (`store=False`); the store is one IEEE rounding;
* not too loose: planted mutants (the bugs a kernel could plausibly have) exceed the bound at least 4x somewhere;
* the fp64 references agree with torch's fp64 ops and autograd."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numerics_bounds as NB  # noqa: E402

F16, F32 = torch.float16, torch.float32
EMU_MAX = 0.5
MUTANT_MIN = 4.0


def _c32(scale):
    """c = fp32(fp32(scale) * fp32(log2 e)), as the kernels form it."""
    return (torch.tensor(scale, dtype=F32) * torch.tensor(NB.LOG2E, dtype=F32)).item()


# ------------------------------------------------------------------------------------------------ attention
def emulate_attention(q, k, v, scale, bk, mutant=None):
    """attention_kernel's rounding schedule: fp32 scores, per key tile an online softmax with the fp32 exponent
    fmaf(S, c, -fp32(m c)), fp16 P in P V, fp32 l and O, out = fp16(O * fp32(1 / l)), lse = m c + log2 l.
    q [N, Lq, D], k / v [N, Lk, D] fp16.  `mutant` plants one bug."""
    c = _c32(scale)
    S = q.float() @ k.float().transpose(-1, -2)
    vf = v.float()
    N, Lq, Lk = S.shape
    m = torch.full((N, Lq, 1), -math.inf)
    l = torch.zeros(N, Lq, 1)
    o = torch.zeros(N, Lq, v.shape[-1])
    n_tiles = (Lk + bk - 1) // bk
    for t in range(n_tiles):
        j0, j1 = t * bk, min(Lk, (t + 1) * bk)
        if mutant == "drop_last_key" and t == n_tiles - 1:
            j1 -= 1
        s = S[..., j0:j1]
        vt = vf[:, j0:j1]
        if mutant == "double_last_key" and t == n_tiles - 1:
            s = torch.cat([s, s[..., -1:]], -1)
            vt = torch.cat([vt, vt[:, -1:]], 1)
        if s.shape[-1] == 0:
            continue
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp2(((m - mn) * c).float())
        if mutant == "skip_alpha" and t == 1:
            alpha = torch.ones_like(alpha)
        mc = (mn * c).float()
        p = torch.exp2((s.double() * c - mc.double()).float())
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + p.half().float() @ vt
        m = mn
    if mutant == "neighbour_l":
        l = l.clone()
        l[:, 0] = l[:, 1]
    out = (o * (1.0 / l)).half()
    if mutant == "one_element":
        out = out.clone()
        i = Lq // 2
        d = out[0, i].float().abs().argmax()                   # the row's largest output: 5 % of it is visible
        out[0, i, d] = (out[0, i, d].float() * 1.05).half()
    lse = (m.double() * c + torch.log2(l.double())).float().squeeze(-1)
    return out, lse


def _attention_case(D, Lq, Lk, regime, kv_segments=1, B=2, heads=2, seed=0):
    q, k, v, scale = NB.attention_inputs(B, heads, D, Lq, Lk, regime, seed=seed, kv_segments=kv_segments)
    qh, kh, vh = (NB.split_heads(t, heads, s).half() for t, s in ((q, 1), (k, kv_segments), (v, kv_segments)))
    return qh, kh, vh, scale


def _attention_cases():
    cases = []
    for D in (40, 64, 80, 160, 512):
        bk = NB.ATT_BK[D]
        heads = 1 if D == 512 else 2
        for Lk in (1, bk - 1, bk, bk + 1, 3 * bk + 1):
            cases.append((D, 65, Lk, "gauss", 1, heads))
        cases += [(D, 1, 3 * bk + 1, "ramp_up", 1, heads), (D, 64, 3 * bk + 1, "ramp_down", 1, heads),
                  (D, 63, 3 * bk + 1, "peaked", 1, heads), (D, 65, bk - 1, "uniform", 1, heads)]
        if D != 512:
            cases += [(D, 65, bk + 1, "jump", 2, heads), (D, 64, bk - 1, "gauss", 2, heads)]
    cases.append((40, 64, 2304, "gauss", 1, 1))
    return cases


@pytest.mark.parametrize("D,Lq,Lk,regime,kv_segments,heads", _attention_cases())
def test_attention_emulation_within_half_the_bound(D, Lq, Lk, regime, kv_segments, heads):
    q, k, v, scale = _attention_case(D, Lq, Lk, regime, kv_segments, heads=heads)
    ref, bound, lse_ref, lse_b = NB.attention_ref_bound(q, k, v, scale, NB.ATT_BK[D])
    out, lse = emulate_attention(q, k, v, scale, NB.ATT_BK[D])
    r_out, r_lse = NB.bound_ratio(out, ref, bound), NB.bound_ratio(lse, lse_ref, lse_b)
    print(f"attention D={D} Lq={Lq} Lk={Lk} {regime} seg={kv_segments}: out {r_out:.3f} lse {r_lse:.3f}")
    assert r_out <= EMU_MAX and r_lse <= EMU_MAX, (r_out, r_lse)


@pytest.mark.parametrize("D", [40, 64, 80, 160, 512])
@pytest.mark.parametrize("mutant", ["one_element", "drop_last_key", "double_last_key", "skip_alpha", "neighbour_l"])
def test_attention_mutants_exceed_the_bound(D, mutant):
    bk = NB.ATT_BK[D]
    heads = 1 if D == 512 else 2
    # the moving maximum of ramp_up makes alpha matter and puts weight on the last key
    q, k, v, scale = _attention_case(D, 65, 3 * bk + 1, "gauss" if mutant == "one_element" else "ramp_up", heads=heads)
    ref, bound, _, _ = NB.attention_ref_bound(q, k, v, scale, bk)
    out, _ = emulate_attention(q, k, v, scale, bk, mutant=mutant)
    r = NB.bound_ratio(out, ref, bound)
    print(f"attention D={D} mutant {mutant}: {r:.1f}x the bound")
    assert r >= MUTANT_MIN, r


def test_attention_reference_matches_torch_fp64():
    q, k, v, scale = _attention_case(80, 37, 150, "gauss", kv_segments=2, B=2, heads=3)
    ref, _, lse, _ = NB.attention_ref_bound(q, k, v, scale, 64)
    want = F.scaled_dot_product_attention(q.double(), k.double(), v.double(), scale=scale)
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)
    s = q.double() @ k.double().transpose(-1, -2) * scale
    assert torch.allclose(lse, torch.logsumexp(s, -1) / math.log(2.0), rtol=1e-12, atol=1e-12)
    rows = torch.tensor([0, 5, 36])
    r2, b2, _, _ = NB.attention_ref_bound(q, k, v, scale, 64, rows=rows, chunk_elems=1)
    full, fb, _, _ = NB.attention_ref_bound(q, k, v, scale, 64)
    assert torch.allclose(r2, full[:, rows], rtol=1e-12, atol=0) and torch.allclose(b2, fb[:, rows], rtol=1e-12)


def test_split_heads_joint_matches_the_segment_walk():
    t = torch.arange(4 * 3 * 6, dtype=F32).view(4, 3, 6)
    x = NB.split_heads(t, 2, kv_segments=2)                     # [B * heads, 2L, D]
    assert x.shape == (8, 6, 3)
    # batch 1 (heads 0, 1) attends to the keys of batch 1 then batch 3; batch 2 to those of batch 0 then batch 2
    assert torch.equal(x[2], torch.cat([t[1, :, :3], t[3, :, :3]]).double())
    assert torch.equal(x[5], torch.cat([t[0, :, 3:], t[2, :, 3:]]).double())


# ------------------------------------------------------------------------------------------------ attention bwd
def emulate_attention_bwd(q, k, v, do, scale, mutant=None):
    """backward.attention_bwd's rounding schedule for one head (q / do [T, D], k / v [Tk, D] fp16)."""
    D = q.shape[-1]
    o, lse = emulate_attention(q[None], k[None], v[None], scale, NB.ATT_BK[D])
    o, lse = o[0], lse[0]
    delta = (do.float() * o.float()).sum(-1, keepdim=True)
    if mutant == "delta_wrong_row":
        delta = delta.roll(1, 0)
    c = torch.tensor(scale * NB.LOG2E, dtype=F32).item()
    S = q.float() @ k.float().t()
    P = torch.exp2((S.double() * c - lse.double()[:, None]).float()).half()
    dP = do.float() @ v.float().t()
    pre = (dP.double() * scale + (-scale * delta).double()).float()
    dS = (pre * P.float()).half()
    return (dS.float() @ k.float()).half(), (dS.float().t() @ q.float()).half(), (P.float().t() @ do.float()).half()


@pytest.mark.parametrize("D,T,Tk", [(64, 193, 193), (40, 129, 77), (80, 65, 130), (160, 64, 65)])
def test_attention_bwd_emulation_within_half_the_bound(D, T, Tk):
    q, k, v, scale = _attention_case(D, T, Tk, "gauss", B=1, heads=1, seed=D)
    scale = D ** -0.5
    do = torch.randn(T, D, generator=torch.Generator().manual_seed(3)).half()
    res = NB.attention_bwd_ref_bound(q[0], k[0], v[0], do, scale)
    got = dict(zip(("dq", "dk", "dv"), emulate_attention_bwd(q[0], k[0], v[0], do, scale)))
    ratios = {n: NB.bound_ratio(got[n], *res[n]) for n in res}
    print(f"attention bwd D={D} T={T} Tk={Tk}: {ratios}")
    assert max(ratios.values()) <= EMU_MAX, ratios
    bad = dict(zip(("dq", "dk", "dv"), emulate_attention_bwd(q[0], k[0], v[0], do, scale, "delta_wrong_row")))
    r = max(NB.bound_ratio(bad[n], *res[n]) for n in ("dq", "dk"))
    print(f"   mutant delta of the wrong row: {r:.1f}x")
    assert r >= MUTANT_MIN


def test_attention_bwd_reference_chunks_agree():
    q, k, v, scale = _attention_case(64, 70, 90, "gauss", B=1, heads=1)
    do = torch.randn(70, 64, generator=torch.Generator().manual_seed(6)).half()
    one = NB.attention_bwd_ref_bound(q[0], k[0], v[0], do, scale)
    many = NB.attention_bwd_ref_bound(q[0], k[0], v[0], do, scale, chunk_rows=16)
    for n in one:
        for a, b in zip(one[n], many[n]):
            assert torch.allclose(a, b, rtol=1e-12, atol=1e-15), n


def test_attention_bwd_reference_matches_autograd():
    q, k, v, scale = _attention_case(40, 50, 70, "gauss", B=1, heads=1)
    do = torch.randn(50, 40, generator=torch.Generator().manual_seed(5)).half()
    res = NB.attention_bwd_ref_bound(q[0], k[0], v[0], do, scale)
    qr, kr, vr = (t[0].double().requires_grad_(True) for t in (q, k, v))
    (torch.softmax(qr @ kr.t() * scale, -1) @ vr * do.double()).sum().backward()
    for n, t in (("dq", qr), ("dk", kr), ("dv", vr)):
        assert torch.allclose(res[n][0], t.grad, rtol=1e-10, atol=1e-12), n


# ------------------------------------------------------------------------------------------------ softmax
def emulate_softmax_rows(s, scale):
    c = _c32(scale)
    m = s.amax(-1, keepdim=True)
    ms = (m * c).float()
    e = torch.exp2((s * c).float() - ms)
    return e * (1.0 / e.sum(-1, keepdim=True))


def _one_off(t, row):
    """t with the largest element of `row` 5 % off, stored as fp16."""
    t = t.half()
    j = t[row].float().abs().argmax()
    t[row, j] = (t[row, j].float() * 1.05).half()
    return t


def _softmax_logits(rows, cols, seed, kind="gauss"):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(rows, cols, generator=g) * 20
    if kind == "peaked":
        s[torch.arange(rows), torch.arange(rows) % cols] += 400.0
    return s


@pytest.mark.parametrize("rows,cols,kind", [(50, 77, "gauss"), (64, 1024, "gauss"), (16, 9216, "gauss"),
                                            (8, 16384, "peaked"), (4, 20480, "gauss")])
def test_softmax_rows_emulation_and_mutant(rows, cols, kind):
    s = _softmax_logits(rows, cols, cols, kind)
    ref, bound = NB.softmax_rows_ref_bound(s, 0.125)
    emu = emulate_softmax_rows(s, 0.125)
    r = NB.bound_ratio(emu, ref, NB.softmax_rows_ref_bound(s, 0.125, store=False)[1])
    assert NB.bound_ratio(emu.half(), ref, bound) <= 1.0
    rm = NB.bound_ratio(_one_off(emu, 1), ref, bound)
    print(f"softmax_rows {rows}x{cols} {kind}: emulation {r:.3f}, mutant {rm:.1f}x")
    assert r <= EMU_MAX and rm >= MUTANT_MIN
    assert torch.allclose(ref, torch.softmax(s.double() * 0.125, -1), rtol=1e-13, atol=0)


def emulate_softmax_groups(x, heads, S):
    x = x[:, :heads * S].unflatten(-1, (heads, S))
    e = torch.exp((x - x.amax(-1, keepdim=True)).float())
    return (e * (1.0 / e.sum(-1, keepdim=True))).flatten(-2)


@pytest.mark.parametrize("heads,S", [(8, 77), (5, 1), (20, 257)])
def test_softmax_groups_emulation_and_mutant(heads, S):
    x = torch.randn(40, heads * S + 13, generator=torch.Generator().manual_seed(S)) * 6
    ref, bound = NB.softmax_groups_ref_bound(x, heads, S)
    emu = emulate_softmax_groups(x, heads, S)
    r = NB.bound_ratio(emu, ref, NB.softmax_groups_ref_bound(x, heads, S, store=False)[1])
    assert NB.bound_ratio(emu.half(), ref, bound) <= 1.0
    rm = NB.bound_ratio(_one_off(emu, 3), ref, bound)
    print(f"softmax_groups heads={heads} S={S}: emulation {r:.3f}, mutant {rm:.1f}x")
    assert r <= EMU_MAX and rm >= MUTANT_MIN


def emulate_softmax_bwd(p, dp, scale, mutant=None):
    dot = (p.float() * dp).sum(-1, keepdim=True)
    if mutant == "delta_wrong_row":
        dot = dot.roll(1, 0)
    return scale * p.float() * (dp - dot)


@pytest.mark.parametrize("rows,cols", [(300, 77), (64, 4800), (8, 16384)])
def test_softmax_bwd_emulation_and_mutant(rows, cols):
    g = torch.Generator().manual_seed(cols)
    p = torch.softmax(torch.randn(rows, cols, generator=g) * 4, -1).half()
    dp = torch.randn(rows, cols, generator=g)
    ref, bound = NB.softmax_bwd_ref_bound(p, dp, 0.125)
    emu = emulate_softmax_bwd(p, dp, 0.125)
    r = NB.bound_ratio(emu, ref, NB.softmax_bwd_ref_bound(p, dp, 0.125, store=False)[1])
    assert NB.bound_ratio(emu.half(), ref, bound) <= 1.0
    rm = NB.bound_ratio(emulate_softmax_bwd(p, dp, 0.125, "delta_wrong_row").half(), ref, bound)
    print(f"softmax_bwd {rows}x{cols}: emulation {r:.3f}, mutant delta of the wrong row {rm:.1f}x")
    assert r <= EMU_MAX and rm >= MUTANT_MIN
    sr = (torch.randn(rows, cols, generator=g, dtype=torch.float64) * 4).requires_grad_(True)
    p64 = torch.softmax(sr * 0.125, -1)
    (p64 * dp.double()).sum().backward()
    assert torch.allclose(NB.softmax_bwd_ref_bound(p64.detach(), dp, 0.125)[0], sr.grad, rtol=1e-9, atol=1e-18)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _butterfly(x):
    """warp_sum over the lane axis (dim 1, 32 lanes) in fp32, xor 16 .. 1."""
    for o in (16, 8, 4, 2, 1):
        x = x + x[:, torch.arange(32) ^ o]
    return x


def _ln_stats(x, eps, Ce):
    """fp32 (mean, rstd) of layer_norm_kernel / layer_norm_bwd_kernel over the first Ce channels: lane l sums its
    vectors l, l + 32, ... in order, then butterfly warp sums."""
    rows, C = x.shape
    f = x.float()
    V = C // 8
    NV = (V + 31) // 32
    pad = torch.zeros(rows, NV * 32 * 8)
    pad[:, :Ce] = f[:, :Ce]
    mask = torch.zeros(NV * 32 * 8, dtype=torch.bool)
    mask[:Ce] = True
    lanes = pad.view(rows, NV, 32, 8).transpose(1, 2).reshape(rows, 32, NV * 8)       # per-lane element order
    lmask = mask.view(NV, 32, 8).transpose(0, 1).reshape(32, NV * 8)
    s = torch.zeros(rows, 32)
    for e in range(NV * 8):
        s = s + lanes[:, :, e]
    mean = (_butterfly(s)[:, :1] / Ce).float()
    q = torch.zeros(rows, 32)
    for e in range(NV * 8):
        d = torch.where(lmask[:, e], lanes[:, :, e] - mean, torch.zeros(()))
        q = q + d * d
    rstd = (1.0 / torch.sqrt(_butterfly(q)[:, :1].double() / Ce + eps)).float()
    return mean, rstd


def emulate_layer_norm(x, gamma, beta, eps, mutant=None):
    """layer_norm_kernel in fp32."""
    mean, rstd = _ln_stats(x, eps, x.shape[1] - 8 if mutant == "stats_c_minus_8" else x.shape[1])
    return (((x.float() - mean) * rstd) * gamma) + beta


def emulate_layer_norm_bwd(x, dy, gamma, eps, add=None, mutant=None):
    """layer_norm_bwd_kernel in fp32: xhat in place, m1 = mean(dy g), m2 = mean(dy g xhat), dx = rstd (dy g - m1 -
    xhat m2) (+ add), dgamma = sum dy xhat, dbeta = sum dy.  Returns fp32 (dx, dgamma, dbeta)."""
    C = x.shape[1]
    mean, rstd = _ln_stats(x, eps, C)
    xhat = (x.float() - mean) * rstd
    t = dy.float() * gamma
    m1 = t.sum(-1, keepdim=True) / C
    m2 = (t * xhat).sum(-1, keepdim=True) / C
    if mutant == "drop_mean_grad":
        m1 = torch.zeros_like(m1)
    dx = rstd * (t - m1 - xhat * m2)
    if add is not None:
        dx = add.float() + dx
    return dx, (dy.float() * xhat).sum(0), dy.float().sum(0)


@pytest.mark.parametrize("C,in_f32,add", [(8, True, True), (264, False, False), (640, True, True), (2048, False, True)])
def test_layer_norm_bwd_emulation_mutant_and_reference(C, in_f32, add):
    g = torch.Generator().manual_seed(C + 1)
    rows = 97
    x = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(F32 if in_f32 else F16)
    dy = torch.randn(rows, C, generator=g).half()
    gamma = torch.randn(C, generator=g) * 0.3 + 1.0
    addt = torch.randn(rows, C, generator=g) if add else None
    res = NB.layer_norm_bwd_ref_bound(x, dy, gamma, 1e-5, addt, store=False)
    emu = dict(zip(("dx", "dgamma", "dbeta"), emulate_layer_norm_bwd(x, dy, gamma, 1e-5, addt)))
    ratios = {n: NB.bound_ratio(emu[n], *res[n]) for n in res}
    full = NB.layer_norm_bwd_ref_bound(x, dy, gamma, 1e-5, addt, out_f32=False)
    assert NB.bound_ratio(emu["dx"].half(), *full["dx"]) <= 1.0
    bad = emulate_layer_norm_bwd(x, dy, gamma, 1e-5, addt, "drop_mean_grad")[0]
    rm = NB.bound_ratio(bad, *res["dx"])
    print(f"layer_norm_bwd C={C}: emulation {ratios}, mutant mean-gradient term dropped {rm:.1f}x")
    assert max(ratios.values()) <= EMU_MAX and rm >= MUTANT_MIN
    xr = x.double().requires_grad_(True)
    gr = gamma.double().requires_grad_(True)
    br = torch.zeros(C, dtype=torch.float64, requires_grad=True)
    (F.layer_norm(xr, (C,), gr, br, 1e-5) * dy.double()).sum().backward()
    want = {"dx": xr.grad + (addt.double() if add else 0), "dgamma": gr.grad, "dbeta": br.grad}
    for n in want:
        assert torch.allclose(res[n][0], want[n], rtol=1e-9, atol=1e-12), n


@pytest.mark.parametrize("C", [8, 256, 264, 512, 520, 768, 776, 1024, 1032, 1280, 1288, 1536, 1544, 1792, 1800, 2048])
@pytest.mark.parametrize("in_f32", [True, False])
def test_layer_norm_emulation_and_mutant(C, in_f32):
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(33, C, generator=g) * 2 + 0.3).to(F32 if in_f32 else F16)
    gamma = torch.randn(C, generator=g) * 0.2 + 1.0
    beta = torch.randn(C, generator=g) * 0.2
    ref, bound = NB.layer_norm_ref_bound(x, gamma, beta, 1e-5)
    emu = emulate_layer_norm(x, gamma, beta, 1e-5)
    r = NB.bound_ratio(emu, ref, NB.layer_norm_ref_bound(x, gamma, beta, 1e-5, store=False)[1])
    assert NB.bound_ratio(emu.half(), ref, bound) <= 1.0
    msg = f"layer_norm C={C} {'f32' if in_f32 else 'f16'}: emulation {r:.3f}"
    if C > 8:
        rm = NB.bound_ratio(emulate_layer_norm(x, gamma, beta, 1e-5, "stats_c_minus_8").half(), ref, bound)
        msg += f", mutant statistics over C-8 channels {rm:.1f}x"
        assert rm >= MUTANT_MIN
    print(msg)
    assert r <= EMU_MAX
    assert torch.allclose(ref, F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5), rtol=1e-12,
                          atol=1e-12)


# ------------------------------------------------------------------------------------------------ GroupNorm
def _gn_stats(x, eps, groups, sms=132):
    """gn_stats_kernel: per-thread fp32 shifted sums over the kernel's pixel partition, merged in fp64; returns the
    fp32 (mean, rstd) [NB, groups] the apply and backward kernels read."""
    NBt, H, W, C = x.shape
    HW = H * W
    V = C // 8
    rpb = max(1, 256 // V)
    target = (sms * 8 + NBt - 1) // NBt
    ppc = max((HW + target - 1) // target, rpb * 4)
    f = x.float().reshape(NBt, HW, C)
    S1 = torch.zeros(NBt, C, dtype=torch.float64)
    S2 = torch.zeros(NBt, C, dtype=torch.float64)
    for p0 in range(0, HW, ppc):
        p1 = min(HW, p0 + ppc)
        for r in range(rpb):
            idx = torch.arange(p0 + r, p1, rpb)
            if idx.numel() == 0:
                continue
            xs = f[:, idx]
            sh = xs[:, 0]
            s = torch.zeros(NBt, C)
            q = torch.zeros(NBt, C)
            for u in range(idx.numel()):
                d = xs[:, u] - sh
                q = (q.double() + d.double() * d.double()).float()         # fmaf(d, d, q)
                s = s + d
            n, shd, s1 = float(idx.numel()), sh.double(), s.double()
            S1 += s1 + n * shd
            S2 += q.double() + 2.0 * shd * s1 + n * shd * shd
    cg = C // groups
    su, sq = S1.view(NBt, groups, cg).sum(-1), S2.view(NBt, groups, cg).sum(-1)
    mean = su / (HW * cg)
    var = (sq / (HW * cg) - mean * mean).clamp_min(0)
    return mean.float(), (1.0 / torch.sqrt(var + eps)).float()


def emulate_group_norm(x, gamma, beta, eps, groups, silu, sms=132, mutant=None):
    """gn_apply_kernel with _gn_stats: t = x a + b and SiLU in fp32 (before the fp16 store).  x [NB, H, W, C]."""
    NBt, H, W, C = x.shape
    f = x.float().reshape(NBt, H * W, C)
    gmean, grstd = _gn_stats(x, eps, groups, sms)
    grp = torch.arange(C) // (C // groups)
    if mutant is not None:                                   # channel `mutant` normalised with its neighbour group
        grp = grp.clone()
        grp[mutant] = grp[mutant] - 1
    a = grstd[:, grp] * gamma
    b = beta - gmean[:, grp] * a
    t = (f.double() * a[:, None].double() + b[:, None].double()).float()
    y = t / (1.0 + torch.exp(-t)) if silu else t
    return y.view(NBt, H, W, C)


def emulate_group_norm_bwd(x, dy, gamma, beta, eps, groups, silu, add=None, mutant=None):
    """gn_bwd_sums_kernel + gn_bwd_apply_kernel in fp32: S = per-channel (sum dz, sum dz xhat), A / B = group sums of
    gamma S over HW cg, dx = rstd (dz gamma - A - xhat B) (+ add); dgamma / dbeta = S summed over the images.
    `mutant` = g: group g's A and B are summed over the channels of group g - 1."""
    NBt, H, W, C = x.shape
    cg = C // groups
    f = x.float().reshape(NBt, H * W, C)
    gmean, grstd = _gn_stats(x, eps, groups)
    grp = torch.arange(C) // cg
    rs = grstd[:, grp][:, None]
    ms = -gmean[:, grp][:, None] * rs
    a = rs * gamma
    b = beta - gmean[:, grp][:, None] * a
    d = dy.float().reshape(NBt, H * W, C)
    if silu:
        z = f * a + b
        sg = 1.0 / (1.0 + torch.exp(-z))
        dz = d * (sg * (1.0 + z * (1.0 - sg)))
    else:
        dz = d
    xhat = f * rs + ms
    S0, S1 = dz.sum(1), (dz * xhat).sum(1)                       # [NB, C]
    inv_m = 1.0 / (H * W * cg)
    A = (gamma * S0).view(NBt, groups, cg).sum(-1) * inv_m
    B = (gamma * S1).view(NBt, groups, cg).sum(-1) * inv_m
    if mutant is not None:
        A, B = A.clone(), B.clone()
        A[:, mutant], B[:, mutant] = A[:, mutant - 1], B[:, mutant - 1]
    dx = dz * (rs * gamma) - (rs * A[:, grp][:, None]) - xhat * (rs * B[:, grp][:, None])
    dx = dx.view(NBt, H, W, C)
    if add is not None:
        dx = add.float() + dx
    return dx, S1.sum(0), S0.sum(0)


@pytest.mark.parametrize("C1,C2,in_f32,silu,add", [(640, 320, False, True, True), (1280, 640, True, False, False),
                                                   (320, 0, True, True, True)])
def test_group_norm_bwd_emulation_mutant_and_reference(C1, C2, in_f32, silu, add):
    g = torch.Generator().manual_seed(C1 + C2 + 3)
    H, W = 5, 7
    C = C1 + C2
    x = torch.cat([torch.randn(2, H, W, C1, generator=g) * 1.5 + 0.3,
                   torch.randn(2, H, W, C2, generator=g) * 0.7 - 0.2], -1).to(F32 if in_f32 else F16)
    dy = torch.randn(2, H, W, C, generator=g).half()
    gamma = torch.randn(C, generator=g) * 0.3 + 1.0
    beta = torch.randn(C, generator=g) * 0.2
    addt = torch.randn(2, H, W, C, generator=g) if add else None
    cnt = NB.gn_thread_count(2, H * W, C)
    res = NB.group_norm_bwd_ref_bound(x, dy, gamma, beta, 1e-5, 32, silu, cnt, addt, store=False)
    emu = dict(zip(("dx", "dgamma", "dbeta"), emulate_group_norm_bwd(x, dy, gamma, beta, 1e-5, 32, silu, addt)))
    ratios = {n: NB.bound_ratio(emu[n], *res[n]) for n in res}
    full = NB.group_norm_bwd_ref_bound(x, dy, gamma, beta, 1e-5, 32, silu, cnt, addt, out_f32=False)
    assert NB.bound_ratio(emu["dx"].half(), *full["dx"]) <= 1.0
    gs = C1 // (C // 32) if C2 else 5                         # the straddling group, if any
    bad = emulate_group_norm_bwd(x, dy, gamma, beta, 1e-5, 32, silu, addt, mutant=gs)[0]
    rm = NB.bound_ratio(bad, *res["dx"])
    print(f"group_norm_bwd ({C1}, {C2}): emulation {ratios}, mutant group {gs} summed over its neighbour {rm:.1f}x")
    assert max(ratios.values()) <= EMU_MAX and rm >= MUTANT_MIN
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y = F.group_norm(xr.permute(0, 3, 1, 2), 32, gr, br, 1e-5)
    ((F.silu(y) if silu else y) * dy.double().permute(0, 3, 1, 2)).sum().backward()
    want = {"dx": xr.grad + (addt.double() if add else 0), "dgamma": gr.grad, "dbeta": br.grad}
    for n in want:
        assert torch.allclose(res[n][0], want[n], rtol=1e-9, atol=1e-12), n


GN_CASES = [  # (C1, C2, H, W, in_f32, silu)
    (320, 0, 5, 7, False, True), (1280, 640, 3, 5, True, True), (640, 320, 7, 9, False, False),
    (640, 640, 4, 5, True, True), (320, 320, 6, 11, False, True), (1280, 1280, 2, 3, False, True),
    (128, 0, 50, 37, True, False)]


@pytest.mark.parametrize("C1,C2,H,W,in_f32,silu", GN_CASES)
def test_group_norm_emulation_within_half_the_bound(C1, C2, H, W, in_f32, silu):
    g = torch.Generator().manual_seed(C1 + C2)
    dt = F32 if in_f32 else F16
    x = torch.cat([torch.randn(2, H, W, C1, generator=g) + 0.5, torch.randn(2, H, W, C2, generator=g) * 2.0], -1).to(dt)
    C = C1 + C2
    gamma = torch.randn(C, generator=g) * 0.2 + 1.0
    beta = torch.randn(C, generator=g) * 0.2
    cnt = NB.gn_thread_count(2, H * W, C)
    ref, bound = NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, silu, cnt)
    emu = emulate_group_norm(x, gamma, beta, 1e-5, 32, silu)
    r = NB.bound_ratio(emu, ref, NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, silu, cnt, store=False)[1])
    assert NB.bound_ratio(emu.half(), ref, bound) <= 1.0
    print(f"group_norm ({C1}, {C2}) {H}x{W} {'f32' if in_f32 else 'f16'} silu={silu}: emulation {r:.3f}")
    assert r <= EMU_MAX
    want = F.group_norm(x.double().permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5)
    want = (F.silu(want) if silu else want).permute(0, 2, 3, 1)
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("C1,C2", [(1280, 640), (640, 320)])
def test_group_norm_straddling_channel_in_the_wrong_group_exceeds_the_bound(C1, C2):
    C = C1 + C2
    cg = C // 32
    assert C1 % cg                                            # a group straddles the concatenation
    g = torch.Generator().manual_seed(7)
    x = torch.cat([torch.randn(2, 4, 6, C1, generator=g) + 0.5, torch.randn(2, 4, 6, C2, generator=g) * 2.0], -1).half()
    gamma, beta = torch.ones(C), torch.zeros(C)
    ref, bound = NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, True, NB.gn_thread_count(2, 24, C))
    r = NB.bound_ratio(emulate_group_norm(x, gamma, beta, 1e-5, 32, True, mutant=C1).half(), ref, bound)
    print(f"group_norm ({C1}, {C2}): channel {C1} in the neighbour group {r:.1f}x the bound")
    assert r >= MUTANT_MIN


def test_group_norm_mean50_stress_emulation():
    """|mean| >> std: the shifted sums keep the variance; an unshifted fp32 sum of squares would not."""
    g = torch.Generator().manual_seed(41)
    C = 128
    x = (torch.randn(1, 48, 48, C, generator=g) + 50.0 * (1.0 + 0.2 * torch.arange(C) / C)).float()
    gamma = torch.randn(C, generator=g) * 0.2 + 1.0
    beta = torch.randn(C, generator=g) * 0.2
    cnt = NB.gn_thread_count(1, 48 * 48, C)
    _, bound = NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, True, cnt, store=False)
    ref, full = NB.group_norm_ref_bound(x, gamma, beta, 1e-5, 32, True, cnt)
    emu = emulate_group_norm(x, gamma, beta, 1e-5, 32, True)
    r = NB.bound_ratio(emu, ref, bound)
    assert NB.bound_ratio(emu.half(), ref, full) <= 1.0
    print(f"group_norm mean-50 stress: emulation {r:.3f}")
    assert r <= EMU_MAX
