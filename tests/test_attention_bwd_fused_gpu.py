"""GPU tests of the fused flash attention backward (csrc/attention_bwd.cu, `ops.attention_bwd`): every element of dQ,
dK and dV within the fp64 bound of tests/numerics_bounds.py at head widths 40 / 64 / 80 / 160, plain and joint
(kv_segments = 2), at the kernels' tile boundaries and at training lengths; bitwise reruns; the memory footprint in
a fused d(qkv) buffer; the tiny SD-2 and SD-1 joint UNets against the fp32 oracle's autograd; and the memory the
SD-1 joint level-0 backward needs at 768 x 768."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import attention_bwd_cases as ABC  # noqa: E402
import footprint_cases as FC  # noqa: E402
import numerics_bounds as NB  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = torch.float16
REGIMES = ["gauss", "peaked", "uniform", "ramp_up"]
TILE = 64                                    # query rows of a dQ CTA, key rows of a dK/dV CTA, keys of a dQ tile


def fused_bwd(q, k, v, do, heads, scale, kv_segments=1):
    """The fused kernels on their own, whatever backward.attention_bwd would route the shape to."""
    from diffusion_e2e_ft_b200 import ops
    C = q.shape[-1]
    o, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)
    delta = ops.rowdot_heads_d(do, o, heads, C // heads)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    return ops.attention_bwd(q, k, v, do, lse, delta, dq, dk, dv, heads, scale, kv_segments)


def _inputs(B, heads, D, T, Tk, regime, kv_segments, seed):
    q, k, v, scale = NB.attention_inputs(B, heads, D, T, Tk, regime, seed=seed, device=DEV, kv_segments=kv_segments)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    do = torch.randn(B, T, q.shape[-1], generator=g).half().to(DEV)
    return q, k, v, do, scale


def _heads(t, heads):
    return t.double().unflatten(-1, (heads, -1)).transpose(1, 2)             # [B, heads, L, D]


def check_within_bound(q, k, v, do, heads, scale, kv_segments, got, tag):
    """Every element of dq / dk / dv against attention_bwd_ref_bound.  A joint pair (images i, i + B/2) is one
    attention problem of 2T queries over 2Tk keys, as the reference's joint processor concatenates them."""
    B = q.shape[0]
    qh, kh, vh, doh = (_heads(t, heads) for t in (q, k, v, do))
    gq, gk, gv = (_heads(t, heads) for t in got)
    if kv_segments == 2:
        h = B // 2
        pair = lambda t: torch.cat([t[:h], t[h:]], 2)                        # [B/2, heads, 2L, D]
        qh, kh, vh, doh, gq, gk, gv = (pair(t) for t in (qh, kh, vh, doh, gq, gk, gv))
    worst = {}
    for b in range(qh.shape[0]):
        for hh in range(heads):
            res = NB.attention_bwd_ref_bound(qh[b, hh], kh[b, hh], vh[b, hh], doh[b, hh], scale)
            for name, g_ in (("dq", gq[b, hh]), ("dk", gk[b, hh]), ("dv", gv[b, hh])):
                worst[name] = max(worst.get(name, 0.0), NB.bound_ratio(g_, *res[name]))
            del res
    print(f"{tag}: max err / bound {', '.join(f'{k_} {v_:.3f}' for k_, v_ in worst.items())}")
    assert max(worst.values()) <= 1.0, worst


# ------------------------------------------------------------------------------------------------ fp64 bounds
_EDGES = [(n, n) for n in (TILE - 1, TILE, TILE + 1, 3 * TILE + 1)] + [(TILE + 1, 2 * TILE - 1), (3 * TILE + 1, 80)]


@pytest.mark.parametrize("D", [40, 64, 80, 160])
@pytest.mark.parametrize("kv_segments", [1, 2])
@pytest.mark.parametrize("T,Tk", _EDGES)
def test_fused_bwd_within_bound_at_tile_edges(D, kv_segments, T, Tk):
    """Lengths at the 64-row tiles of both kernels (and the 32-query tiles of the D = 80 / 160 dK/dV kernel: 63, 65,
    193 are 32 k -+ 1); the input regime cycles with the case."""
    regime = REGIMES[(D + T + Tk + kv_segments) % 4]
    B, heads = (4 if kv_segments == 2 else 2), 2
    q, k, v, do, scale = _inputs(B, heads, D, T, Tk, regime, kv_segments, seed=D + T + 7 * Tk)
    got = fused_bwd(q, k, v, do, heads, scale, kv_segments)
    torch.cuda.synchronize()
    check_within_bound(q, k, v, do, heads, scale, kv_segments, got,
                       f"fused bwd D={D} kv={kv_segments} T={T} Tk={Tk} {regime}")


@pytest.mark.parametrize("T,D,heads,kv_segments", [(4800, 64, 5, 1), (6688, 40, 8, 1), (9216, 64, 5, 1),
                                                   (4800, 40, 8, 2)])
def test_fused_bwd_training_lengths_within_bound(T, D, heads, kv_segments):
    """4800 = 480 x 640 (Hypersim), 6688 = 352 x 1216 (Virtual KITTI crop), 9216 = 768 x 768, each at level 0."""
    from diffusion_e2e_ft_b200 import backward as bw
    B = 2 if kv_segments == 2 else 1
    q, k, v, do, scale = _inputs(B, heads, D, T, T, "gauss", kv_segments, seed=T + D)
    got = bw.attention_bwd(q, k, v, do, heads, scale, kv_segments=kv_segments)
    torch.cuda.synchronize()
    check_within_bound(q, k, v, do, heads, scale, kv_segments, got, f"fused bwd D={D} heads={heads} T={T}")


# ------------------------------------------------------------------------------------------------ determinism
@pytest.mark.parametrize("D", [40, 64, 80, 160])
@pytest.mark.parametrize("kv_segments", [1, 2])
def test_fused_bwd_reruns_are_bitwise_equal(D, kv_segments):
    q, k, v, do, scale = _inputs(4, 3, D, 333, 333, "gauss", kv_segments, seed=D)
    a = fused_bwd(q, k, v, do, 3, scale, kv_segments)
    b = fused_bwd(q, k, v, do, 3, scale, kv_segments)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))


# ------------------------------------------------------------------------------------------------ footprint
@pytest.mark.parametrize("D,Lq,Lk,kv_segments", [(40, TILE + 1, 2 * TILE + 1, 1), (64, 3 * TILE + 1, TILE - 1, 1),
                                                 (80, TILE, TILE, 2), (160, TILE - 1, 3 * TILE + 1, 1)])
def test_fused_bwd_footprint_in_a_fused_dqkv_buffer(D, Lq, Lk, kv_segments):
    """dq / dk / dv are column blocks of fused [B, L, 3C] buffers: the other columns, the batch gaps and the guard
    bands keep their sentinels, inputs stay unchanged, poisoned memory outside the inputs changes nothing, and the
    strided call equals the compact one."""
    from test_kernel_footprint_gpu import footprint_violations
    B = 4 if kv_segments == 2 else 2
    case = FC.paired(ABC.attention_bwd_case, f"attention_bwd_fused_d{D}_{Lq}_{Lk}", D, B=B, Lq=Lq, Lk=Lk,
                     kv_segments=kv_segments)
    bad = footprint_violations(case)
    assert not bad, "; ".join(bad)


@pytest.mark.parametrize("case", ABC.attention_bwd_cases(), ids=lambda c: c.name)
def test_fused_bwd_footprint_cases(case):
    """The attention_bwd_cases table: ragged lengths at every head width and a joint case."""
    from test_kernel_footprint_gpu import footprint_violations
    bad = footprint_violations(case)
    assert not bad, f"{case.name}: " + "; ".join(bad)


def test_cuda_tensors_take_the_fused_kernels(monkeypatch):
    """Every key count above one, cross-attention over 77 tokens included, and every joint call: one fused call."""
    from diffusion_e2e_ft_b200 import backward as bw
    from diffusion_e2e_ft_b200 import ops
    seen = []
    fused = ops.attention_bwd
    monkeypatch.setattr(ops, "attention_bwd", lambda *a, **k: (seen.append(a[1].shape[1]), fused(*a, **k))[1])
    monkeypatch.setattr(bw, "_attention_bwd_gemm", lambda *a, **k: pytest.fail("GEMM composition on CUDA tensors"))
    for Tk, kv in ((1, 1), (2, 1), (77, 1), (144, 1), (40, 2)):
        q, k, v, do, scale = _inputs(4 if kv == 2 else 2, 2, 64, 70, Tk, "gauss", kv, seed=Tk)
        bw.attention_bwd(q, k, v, do, 2, scale, kv_segments=kv)
    assert seen == [2, 77, 144, 40]


# ------------------------------------------------------------------------------------------------ graph level
def test_tiny_sd2_unet_backward_on_the_fused_kernels():
    """24 x 24 latents: self-attention over 576 and 144 keys takes the fused kernels; gates of
    tests/test_engine_gpu.py's UNet-backward check."""
    import engine_checks as EC
    r = EC.run_unet_backward_tiny(device=DEV, hw=(24, 24))
    print("tiny_sd2_backward", r)
    assert not r["missing"], r["missing"]
    assert r["forward"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


def test_tiny_sd1_joint_unet_backward_on_the_fused_kernels(monkeypatch):
    """SD-1 head widths, joint attention (kv_segments = 2 in one call) at 24 x 20 latents; gates of
    tests/test_sd1_attention_gpu.py."""
    import engine_checks as EC
    import sd1_checks as S
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    S.sd1_tiny(monkeypatch)
    r = EC.run_unet_backward_tiny(device=DEV, hw=(24, 20), kind="geowizard")
    print("tiny_sd1_backward", r)
    assert not r["missing"], r["missing"]
    assert r["forward"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


# ------------------------------------------------------------------------------------------------ memory
def test_sd1_joint_level0_backward_memory_at_768():
    """One depth / normal pair at 768 x 768 (T = 9216 per image, 8 heads x 40): P and dS of the pair would be
    2 x 8 x 18432^2 x 2 B x 2 = 10.9 GB.  The fused backward allocates O, lse, delta and dq / dk / dv only."""
    from diffusion_e2e_ft_b200 import backward as bw
    B, T, heads, D = 2, 9216, 8, 40
    C = heads * D
    g = torch.Generator(device="cpu").manual_seed(3)
    qkv = (torch.randn(B, T, 3 * C, generator=g) * 0.5).half().to(DEV)
    do = torch.randn(B, T, C, generator=g).half().to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    dq, dk, dv = bw.attention_bwd(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], do, heads, D ** -0.5,
                                  kv_segments=2)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    act = B * T * C * 2                                     # one [B, T, C] fp16 tensor: 11.8 MB
    print(f"sd1 joint level-0 backward at 768^2: peak growth {growth / 1e6:.1f} MB")
    assert growth <= 5 * act, (growth, act)              # dq, dk, dv, O + lse / delta, slack
    assert torch.isfinite(dq.float()).all() and torch.isfinite(dk.float()).all() and torch.isfinite(dv.float()).all()
