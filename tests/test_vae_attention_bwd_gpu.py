"""GPU tests of the d=512 attention in training (csrc/attention_d512_bwd.cu, the LSE store of attention_d512_kernel,
`ops.attention_d512(..., want_lse=True)`, `ops.rowdot_d512`, `ops.attention_d512_bwd`): every element of dQ, dK and
dV within the fp64 bound of tests/numerics_bounds.py at ragged lengths around each tile and at 768 x 768, sampled rows
and keys at 65536; bitwise reruns; O unchanged by the LSE store; the memory footprint of the new entry points; the
training forward of the block and of the decoder equal to inference with memory-efficient attention on; the block's
data gradient against the unfused path and the fp32 oracle; the block at L = 65536 with its memory; and a tiny
Marigold E2E micro-step on the fused path against the oracle's autograd."""
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import numerics_bounds as NB  # noqa: E402
import vae_attention_bwd_cases as VC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REGIMES = ["gauss", "peaked", "uniform", "ramp_up"]
GOLDEN = os.path.join(HERE, "golden", "attention_d512_o.pt")


def fused_bwd(q, k, v, do, scale):
    """Forward with lse, delta and the fused backward: what the training block runs."""
    from diffusion_e2e_ft_b200 import ops
    o, lse = ops.attention_d512(q, k, v, scale, want_lse=True)
    delta = ops.rowdot_d512(do, o)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    return ops.attention_d512_bwd(q, k, v, do, lse, delta, dq, dk, dv, scale)


def _inputs(B, T, Tk, regime, seed):
    q, k, v, scale = NB.attention_inputs(B, 1, 512, T, Tk, regime, seed=seed, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    do = torch.randn(B, T, 512, generator=g).half().to(DEV)
    return q, k, v, do, scale


def check_within_bound(q, k, v, do, scale, got, tag):
    worst = {}
    for b in range(q.shape[0]):
        res = NB.attention_bwd_ref_bound(q[b].double(), k[b].double(), v[b].double(), do[b].double(), scale)
        for name, g_ in zip(("dq", "dk", "dv"), got):
            worst[name] = max(worst.get(name, 0.0), NB.bound_ratio(g_[b].double(), *res[name]))
        del res
    print(f"{tag}: max err / bound {', '.join(f'{k_} {v_:.3f}' for k_, v_ in worst.items())}")
    assert max(worst.values()) <= 1.0, worst


# ------------------------------------------------------------------------------------------------ fp64 bounds
# 16-query / 16-key tiles of the dK and dQ kernels, 32-query tiles of the dV kernel, 64-row resident blocks
_EDGES = [(1, 1), (15, 17), (17, 15), (31, 33), (33, 31), (63, 65), (65, 63), (70, 77), (1, 65), (65, 1)]


@pytest.mark.parametrize("T,Tk", _EDGES)
def test_d512_bwd_within_bound_at_tile_edges(T, Tk):
    regime = REGIMES[(T + Tk) % 4]
    q, k, v, do, scale = _inputs(2, T, Tk, regime, seed=T + 7 * Tk)
    got = fused_bwd(q, k, v, do, scale)
    torch.cuda.synchronize()
    check_within_bound(q, k, v, do, scale, got, f"d512 bwd T={T} Tk={Tk} {regime}")


def test_d512_bwd_within_bound_at_768():
    """9216 = 768 x 768 latents / 8, the decoder mid-block at the training resolution."""
    q, k, v, do, scale = _inputs(1, 9216, 9216, "gauss", seed=9216)
    got = fused_bwd(q, k, v, do, scale)
    torch.cuda.synchronize()
    check_within_bound(q, k, v, do, scale, got, "d512 bwd T=9216")


def test_d512_bwd_sampled_at_65536():
    """L = 65536 (2048 x 2048 images): dQ of sampled query rows against their fp64 bound (a row of dQ needs only its
    own query), dK / dV of sampled keys against fp64 sums over every query (lse in fp64 over all keys)."""
    L = 65536
    q, k, v, do, scale = _inputs(1, L, L, "gauss", seed=65536)
    got = [t[0] for t in fused_bwd(q, k, v, do, scale)]
    torch.cuda.synchronize()
    g = torch.Generator(device="cpu").manual_seed(1)
    rows = torch.randint(0, L, (24,), generator=g).to(DEV)
    keys = torch.cat([torch.randint(0, L, (22,), generator=g), torch.tensor([0, L - 1])]).to(DEV)
    qd, kd, vd, dod = (t[0].double() for t in (q, k, v, do))
    res = NB.attention_bwd_ref_bound(qd[rows], kd, vd, dod[rows], scale)
    r = NB.bound_ratio(got[0][rows].double(), *res["dq"])
    print(f"d512 bwd L=65536 sampled dq rows: max err / bound {r:.3f}")
    assert r <= 1.0
    dk = torch.zeros(len(keys), 512, dtype=torch.float64, device=DEV)
    dv = torch.zeros_like(dk)
    for i in range(0, L, 2048):
        qc, doc = qd[i:i + 2048], dod[i:i + 2048]
        s = qc @ kd.t() * scale
        lse = s.logsumexp(-1, keepdim=True)
        o = torch.exp(s - lse) @ vd
        p = torch.exp(s[:, keys] - lse)
        ds = p * (doc @ vd[keys].t() - (doc * o).sum(-1, keepdim=True)) * scale
        dk += ds.t() @ qc
        dv += p.t() @ doc
        del s
    for name, ref, gk in (("dk", dk, got[1][keys]), ("dv", dv, got[2][keys])):
        rel = ((gk.double() - ref).norm() / ref.norm()).item()
        print(f"d512 bwd L=65536 sampled {name} keys: rel err {rel:.2e}")
        assert rel <= 5e-3, (name, rel)


# ------------------------------------------------------------------------------------------------ determinism, O bits
def test_d512_bwd_reruns_are_bitwise_equal():
    q, k, v, do, scale = _inputs(3, 333, 333, "gauss", seed=3)
    a = fused_bwd(q, k, v, do, scale)
    b = fused_bwd(q, k, v, do, scale)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))


def _golden_inputs():
    g = torch.Generator(device="cpu").manual_seed(512)
    qkv = (torch.randn(2, 77, 1536, generator=g) * 0.6).half().to(DEV)
    return qkv[..., :512], qkv[..., 512:1024], qkv[..., 1024:]


def test_lse_entry_keeps_the_output_bits():
    """O of the LSE entry equals b200_attention_d512's bit for bit, and both equal the output the kernel gave before
    it had the LSE store (tests/golden/attention_d512_o.pt); lse is the log2-domain log-sum-exp."""
    from diffusion_e2e_ft_b200 import ops
    q, k, v = _golden_inputs()
    scale = 512 ** -0.5
    plain = ops.attention_d512(q, k, v, scale)
    o, lse = ops.attention_d512(q, k, v, scale, want_lse=True)
    torch.cuda.synchronize()
    assert torch.equal(o.view(torch.int16), plain.view(torch.int16))
    want = torch.load(GOLDEN)
    assert torch.equal(o.view(torch.int16).cpu(), want)
    ref = (q.double() @ k.double().transpose(1, 2) * scale).logsumexp(-1) / math.log(2.0)
    assert (lse.double() - ref).abs().max().item() <= 1e-4
    for Lq, Lk in ((9216, 9216), (65, 1)):
        q2, k2, v2, _, scale = _inputs(2, Lq, Lk, "gauss", seed=Lq)
        a = ops.attention_d512(q2, k2, v2, scale)
        b, _ = ops.attention_d512(q2, k2, v2, scale, want_lse=True)
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------ footprint
@pytest.mark.parametrize("case", VC.vae_attention_bwd_cases(), ids=lambda c: c.name)
def test_new_entry_points_keep_their_footprint(case):
    """Guard bands, the other columns of the fused rows and the batch gaps keep their sentinels, inputs stay unchanged,
    poisoned memory outside the inputs changes nothing, and the strided call equals the compact one."""
    from test_kernel_footprint_gpu import footprint_violations
    bad = footprint_violations(case)
    assert not bad, f"{case.name}: " + "; ".join(bad)


# ------------------------------------------------------------------------------------------------ block and decoder
def _block(seed=0):
    from diffusion_e2e_ft_b200.vae import VAEAttention
    torch.manual_seed(seed)
    att = VAEAttention(512, 32).eval().requires_grad_(False)
    with torch.no_grad():
        for p in att.parameters():
            p.normal_(0, 0.05)
        att.group_norm.weight.add_(1.0)
    return att.to(DEV)


def test_block_training_forward_equals_inference_forward():
    from diffusion_e2e_ft_b200 import autograd_blocks as ab
    att = _block()
    att.memory_efficient = True
    x = torch.randn(2, 24, 20, 512, device=DEV)
    with torch.no_grad():
        want = att.run(x)
    got = ab.vae_attention(att, x.clone().requires_grad_(True))
    torch.cuda.synchronize()
    assert torch.equal(got.detach(), want)


def test_decoder_training_forward_equals_inference_forward_memory_efficient():
    """The GPU twin of test_block_forward_cpu's decoder check, on a decoder whose mid-block is 512 wide."""
    import engine_checks as EC
    import make_golden as MG
    from oracle.vae import AutoencoderKLRef
    from oracle.unet import seeded_init
    vae_ref = seeded_init(AutoencoderKLRef(MG.tiny_vae_config(block_out_channels=(64, 128, 512))), seed=77).eval()
    _, vae = EC.engine_from_oracle(MG.build_tiny()[0], vae_ref, DEV)
    vae.enable_xformers_memory_efficient_attention()
    z = MG.inputs(4, 2, 4, 12, 10, scale=0.5).to(DEV)
    with torch.no_grad():
        want = vae.decoder(z)
    got = vae.decoder(z.clone().requires_grad_(True))
    torch.cuda.synchronize()
    assert torch.equal(got.detach(), want)


def _oracle_dx(att, x, dout):
    from oracle.vae import VAEAttention as Ref
    ref = Ref(512, 32, att.eps).to(DEV)
    ref.load_state_dict(att.state_dict())
    xr = x.detach().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ref(xr).backward(dout.permute(0, 3, 1, 2))
    return xr.grad.permute(0, 2, 3, 1)


@pytest.mark.parametrize("hw", [(24, 20), (96, 96)])
def test_block_dx_matches_unfused_and_oracle(hw):
    """d/dx of the block: fused path within 2e-3 (relative L2) of the unfused path and within 5e-3 of fp32 autograd
    through the oracle (fp16 GEMM operands on both engine paths).  96 x 96 = 768^2 / 8."""
    from diffusion_e2e_ft_b200 import autograd_blocks as ab
    torch.backends.cuda.matmul.allow_tf32 = False
    att = _block(1)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, *hw, 512, generator=g).to(DEV)
    dout = torch.randn(2, *hw, 512, generator=g).to(DEV)
    grads = {}
    for me in (True, False):
        att.memory_efficient = me
        xe = x.clone().requires_grad_(True)
        ab.vae_attention(att, xe).backward(dout)
        grads[me] = xe.grad
    want = _oracle_dx(att, x, dout)
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()          # noqa: E731
    r_unf, r_fused, r_ref = rel(grads[True], grads[False]), rel(grads[True], want), rel(grads[False], want)
    print(f"block dx {hw}: fused vs unfused {r_unf:.2e}, fused vs oracle {r_fused:.2e}, unfused vs oracle {r_ref:.2e}")
    assert r_unf <= 2e-3 and r_fused <= 5e-3, (r_unf, r_fused, r_ref)


def test_block_forward_backward_at_65536_in_linear_memory():
    """L = 65536 (a 2048 x 2048 image): one image has 2^32 scores, which the unfused path cannot index, so training
    takes the flash kernels even without memory-efficient attention.  The backward's peak growth stays a few hundred
    MB; an L x L fp16 buffer alone would be 8.6 GB."""
    from diffusion_e2e_ft_b200 import autograd_blocks as ab
    att = _block(2)
    x = torch.randn(1, 256, 256, 512, device=DEV, requires_grad=True)
    out = ab.vae_attention(att, x)
    dout = torch.randn_like(out)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out.backward(dout)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    print(f"attention block backward at L=65536: peak growth {growth / 1e6:.1f} MB")
    assert growth <= 600e6, growth
    assert torch.isfinite(x.grad).all() and x.grad.abs().max() > 0


# ------------------------------------------------------------------------------------------------ E2E micro-step
@pytest.mark.parametrize("modality,tol", [("depth", 3e-2), ("normals", 6e-2)])
def test_training_micro_step_gradients_match_oracle_memory_efficient(monkeypatch, modality, tol):
    """engine_checks.run_training_step_tiny (the gates of test_engine_gpu's micro-step check) with a VAE whose
    mid-blocks are 512 wide and `vae.enable_xformers_memory_efficient_attention()`: the decoder's attention
    backward runs the fused d=512 kernels."""
    import engine_checks as EC
    import make_golden as MG
    from diffusion_e2e_ft_b200 import ops
    from oracle.vae import AutoencoderKLRef
    from oracle.unet import seeded_init
    build = MG.build_tiny

    def build_512(kind="marigold"):
        unet, _ = build(kind)
        vae = seeded_init(AutoencoderKLRef(MG.tiny_vae_config(block_out_channels=(64, 128, 512))), seed=77).eval()
        return unet, vae
    monkeypatch.setattr(MG, "build_tiny", build_512)
    efo = EC.engine_from_oracle

    def efo_me(*a, **k):
        unet, vae = efo(*a, **k)
        vae.enable_xformers_memory_efficient_attention()
        return unet, vae
    monkeypatch.setattr(EC, "engine_from_oracle", efo_me)
    calls = []
    bwd = ops.attention_d512_bwd
    monkeypatch.setattr(ops, "attention_d512_bwd", lambda *a, **k: (calls.append(a[0].shape), bwd(*a, **k))[1])
    r = EC.run_training_step_tiny(modality=modality)
    print(r, calls)
    assert len(calls) == 1                                   # the decoder's mid-block attention
    assert not r["missing"], r["missing"]
    assert r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= tol and r["grad_worst"] <= 3 * tol, r
