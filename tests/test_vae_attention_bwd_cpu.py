"""CPU tests of the VAE mid-block attention in training on the d=512 flash path: which path the differentiable forward
takes, what the fused path saves, its data gradient against fp32 autograd of oracle/vae.py with the kernels restated
in torch (this file and tests/cpu_emulation.py), the argument checks of the new entry points (they return before any
device work), their declaration and binding, and the footprint cases of tests/vae_attention_bwd_cases.py."""
import ctypes
import math
import os
import re

import pytest
import torch

import cpu_emulation
import vae_attention_bwd_cases as VC
from footprint_cases import GUARD as FC_GUARD
from diffusion_e2e_ft_b200 import autograd_blocks as ab
from diffusion_e2e_ft_b200 import lib as _lib
from diffusion_e2e_ft_b200 import ops
from diffusion_e2e_ft_b200 import vae as vae_mod

HERE = os.path.dirname(os.path.abspath(__file__))
F16, F32 = torch.float16, torch.float32


# ------------------------------------------------------------------------------------------------ kernel emulation
def _check_view(t, C=512):
    """What the C entry points check of an fp16 operand."""
    assert t.dtype == F16 and t.shape[-1] == C and t.stride(-1) == 1
    assert t.stride(1) % 8 == 0 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0


def attention_d512(q, k, v, scale, out=None, want_lse=False):
    for t in (q, k, v):
        _check_view(t)
    s = q.float() @ k.float().transpose(1, 2) * scale
    o = (torch.softmax(s, -1) @ v.float()).half()
    if out is not None:
        out.copy_(o)
        o = out
    return (o, s.logsumexp(-1) / math.log(2.0)) if want_lse else o


def rowdot_d512(a, c):
    _check_view(a)
    _check_view(c)
    return (a.float() * c.float()).sum(-1)


def attention_d512_bwd(q, k, v, do, lse, delta, dq, dk, dv, scale):
    """The rounding of csrc/attention_d512_bwd.cu: P = fp16(exp2(fmaf(S, c, -lse))), dS = fp16(fmaf(dP, s, -s delta) P),
    fp32 sums, fp16 outputs."""
    for t in (q, k, v, do, dq, dk, dv):
        _check_view(t)
    assert lse.dtype == F32 and delta.dtype == F32 and lse.shape == delta.shape == q.shape[:2]
    c = torch.tensor(scale * 1.4426950408889634, dtype=F32)
    s = q.float() @ k.float().transpose(1, 2)
    p = torch.exp2(s * c - lse[..., None]).half().float()
    dp = do.float() @ v.float().transpose(1, 2)
    ds = ((dp * scale - scale * delta[..., None]) * p).half().float()
    dq.copy_((ds @ k.float()).half())
    dk.copy_((ds.transpose(1, 2) @ q.float()).half())
    dv.copy_((p.transpose(1, 2) @ do.float()).half())
    return dq, dk, dv


@pytest.fixture
def emulated(monkeypatch):
    """The kernels restated in torch; records which d=512 ops run."""
    cpu_emulation.install(monkeypatch)
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)
    seen = []
    for fn in (attention_d512, rowdot_d512, attention_d512_bwd):
        monkeypatch.setattr(ops, fn.__name__, lambda *a, _f=fn, **k: (seen.append(_f.__name__), _f(*a, **k))[1])
    softmax = ops.softmax_rows
    monkeypatch.setattr(ops, "softmax_rows", lambda *a, **k: (seen.append("softmax_rows"), softmax(*a, **k))[1])
    return seen


def _block(ch=512, seed=0):
    from diffusion_e2e_ft_b200.vae import VAEAttention
    torch.manual_seed(seed)
    att = VAEAttention(ch, 32).eval().requires_grad_(False)
    with torch.no_grad():
        for p in att.parameters():
            p.normal_(0, 0.05)
        att.group_norm.weight.add_(1.0)
    return att


# ------------------------------------------------------------------------------------------------ path selection
@pytest.mark.parametrize("ch,memory_efficient,limit,want", [
    (512, False, None, "unfused"),                 # the default
    (512, True, None, "fused"),                    # enable_xformers_memory_efficient_attention
    (512, False, 30 * 32, "fused"),                # one image's scores past the unfused path's index limit
    (128, True, None, "unfused"),                  # no flash kernel for other widths
    (128, False, 30 * 32, "unfused"),
])
def test_training_takes_the_inference_path(emulated, monkeypatch, ch, memory_efficient, limit, want):
    """The differentiable forward asks vae.use_fused_attention, as inference does, and its backward follows."""
    if limit is not None:
        monkeypatch.setattr(vae_mod, "UNFUSED_MAX_SCORES", limit)      # 5 x 6 = 30 tokens, Lp = 32
    att = _block(ch)
    att.memory_efficient = memory_efficient
    x = torch.randn(2, 5, 6, ch, requires_grad=True)
    out = ab.vae_attention(att, x)
    fwd = list(emulated)
    out.backward(torch.randn_like(out))
    bwd = emulated[len(fwd):]
    if want == "fused":
        assert fwd == ["attention_d512"] and bwd == ["rowdot_d512", "attention_d512_bwd"]
    else:
        assert fwd == ["softmax_rows"] and bwd == []
    assert x.grad is not None and torch.isfinite(x.grad).all()


def test_fused_training_path_saves_no_score_matrix(emulated):
    """Fused: x, GroupNorm mean / rstd, hn, qkv, O and lse, all O(L); the unfused path saves P [B, L, Lp]."""
    B, H, W, C = 2, 6, 5, 512
    L = H * W
    att = _block()
    for me, scores in ((True, False), (False, True)):
        att.memory_efficient = me
        out = ab.vae_attention(att, torch.randn(B, H, W, C, requires_grad=True))
        saved = [t for t in out.grad_fn.saved if torch.is_tensor(t)]
        has_scores = any(t.dim() >= 2 and tuple(t.shape[-2:]) == (L, (L + 7) // 8 * 8) for t in saved)
        assert has_scores == scores
        if me:
            assert len(saved) == 6 and max(t.numel() for t in saved) == B * L * 3 * C      # qkv is the largest
            lse = saved[-1]
            assert lse.dtype == F32 and tuple(lse.shape) == (B, L)


def _oracle_dx(att, x, dout):
    """fp32 autograd through oracle/vae.py's VAEAttention (NCHW) with the same weights."""
    from oracle.vae import VAEAttention as Ref
    ref = Ref(att.ch, att.groups, att.eps)
    ref.load_state_dict(att.state_dict())
    xr = x.detach().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ref(xr).backward(dout.permute(0, 3, 1, 2))
    return xr.grad.permute(0, 2, 3, 1)


@pytest.mark.parametrize("hw", [(8, 8), (5, 7), (1, 1)])
def test_fused_dx_matches_oracle_autograd(emulated, hw):
    """d/dx of the block on the fused path (out-projection, delta, the d=512 backward, the QKV projection, GroupNorm
    backward) against fp32 autograd; the unfused path for scale."""
    att = _block()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, *hw, 512, generator=g)
    dout = torch.randn(2, *hw, 512, generator=g)
    want = _oracle_dx(att, x, dout)
    errs = {}
    for me in (True, False):
        att.memory_efficient = me
        xe = x.clone().requires_grad_(True)
        ab.vae_attention(att, xe).backward(dout)
        errs[me] = ((xe.grad - want).norm() / want.norm()).item()
    assert emulated.count("attention_d512_bwd") == 1
    assert errs[True] <= 3e-3 and errs[False] <= 3e-3, errs


def test_fused_training_forward_equals_inference_forward(emulated):
    """With memory-efficient attention on, the differentiable forward runs forward_fused: the same bits."""
    att = _block()
    att.memory_efficient = True
    x = torch.randn(2, 6, 7, 512)
    with torch.no_grad():
        want = att.run(x)
    got = ab.vae_attention(att, x.clone().requires_grad_(True))
    assert torch.equal(got.detach(), want)


# ------------------------------------------------------------------------------------------------ argument checks
def _bwd_args(**over):
    a = dict(q=16, q_bs=64 * 1536, q_ls=1536, k=16, k_bs=64 * 1536, k_ls=1536, v=16, v_bs=64 * 1536, v_ls=1536,
             do=16, do_bs=64 * 512, do_ls=512, lse=16, delta=16, dq=16, dq_bs=64 * 1536, dq_ls=1536, dk=16,
             dk_bs=64 * 1536, dk_ls=1536, dv=16, dv_bs=64 * 1536, dv_ls=1536, B=2, Lq=64, Lk=64, scale=0.044,
             stream=None)
    a.update(over)
    return [ctypes.c_void_p(x) if k_ in ("q", "k", "v", "do", "lse", "delta", "dq", "dk", "dv") else x
            for k_, x in a.items()]


@pytest.mark.parametrize("bad,msg", [(dict(q=0), "null pointer"), (dict(do=0), "null pointer"),
                                     (dict(lse=0), "null pointer"), (dict(delta=0), "null pointer"),
                                     (dict(dk=0), "null pointer"), (dict(B=0), "bad shape"),
                                     (dict(B=65536), "bad shape"), (dict(Lq=0), "bad shape"),
                                     (dict(Lk=-1), "bad shape"), (dict(do_ls=516), "multiples of 8"),
                                     (dict(dv_ls=504), "row strides >= 512"), (dict(k_bs=-8), "batch strides >= 0"),
                                     (dict(dq=24), "16-byte aligned"), (dict(v=40), "16-byte aligned"),
                                     (dict(delta=18), "4-byte aligned"), (dict(lse=2), "4-byte aligned")])
def test_backward_rejects_bad_arguments_before_launch(bad, msg):
    L = _lib.load()
    assert L.b200_attention_d512_bwd(*_bwd_args(**bad)) < 0
    assert msg in L.b200_last_error_string().decode()


@pytest.mark.parametrize("bad,msg", [(dict(a=0), "null pointer"), (dict(out=0), "null pointer"),
                                     (dict(B=0), "bad shape"), (dict(L=0), "bad shape"),
                                     (dict(a_ls=1540), "multiples of 8"), (dict(c_ls=256), "row strides >= 512"),
                                     (dict(c=8), "16-byte aligned"), (dict(out=6), "4-byte aligned")])
def test_rowdot_rejects_bad_arguments_before_launch(bad, msg):
    a = dict(a=16, a_bs=8 * 1536, a_ls=1536, c=16, c_bs=8 * 512, c_ls=512, B=2, L=8, out=16, stream=None)
    a.update(bad)
    args = [ctypes.c_void_p(x) if k_ in ("a", "c", "out") else x for k_, x in a.items()]
    L = _lib.load()
    assert L.b200_rowdot_d512(*args) < 0
    assert msg in L.b200_last_error_string().decode()


def _lse_call(L, lse=16, **over):
    a = dict(q=16, q_ls=1536, k=16, v=16, out=16, o_ls=512, B=1, Lq=64, Lk=64)
    a.update(over)
    return L.b200_attention_d512_lse(a["q"], a["q_ls"] * a["Lq"], a["q_ls"], a["k"], 1536 * a["Lk"], 1536, a["v"],
                                     1536 * a["Lk"], 1536, a["out"], a["o_ls"] * a["Lq"], a["o_ls"], a["B"], a["Lq"],
                                     a["Lk"], 0.044, lse, None)


def test_forward_with_lse_rejects_bad_arguments_before_launch():
    """The checks of b200_attention_d512, and lse's alignment."""
    L = _lib.load()
    for kw, msg in ((dict(q=None), b"null pointer"), (dict(out=None), b"null pointer"), (dict(Lq=0), b"bad shape"),
                    (dict(B=0), b"bad shape"), (dict(q_ls=1540), b"multiples of 8"), (dict(o_ls=504), b">= 512"),
                    (dict(out=24), b"16-byte aligned"), (dict(lse=18), b"lse must be 4-byte aligned")):
        assert _lse_call(L, **kw) < 0 and msg in L.b200_last_error_string(), kw


# ------------------------------------------------------------------------------------------------ declaration
def test_declaration_agrees_with_the_binding():
    """include/b200_e2eft_vae_attention.h declares what lib.py binds; the main header, lib.EXPORTS, the attention
    backward's table and the ABI version (17) stay as they were."""
    inc = os.path.join(os.path.dirname(HERE), "include")
    strip = lambda f: re.sub(r"/\*.*?\*/", " ", open(os.path.join(inc, f)).read(), flags=re.S)    # noqa: E731
    header = strip("b200_e2eft_vae_attention.h")
    names = set(re.findall(r"\b(b200_\w+)\s*\(", header))
    assert names == set(_lib._SIGS_VAE_ATTENTION) == {"b200_attention_d512_lse", "b200_rowdot_d512",
                                                      "b200_attention_d512_bwd"}
    for name in names:
        decl = re.search(rf"\b{name}\(([^)]*)\)", header)
        assert len(decl.group(1).split(",")) == len(_lib._SIGS_VAE_ATTENTION[name][1]), name
    assert not names & set(_lib.EXPORTS) and not names & set(_lib._SIGS_ATTENTION_BWD)
    assert not names & set(re.findall(r"\b(b200_\w+)\s*\(", strip("b200_e2eft.h")))
    assert set(_lib._SIGS_ATTENTION_BWD) == {"b200_attention_bwd"}
    assert _lib.load().b200_abi_version() == _lib.ABI_VERSION == 17


def test_d512_forward_signature_is_unchanged():
    """b200_attention_d512 keeps its binding; the LSE entry takes one more pointer before the stream."""
    old = _lib._SIGS["b200_attention_d512"][1]
    new = _lib._SIGS_VAE_ATTENTION["b200_attention_d512_lse"][1]
    assert new[:-2] == old[:-1] and len(new) == len(old) + 1


def test_footprint_cases_are_well_formed():
    """Every operand view inside its backing buffer; the compact twin holds the same input values; dq / dk / dv of
    the strided cases are column blocks of wider rows."""
    cases = VC.vae_attention_bwd_cases()
    assert {c.entry for c in cases} == set(_lib._SIGS_VAE_ATTENTION)
    for case in cases:
        for name, o in case.ops.items():
            assert int(o.mask.sum()) == o.index.numel() == torch.Size(o.shape).numel(), (case.name, name)
            assert int(o.index.max()) < o.size - FC_GUARD, (case.name, name)
            if o.values is not None:
                assert torch.equal(o.values, case.compact.ops[name].values), (case.name, name)
        if case.entry == "b200_attention_d512_bwd":
            assert case.ops["dq"].strides[1] > 512 and case.compact.ops["dq"].strides[1] == 512
