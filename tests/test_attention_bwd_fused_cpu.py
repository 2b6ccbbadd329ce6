"""CPU checks of the attention backward's host side: the GEMM composition backward.attention_bwd runs on tensors off
the device, with the kernels replaced by tests/cpu_emulation.py, joint pairs included; the argument checks of
b200_attention_bwd through the bindings (they return before any device work); its declaration and binding; and the
footprint cases of tests/attention_bwd_cases.py."""
import ctypes
import os
import re

import pytest
import torch

import attention_bwd_cases as ABC
import cpu_emulation
from footprint_cases import GUARD as FC_GUARD
from diffusion_e2e_ft_b200 import backward as bw
from diffusion_e2e_ft_b200 import lib as _lib
from diffusion_e2e_ft_b200 import ops

HERE = os.path.dirname(os.path.abspath(__file__))
F16 = torch.float16


@pytest.fixture
def calls(monkeypatch):
    cpu_emulation.install(monkeypatch)
    seen = []
    gemm = bw._attention_bwd_gemm
    monkeypatch.setattr(bw, "_attention_bwd_gemm", lambda *a, **k: (seen.append("gemm"), gemm(*a, **k))[1])
    return seen


def _run(B, T, Tk, heads, D, kv_segments=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    C = heads * D
    q, do = (torch.randn(B, T, C, generator=g).half() for _ in range(2))
    k, v = (torch.randn(B, Tk, C, generator=g).half() for _ in range(2))
    scale = D ** -0.5
    got = bw.attention_bwd(q, k, v, do, heads, scale, kv_segments=kv_segments)
    # fp32 autograd of the same attention (joint: image b sees the keys of its pair)
    split = lambda t: t.float().unflatten(-1, (heads, D)).transpose(1, 2)
    qr, kr, vr = (split(t).requires_grad_(True) for t in (q, k, v))
    kk, vv = kr, vr
    if kv_segments == 2:
        h = B // 2
        kk = torch.cat([torch.cat([kr[:h], kr[h:]], 2)] * 2, 0)
        vv = torch.cat([torch.cat([vr[:h], vr[h:]], 2)] * 2, 0)
    (torch.softmax(qr @ kk.transpose(-1, -2) * scale, -1) @ vv * split(do)).sum().backward()
    back = lambda t: t.transpose(1, 2).flatten(2)
    for i, (a, r) in enumerate(zip(got, (qr.grad, kr.grad, vr.grad))):
        if Tk * kv_segments == 1 and i < 2:
            assert not a.any()                           # one key: dQ = dK = 0 exactly
            continue
        r = back(r)
        assert ((a.float() - r).norm() / r.norm()).item() <= 3e-3


@pytest.mark.parametrize("Tk,kv_segments,want", [(1, 1, False), (1, 2, True), (2, 1, True), (77, 1, True), (40, 2, True),
                                                 (144, 1, True)])
def test_host_composition_off_the_device(calls, Tk, kv_segments, want):
    """One key: the exact closed form.  Otherwise tensors off the device take the per-image GEMM composition (one
    joint pair at a time), which matches fp32 autograd with the kernels restated in torch.  CUDA tensors take the
    fused kernels (tests/test_attention_bwd_fused_gpu.py)."""
    _run(2 if kv_segments == 1 else 4, 70, Tk, 2, 64, kv_segments)
    assert bool(calls) == want


def test_joint_call_needs_an_even_batch():
    with pytest.raises(AssertionError):
        bw.attention_bwd(*(torch.zeros(3, 8, 64, dtype=F16),) * 4, 1, 0.125, kv_segments=2)


# ------------------------------------------------------------------------------------------------ argument checks
def _args(**over):
    a = dict(q=16, q_bs=8 * 64, q_ls=64, k=16, k_bs=8 * 64, k_ls=64, v=16, v_bs=8 * 64, v_ls=64, do=16,
             do_bs=8 * 64, do_ls=64, lse=16, delta=16, dq=16, dq_bs=8 * 64, dq_ls=64, dk=16, dk_bs=8 * 64, dk_ls=64,
             dv=16, dv_bs=8 * 64, dv_ls=64, B=2, heads=1, head_dim=64, Lq=8, Lk=8, kv_segments=1, scale=0.125,
             stream=None)
    a.update(over)
    return [ctypes.c_void_p(x) if k_ in ("q", "k", "v", "do", "lse", "delta", "dq", "dk", "dv") else x
            for k_, x in a.items()]


@pytest.mark.parametrize("bad,msg", [(dict(head_dim=32), "head_dim=32"), (dict(head_dim=512), "head_dim=512"),
                                     (dict(q=0), "null pointer"), (dict(lse=0), "null pointer"),
                                     (dict(dv=0), "null pointer"), (dict(B=0), "bad shape"),
                                     (dict(Lq=0), "bad shape"), (dict(Lk=0), "bad shape"),
                                     (dict(heads=70000), "bad shape"), (dict(kv_segments=3), "kv_segments=3"),
                                     (dict(B=3, kv_segments=2), "kv_segments=2 B=3"),
                                     (dict(do_ls=60), "multiples of 8"), (dict(dk_bs=12), "multiples of 8"),
                                     (dict(dq=24), "16-byte aligned"), (dict(delta=18), "4-byte aligned")])
def test_bad_arguments_are_rejected_before_launch(bad, msg):
    L = _lib.load()
    rc = L.b200_attention_bwd(*_args(**bad))
    assert rc < 0
    assert msg in L.b200_last_error_string().decode()


# ------------------------------------------------------------------------------------------------ declaration
def test_declaration_agrees_with_the_binding():
    """include/b200_e2eft_attention_bwd.h declares what lib.py binds; the main header's ABI stays 17."""
    inc = os.path.join(os.path.dirname(HERE), "include")
    header = re.sub(r"/\*.*?\*/", " ", open(os.path.join(inc, "b200_e2eft_attention_bwd.h")).read(), flags=re.S)
    assert set(re.findall(r"\b(b200_\w+)\s*\(", header)) == set(_lib._SIGS_ATTENTION_BWD) == {"b200_attention_bwd"}
    decl = re.search(r"\bb200_attention_bwd\(([^)]*)\)", header)
    assert len(decl.group(1).split(",")) == len(_lib._SIGS_ATTENTION_BWD["b200_attention_bwd"][1])
    assert not set(_lib._SIGS_ATTENTION_BWD) & set(_lib.EXPORTS)
    assert _lib.load().b200_abi_version() == _lib.ABI_VERSION == 17


def test_footprint_cases_are_well_formed():
    """Every operand view inside its backing buffer; dq / dk / dv footprints exactly their views (the other columns of
    the fused d(qkv) rows outside); the compact twin holds the same values."""
    for case in ABC.attention_bwd_cases():
        for name, o in case.ops.items():
            assert int(o.mask.sum()) == o.index.numel() == torch.Size(o.shape).numel(), (case.name, name)
            assert int(o.index.max()) < o.size - FC_GUARD, (case.name, name)
            if o.values is not None:
                assert torch.equal(o.values, case.compact.ops[name].values), (case.name, name)
        q = case.ops["dq"]
        assert q.strides[1] > q.shape[2]                   # strided case: row pitch wider than the head block
