"""Footprint cases of b200_attention_bwd (include/b200_e2eft_attention_bwd.h) in the form of tests/footprint_cases.py:
which elements of each operand the fused attention backward may read or write.  Pure index arithmetic, so the table
can be checked without a GPU (tests/test_attention_bwd_fused_cpu.py); tests/test_attention_bwd_fused_gpu.py runs the
cases through tests/test_kernel_footprint_gpu.py's harness."""
import math

import torch

import footprint_cases as FC


def attention_bwd_case(name, D, *, B=2, heads=2, Lq=70, Lk=77, kv_segments=1, compact=False):
    """b200_attention_bwd: the strided layout puts q / k / v and dq / dk / dv in column blocks of fused [B, L, 3C]
    buffers (the other columns and the batch gaps outside every footprint); lse is the true log-sum-exp of the inputs,
    so P stays a probability."""
    v = FC._Vals(name)
    C = heads * D
    ls = C if compact else 3 * C + 8
    q_bs, k_bs = (Lq * C, Lk * C) if compact else (Lq * ls + 16, (Lk + 2) * ls)
    vals = {n: v.randn((B, L_, C), FC.F16) for n, L_ in (("q", Lq), ("k", Lk), ("v", Lk), ("do", Lq))}
    scale = D ** -0.5
    qh = vals["q"].double().unflatten(-1, (heads, D)).transpose(1, 2)
    kh = vals["k"].double().unflatten(-1, (heads, D)).transpose(1, 2)
    if kv_segments == 2:
        kh = torch.cat([torch.cat([kh[:B // 2], kh[B // 2:]], 2)] * 2, 0)
    lse = torch.logsumexp(qh @ kh.transpose(-1, -2) * scale, -1) / math.log(2.0)
    ops = {n: FC.Op("in", FC.F16, (B, L_, C), (bs, ls, 1), pad=ls, values=vals[n])
           for n, L_, bs in (("q", Lq, q_bs), ("k", Lk, k_bs), ("v", Lk, k_bs), ("do", Lq, q_bs))}
    ops["lse"] = FC.Op("in", FC.F32, (B, heads, Lq), values=lse.to(FC.F32))
    ops["delta"] = FC.Op("in", FC.F32, (B, heads, Lq), values=v.randn((B, heads, Lq), FC.F32, 0.5))
    for n, L_, bs in (("dq", Lq, q_bs), ("dk", Lk, k_bs), ("dv", Lk, k_bs)):
        ops[n] = FC.Op("out", FC.F16, (B, L_, C), (bs, ls, 1), pad=ls)

    def call(L, p, s):
        a = {n: FC._v(p[n]) for n in ops}
        return L.b200_attention_bwd(a["q"], q_bs, ls, a["k"], k_bs, ls, a["v"], k_bs, ls, a["do"], q_bs, ls, a["lse"],
                                    a["delta"], a["dq"], q_bs, ls, a["dk"], k_bs, ls, a["dv"], k_bs, ls, B, heads, D, Lq,
                                    Lk, kv_segments, scale, s)
    return FC.Case(name, "b200_attention_bwd", ops, call, meta=dict(heads=heads, D=D, kv_segments=kv_segments,
                                                                   scale=scale))


def attention_bwd_cases():
    """Every head width at ragged lengths, plus a joint case; each with its compact twin."""
    c = [FC.paired(attention_bwd_case, f"attention_bwd_d{D}", D) for D in (40, 64, 80, 160)]
    c.append(FC.paired(attention_bwd_case, "attention_bwd_d80_joint", 80, B=4, Lk=70, kv_segments=2))
    return c
