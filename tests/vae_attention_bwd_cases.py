"""Footprint cases of the d=512 training entry points (include/b200_e2eft_vae_attention.h) in the form of
tests/footprint_cases.py: which elements of each operand b200_attention_d512_lse, b200_rowdot_d512 and
b200_attention_d512_bwd may read or write.  Pure index arithmetic, so the table can be checked without a GPU
(tests/test_vae_attention_bwd_cpu.py); tests/test_vae_attention_bwd_gpu.py runs the cases through
tests/test_kernel_footprint_gpu.py's harness."""
import math

import footprint_cases as FC

D = 512
QKV = 3 * D + 8                  # strided layout: column blocks of fused [B, L, 1536] rows, padded by 8 elements


def _qkv_ops(v, B, Lq, Lk, compact, names=("q", "k", "v"), role="in"):
    """q / k / v (or dq / dk / dv) as column blocks of one fused buffer per length, batch gaps between images."""
    ls = D if compact else QKV
    q_bs, k_bs = (Lq * D, Lk * D) if compact else (Lq * ls + 16, (Lk + 2) * ls)
    ops, geo = {}, {}
    for n, L_, bs, col in ((names[0], Lq, q_bs, 0), (names[1], Lk, k_bs, D), (names[2], Lk, k_bs, 2 * D)):
        vals = v.randn((B, L_, D), FC.F16, 0.3 if n in ("q", "k") else 1.0) if role == "in" else None
        ops[n] = FC.Op(role, FC.F16, (B, L_, D), (bs, ls, 1), offset=0 if compact else col, pad=ls, values=vals)
        geo[n] = (bs, ls)
    return ops, geo


def attention_d512_lse_case(name, B=2, Lq=70, Lk=77, compact=False):
    """b200_attention_d512_lse: q / k / v in place in fused QKV rows, o and lse [B, Lq] written."""
    v = FC._Vals(name)
    ops, geo = _qkv_ops(v, B, Lq, Lk, compact)
    o_ls = D if compact else D + 8
    o_bs = Lq * o_ls if compact else Lq * o_ls + 8
    ops["o"] = FC.Op("out", FC.F16, (B, Lq, D), (o_bs, o_ls, 1), pad=o_ls)
    ops["lse"] = FC.Op("out", FC.F32, (B, Lq))

    def call(L, p, s):
        a = {n: FC._v(p[n]) for n in ops}
        return L.b200_attention_d512_lse(a["q"], *geo["q"], a["k"], *geo["k"], a["v"], *geo["v"], a["o"], o_bs, o_ls,
                                         B, Lq, Lk, D ** -0.5, a["lse"], s)
    return FC.Case(name, "b200_attention_d512_lse", ops, call, meta=dict(heads=1, D=D, scale=D ** -0.5))


def rowdot_d512_case(name, B=2, L=37, compact=False):
    """b200_rowdot_d512: a is a column block of fused rows, c has padded rows."""
    v = FC._Vals(name)
    a_ls, c_ls = (D, D) if compact else (QKV, D + 8)
    a_bs, c_bs = (L * D, L * D) if compact else (L * a_ls + 16, L * c_ls + 8)
    ops = {"a": FC.Op("in", FC.F16, (B, L, D), (a_bs, a_ls, 1), offset=0 if compact else D, pad=a_ls,
                      values=v.randn((B, L, D), FC.F16)),
           "c": FC.Op("in", FC.F16, (B, L, D), (c_bs, c_ls, 1), pad=c_ls, values=v.randn((B, L, D), FC.F16)),
           "out": FC.Op("out", FC.F32, (B, L))}

    def call(L_, p, s):
        return L_.b200_rowdot_d512(FC._v(p["a"]), a_bs, a_ls, FC._v(p["c"]), c_bs, c_ls, B, L, FC._v(p["out"]), s)
    return FC.Case(name, "b200_rowdot_d512", ops, call, meta=dict(D=D))


def attention_d512_bwd_case(name, B=2, Lq=70, Lk=77, compact=False):
    """b200_attention_d512_bwd: q / k / v in fused QKV rows and dq / dk / dv in fused d(QKV) rows (the other columns
    and the batch gaps outside every footprint); lse is the true log-sum-exp of the inputs, so P stays a
    probability."""
    v = FC._Vals(name)
    ops, geo = _qkv_ops(v, B, Lq, Lk, compact)
    dops, dgeo = _qkv_ops(v, B, Lq, Lk, compact, names=("dq", "dk", "dv"), role="out")
    do_ls = D if compact else D + 8
    do_bs = Lq * do_ls if compact else Lq * do_ls + 24
    ops["do"] = FC.Op("in", FC.F16, (B, Lq, D), (do_bs, do_ls, 1), pad=do_ls, values=v.randn((B, Lq, D), FC.F16))
    q, k = ops["q"].values.double(), ops["k"].values.double()
    lse = (q @ k.transpose(1, 2) * D ** -0.5).logsumexp(-1) / math.log(2.0)
    ops["lse"] = FC.Op("in", FC.F32, (B, Lq), values=lse.to(FC.F32))
    ops["delta"] = FC.Op("in", FC.F32, (B, Lq), values=v.randn((B, Lq), FC.F32, 0.5))
    ops.update(dops)

    def call(L, p, s):
        a = {n: FC._v(p[n]) for n in ops}
        return L.b200_attention_d512_bwd(a["q"], *geo["q"], a["k"], *geo["k"], a["v"], *geo["v"], a["do"], do_bs,
                                         do_ls, a["lse"], a["delta"], a["dq"], *dgeo["dq"], a["dk"], *dgeo["dk"],
                                         a["dv"], *dgeo["dv"], B, Lq, Lk, D ** -0.5, s)
    return FC.Case(name, "b200_attention_d512_bwd", ops, call, meta=dict(heads=1, D=D, scale=D ** -0.5))


def vae_attention_bwd_cases():
    """Ragged lengths around the 16 / 32 / 64-row tiles, a single key and a single query; each with its compact
    twin."""
    return [FC.paired(attention_d512_lse_case, "attention_d512_lse"),
            FC.paired(attention_d512_lse_case, "attention_d512_lse_lk1", B=1, Lk=1),
            FC.paired(rowdot_d512_case, "rowdot_d512"),
            FC.paired(attention_d512_bwd_case, "attention_d512_bwd"),
            FC.paired(attention_d512_bwd_case, "attention_d512_bwd_lq1", B=1, Lq=1, Lk=33),
            FC.paired(attention_d512_bwd_case, "attention_d512_bwd_lk1", B=3, Lq=65, Lk=1)]
