"""fp64 references and per-element error bounds for the attention, softmax and normalisation kernels
(diffusion_e2e_ft_b200/csrc/attention.cu, norm.cu, backward.cu and the exp2 / row-bias epilogues of the GEMM that
backward.attention_bwd runs).  The conv / GEMM kernel has its own bound in tests/gemm_geometry.py; its `U_ACC` is reused
here.  Every function takes exactly the fp16 / fp32 values the kernel reads and returns (reference, bound), both fp64
and of the output's shape, so that a test asserts |got - ref| <= bound element by element.

Units and instruction errors
----------------------------
* U16 = 2^-11, U32 = 2^-24: unit roundoff of fp16 / fp32 round-to-nearest.  A value stored as fp16 is off by at most
  U16 |x| + SUB16, SUB16 = 2^-25 (half the fp16 subnormal spacing) covering results below the normal range 2^-14.
* U_ACC = 2^-22 (gemm_geometry.py): unit of one tensor-core fp32 accumulation step.  ASSUMPTION, not measured: see
  gemm_geometry.py.  A wgmma sum of K fp16 x fp16 products (exact in fp32) is off by <= (K + 4) U_ACC sum |a b|.
* Sums on the CUDA cores (fp32 adds in any tree) of n terms are off by <= (depth) U32 sum |terms|, depth <= n - 1.
* `ex2.approx.ftz.f32` (attention.cu:62): EX2 = 2^-22 relative (2 ulp, the figure the CUDA programming guide gives
  for exp2f).  ASSUMPTION, not measured: the PTX ISA states no tighter figure that applies to the whole argument range
  used here.  Results below 2^-126 flush to zero, which the SUB16 terms cover (the values are stored as fp16).
* `exp2f` (norm.cu softmax, the ACT_EXP2 GEMM epilogue, gemm_conv.cuh:1037): CUDA programming guide, 2 ulp full range:
  EXP2F = 2^-22 relative.
* `log2f` (attention.cu:264): 1 ulp full range: LOG2F = 2^-23 relative to the result.
* `__expf(x)` (norm.cu SiLU and softmax_groups): 2 + floor(|1.173 x|) ulp, i.e. relative (2 + 1.173 |x|) 2^-23.
* `__fdividef(x, y)` for 2^-126 <= |y| <= 2^126: 2 ulp, FDIV = 2^-22.  For |y| > 2^126 it returns 0; there the
  exact value t / (1 + e^-t) is below 2^-120 and SUB16 covers it.
* `rsqrtf`: 2 ulp, RSQRT = 2^-22.  `1.0f / x` and `sqrt` in fp64 are correctly rounded.

Attention forward (attention_kernel<D>, attention_d512_kernel)
--------------------------------------------------------------
The kernel forms S = Q K^T with wgmma (fp32, D-term sum; the d512 kernel adds two 256-term partial sums, one more fp32
add), takes c = fp32(fp32(scale) * fp32(log2 e)) (attention.cu:552), and per key tile
    m' = max(m, max_j S_j);  alpha = ex2((m - m') c);  p_j = ex2(fmaf(S_j, c, -fp32(m' c)));
    l = fmaf(l, alpha, sum p_j);  O = alpha O + fp16(p) V_tile          (fp16 P, fp32 l and O)
and finally out = fp16(O * fp32(1 / l)), lse = fmaf(m, c, log2f(l)).  With p_j the exact softmax weights of row i:
* key exponent error, log2 units: E_j = c [(D' + 4) U_ACC sum_d |q_d k_jd|  +  U32 (5 |S_j| + 9 M)], M = max_j |S_j|,
  D' = D, or 256 for the d512 kernel whose two partial sums add once more (U32 |S_j|).  The other U32 terms: the error of c (3 U32 c |S_j - m|), the rounding of m c (U32 c |m|), of fmaf (U32 c |S_j - m|) and of
  (m - m') c (2 U32 c 2M).  A common shift of all exponents cancels in O = sum p v / sum p; only differences matter.
* eps_j = ln2 E_j + EX2 is the relative error of the weight of key j.  The rescale alpha multiplies O and l alike and
  cancels.  Its effect on the output is sum_j p_j eps_j (v_j - ref) / (1 - max eps), bounded with
  |v_j - ref| <= |v_j| + |ref| by (p eps) @ |v| + (sum_j p_j eps_j) |ref|, times 1 + 2 max eps.
* fp16 P in P V against the fp32 p in l: U16 sum_j p_j |v_j|, plus SUB16 sum_j |v_j| / l over the keys whose weight,
  relative to the row maximum, is below 2^-14 (a key stored as a normal fp16 at tile time is also normal relative to the
  final maximum, as the running maximum only grows).  l = sum_j 2^{c (S_j - m)} >= 1.
* P V accumulation: (Lk + n_tiles + 4) U_ACC sum_j p_j |v_j| (one wgmma step per key, one alpha rescale per tile).
* l: fp32 sum of positive terms, relative (Lk + n_tiles + 4) U32 =: g_l, which scales every output of the row.
* 1 / l, O * (1 / l): 2 U32 |ref|; fp16 output: U16 |ref| + SUB16.
* lse (log2 units): sum_j p_j eps_j / ln2 + g_l / ln2 + LOG2F |log2 l| + U32 |lse| + 3 U32 c M (c's error on c m).

Attention backward (backward.attention_bwd)
-------------------------------------------
The forward is re-run for (O, lse) with the bounds above (bO, bL).  Then, per image and head,
    delta = rowdot(dO, O):  fp32, D products    err <= |dO| . bO + (D + 4) U32 |dO| . (|O| + bO)
    P   = fp16(exp2f(fmaf(S, c', -lse)))       c' = fp32(scale * log2 e) (one rounding), S by wgmma:
          exponent error E'_j = c (D + 4) U_ACC sum|q k_j| + U32 c |S_j| + U32 |c S_j - lse| + bL,
          eP = P (ln2 E' + EXP2F)(1 + 2(ln2 E' + EXP2F)) + U16 P + SUB16
    pre = fmaf(dO V^T, s, fp32(-s delta))      err e_pre <= s ((D + 4) U_ACC |dO| |V|^T + U32 |dP| + e_delta + U32 |delta|)
                                                            + U32 |pre|
    dS  = fp16(pre * P)                        err <= (|pre| eP + (P + eP)(e_pre + U32 |pre|))(1 + U16) + U16 |dS| + SUB16
    dQ = fp16(dS K), dK = fp16(dS^T Q), dV = fp16(P^T dO)
          err <= (e_dS @ |K| + (Tk + 4) U_ACC (|dS| + e_dS) @ |K|)(1 + U16) + U16 |dQ| + SUB16, and alike.

Softmax (norm.cu softmax_rows_*, softmax_groups; backward.cu softmax_bwd_rows)
------------------------------------------------------------------------------
softmax_rows: the maximum is exact; c = fp32(fp32(scale) fp32(log2 e)); p_j = fp16(exp2f(s_j c - m c) * fp32(1 / sum)).
  E_j = U32 c (2 |s_j| + 2 |m|) + 3 U32 c |s_j - m|;  eps_j = ln2 E_j + EXP2F;
  sum: depth ceil(cols / 256) + 5 (warp) + 8 (warps) adds, g = depth U32;
  |p - ref| <= ref (eps_j + sum_k ref_k eps_k + g + 2 U32)(1 + 2 max eps) + U16 ref + SUB16.
softmax_groups: p = fp16(__expf(x - m) * (1 / sum)), x - m rounded: eps_j = U32 |x_j - m| + (2 + 1.173 |x_j - m|) 2^-23,
  sum of S terms in sequence: g = S U32; otherwise as above.  Columns >= heads * S are exactly 0.
softmax_bwd_rows: dS = fp16(s P (dP - dot)), dot = sum P dP in fp32 (depth ceil(cols / 256) + 14):
  |dS - ref| <= s P e_dot + 4 U32 s P |dP - dot| + U16 |ref| + SUB16   (the 4th U32: scale passed as fp32).

LayerNorm (norm.cu layer_norm_kernel<T, NV>: one warp per row, lane l owns the 8-vectors l, l + 32, ...)
---------------------------------------------------------------------------------------------------------
  mean: fp32 sum of C terms, depth 8 NV + 5, then / C:  e_mean = (8 NV + 6) U32 sum|x| / C
  var = sum (x - mean')^2 / C + eps: (x - mean') rounded, squared, summed (depth 8 NV + 5) and divided:
        e_var = e_mean^2 + (8 NV + 9) U32 sum (x - mean)^2 / C  (+ the 2 e_mean |x - mean| cross term, which sums to 0
        over the row for the exact mean and is bounded by 2 e_mean sum |x - mean| / C)
  rstd = rsqrtf(var + eps):  e_rstd / rstd = e_var / (2 (var + eps)) + RSQRT
  y = fp16((x - mean') rstd g + b):  |dy| <= |g| rstd (e_mean + |x - mean| (e_rstd / rstd + 3 U32)) + U32 |y| ... then
        U16 |ref| + SUB16.

GroupNorm (norm.cu gn_stats_kernel + gn_apply_kernel; the fused path reads per-channel fp64 sums instead)
--------------------------------------------------------------------------------------------------------
  Statistics: each thread sums d = x - sh (sh its first element of the channel) and d^2 in fp32 over at most `cnt`
  pixels and converts (s1 + n sh, q + 2 sh s1 + n sh^2) to fp64.  The conv / GEMM epilogues form their per-channel
  sums the same way (gemm_conv.cuh, `chan_stats`), over at most HW stored values per thread, so cnt = HW bounds them.  An error delta in s1 moves mean by delta / N and var
  by 2 (sh - mean) delta / N; with |x - sh|, |sh - mean| <= 2 R (R = max_group |x - mean|):
        e_mean = cnt U32 2R,   e_var = cnt U32 (4 R^2 + 8 R^2) + 8 2^-53 (sum x^2 / N)   (fp64 merges)
  mean' = fp32(mean), rstd' = fp32(1 / sqrt(var + eps)):  e_rstd / rstd = e_var / (2 (var + eps)) + U32
  a = fp32(rstd' gamma), b = fp32(beta - mean' a), t = x a + b (fma):
        e_t = |a| ((|x| + |mean|)(e_rstd / rstd + 2 U32) + e_mean + 2 U32 |mean|) + U32 (|beta| + |t|) + U32 |mean a|
  SiLU: y = __fdividef(t, 1 + __expf(-t)):  e_y = 1.1 e_t + |silu(t)| ((2 + 1.173 |t|) 2^-23 + U32 + FDIV)
  output: U16 |ref| + SUB16.

GroupNorm backward (backward.cu gn_mean_rstd_kernel, gn_bwd_sums_kernel, gn_bwd_apply_kernel)
---------------------------------------------------------------------------------------------
  mean, rstd, a, b and t = x a + b as in the forward (same statistics, same e_t).
  silu'(t) = s (1 + t (1 - s)), s = 1 / (1 + __expf(-t)): |silu''| <= 0.5, so
        e_sg = 0.5 e_t + s (1 + |t|)((2 + 1.173 |t|) 2^-23 + 6 U32)      (the division and three products / adds)
  dz = dy silu'(t):  e_dz = |dy| e_sg + U32 |dz|
  xhat' = fmaf(x, rstd', -mean' rstd'):  e_xh = rstd (|x - mean| (e_rstd/rstd + U32) + e_mean (1 + e_rstd/rstd)
        + 2 U32 |mean|) + U32 |xhat|
  pass 1, per channel, fp32 sums over HW pixels (thread sums, shared and global atomics, depth <= HW + 2):
        e_S0 = sum e_dz + (HW + 2) U32 sum |dz|,  e_S1 = sum (e_dz |xhat| + |dz| e_xh) + (HW + 3) U32 sum |dz xhat|
  pass 2: A, B = (sum over the group's cg channels of gamma S0, gamma S1) * fp32(1 / (HW cg)), depth cg + 2;
        k0 = rstd gamma, k1 = rstd A, k2 = rstd B, each with the relative error of rstd plus U32;
        dx = dz k0 - k1 - xhat k2 (three roundings):
        e_dx = e_dz |k0| + |dz| e_k0 + e_k1 + e_xh |k2| + |xhat| e_k2 + 3 U32 (|dz k0| + |k1| + |xhat k2|)
  add: + U32 |dx + add|; fp32 dx is stored exactly, fp16 dx as above.  dgamma, dbeta = S1, S0 summed over the NB
  images in fp32: sum e_S + NB U32 sum |S|.

LayerNorm backward (backward.cu layer_norm_bwd_kernel)
------------------------------------------------------
  mean, rstd as in the forward.  xhat' = (x - mean') rstd':  e_xh = rstd (e_mean + |x - mean| (e_rstd/rstd + 2 U32))
        (1 + e_rstd/rstd);  t = dy gamma (one rounding, U32 |t|)
  m1 = sum t / C, m2 = sum t xhat' / C (depth 8 NV + 5, one more for the division and the product):
        e_m1 = (8 NV + 7) U32 sum |t| / C,  e_m2 = (sum |t| e_xh + (8 NV + 8) U32 sum |t xhat|) / C
  dx = rstd' (t - m1 - xhat' m2):  e_dx = rstd |inner| (e_rstd/rstd)(1 + e_rstd/rstd) + rstd (1 + e_rstd/rstd)
        (U32 |t| + e_m1 + e_xh |m2| + |xhat| e_m2 + 3 U32 (|t| + |m1| + |xhat m2|)) + U32 |dx|; add and store as above.
  dgamma = sum over rows of dy xhat', dbeta = sum dy (shared and global fp32 atomics, depth <= rows + 2):
        e_dgamma = sum |dy| e_xh + (rows + 3) U32 sum |dy xhat|,  e_dbeta = (rows + 2) U32 sum |dy|.
"""
import math

import torch

from gemm_geometry import U_ACC

U16 = 2.0 ** -11
U32 = 2.0 ** -24
SUB16 = 2.0 ** -25
F16_MIN_NORMAL = 2.0 ** -14
EX2 = 2.0 ** -22            # ex2.approx.ftz.f32, PTX ISA: 2 ulp
EXP2F = 2.0 ** -22          # exp2f, 2 ulp
LOG2F = 2.0 ** -23          # log2f, 1 ulp
FDIV = 2.0 ** -22           # __fdividef, 2 ulp
RSQRT = 2.0 ** -22          # rsqrtf, 2 ulp
SILU_LIP = 1.1              # max |silu'| = 1.0998
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634

# key-tile sizes (attention.cu AttCfg / kD5Bk) and query rows per CTA (kWG * 64)
ATT_BK = {40: 128, 64: 128, 80: 64, 160: 64, 512: 32}
ATT_BQ = {40: 192, 64: 192, 80: 192, 160: 128, 512: 64}


def _expf_rel(x):
    return (2.0 + 1.173 * x.abs()) * 2.0 ** -23


def _store(bound, ref, store):
    """Add the fp16 store of the result, |fl16(y) - y| <= U16 |y| + SUB16, unless `store` is False (the bound of the
    fp32 value before the store)."""
    return bound * (1 + U16) + U16 * ref.abs() + SUB16 if store else bound


# ------------------------------------------------------------------------------------------------ attention
def _attention_rows(q, k, v, scale, D, bk):
    """Row statistics of softmax(scale q k^T) v for q [N, r, D], k / v [N, Lk, D] (fp64): a dict with the exact
    weights p, the exponent errors E (log2 units), l, m, ref and the per-key relative weight error eps."""
    c = scale * LOG2E
    Lk = k.shape[1]
    S = q @ k.transpose(-1, -2)
    A = q.abs() @ k.abs().transpose(-1, -2)
    m = S.amax(-1, keepdim=True)
    M = S.abs().amax(-1, keepdim=True)
    e2 = torch.exp2(c * (S - m))
    l = e2.sum(-1, keepdim=True)
    p = e2 / l
    Dacc = D if D <= 256 else D // 2               # the d512 kernel: two 256-term wgmma sums and one fp32 add
    E = c * ((Dacc + 4) * U_ACC * A + U32 * (5 * S.abs() + 9 * M))
    eps = LN2 * E + EX2
    return dict(S=S, m=m, M=M, e2=e2, l=l, p=p, eps=eps, c=c, n_tiles=(Lk + bk - 1) // bk)


def _attention_chunk(qd, kd, vd, scale, bk):
    """attention_ref_bound for a chunk of query rows (fp64 [N, r, D] against all keys), also returning S and p."""
    D, Lk = qd.shape[-1], kd.shape[1]
    va = vd.abs()
    r = _attention_rows(qd, kd, vd, scale, D, bk)
    p, eps, l = r["p"], r["eps"], r["l"]
    ref = p @ vd
    aref = ref.abs()
    g = (Lk + r["n_tiles"] + 4)
    pe = p * eps
    emax = eps.amax(-1, keepdim=True)
    pv = p @ va
    sub = ((r["e2"] < F16_MIN_NORMAL * (1 + 2 * eps)).double() @ va) / l       # eps: the kernel's weight error
    bound = ((U16 + 2 * U32 + g * U32) * aref + (U16 + g * U_ACC) * pv
             + (pe @ va + pe.sum(-1, keepdim=True) * aref) * (1 + 2 * emax) + SUB16 * sub + SUB16)
    lse = (r["c"] * r["m"] + torch.log2(l)).squeeze(-1)
    lse_b = (pe.sum(-1) / LN2 + (g * U32) / LN2 + LOG2F * torch.log2(l).abs().squeeze(-1)
             + U32 * lse.abs() + 3 * U32 * r["c"] * r["M"].squeeze(-1))
    return ref, bound, lse, lse_b, r["S"], p


def attention_ref_bound(q, k, v, scale, bk, chunk_elems=1 << 24, rows=None):
    """Flash attention forward: q [N, Lq, D], k / v [N, Lk, D] (fp16 or any float; N = batch x heads with the joint
    key concatenation already applied), bk the kernel's key tile.  `rows` restricts the reference to these query rows.
    Returns (ref, bound) [N, r, D] and (lse_ref, lse_bound) [N, r] in log2 units, all fp64."""
    qd, kd, vd = q.double(), k.double(), v.double()
    if rows is not None:
        qd = qd[:, rows]
    N, Lq, D = qd.shape
    step = max(1, chunk_elems // max(1, N * kd.shape[1]))
    outs = [_attention_chunk(qd[:, i:i + step], kd, vd, scale, bk)[:4] for i in range(0, Lq, step)]
    return tuple(torch.cat([o[j] for o in outs], 1) for j in range(4))


def attention_bwd_ref_bound(q, k, v, do, scale, chunk_rows=1024):
    """backward.attention_bwd for one head: q / do [T, D], k / v [Tk, D].  Returns {name: (ref, bound)} for dq, dk, dv
    (fp64, the shapes of q, k, v).  Query rows are processed `chunk_rows` at a time; dk and dv accumulate over the
    chunks, so memory stays at a few [chunk_rows, Tk] fp64 matrices."""
    qd, kd, vd, dod = q.double(), k.double(), v.double(), do.double()
    T, D = qd.shape
    Tk = kd.shape[0]
    bk = ATT_BK[D]
    c = scale * LOG2E
    ka, va = kd.abs(), vd.abs()
    dq, e_dq = torch.empty_like(qd), torch.empty_like(qd)
    dk, e_dk1, a_dk = torch.zeros_like(kd), torch.zeros_like(kd), torch.zeros_like(kd)
    dv, e_dv1, a_dv = torch.zeros_like(vd), torch.zeros_like(vd), torch.zeros_like(vd)
    for i in range(0, T, chunk_rows):
        qc, doc = qd[i:i + chunk_rows], dod[i:i + chunk_rows]
        o, bO, lse, bL, S, P = _attention_chunk(qc[None], kd[None], vd[None], scale, bk)
        o, bO, lse, bL, S, P = o[0], bO[0], lse[0], bL[0], S[0], P[0]
        dP = doc @ vd.t()
        delta = (doc * o).sum(-1, keepdim=True)
        pre = scale * (dP - delta)
        dS = P * pre
        e_delta = (doc.abs() * bO).sum(-1, keepdim=True) \
            + (D + 4) * U32 * (doc.abs() * (o.abs() + bO)).sum(-1, keepdim=True)
        ep = LN2 * (c * (D + 4) * U_ACC * (qc.abs() @ ka.t()) + U32 * c * S.abs() + U32 * (c * S - lse[:, None]).abs()
                    + bL[:, None]) + EXP2F
        eP = P * ep * (1 + 2 * ep) + U16 * P + SUB16
        del ep, S
        e_pre = scale * ((D + 4) * U_ACC * (doc.abs() @ va.t()) + U32 * dP.abs() + e_delta + U32 * delta.abs()) \
            + U32 * pre.abs()
        e_dS = (pre.abs() * eP + (P + eP) * (e_pre + U32 * pre.abs())) * (1 + U16) + U16 * dS.abs() + SUB16
        del e_pre, dP
        adS = dS.abs() + e_dS
        dq[i:i + chunk_rows] = dS @ kd
        e_dq[i:i + chunk_rows] = e_dS @ ka + (Tk + 4) * U_ACC * (adS @ ka)
        dk += dS.t() @ qc
        e_dk1 += e_dS.t() @ qc.abs()
        a_dk += adS.t() @ qc.abs()
        dv += P.t() @ doc
        e_dv1 += eP.t() @ doc.abs()
        a_dv += (P + eP).t() @ doc.abs()
    return {"dq": (dq, e_dq * (1 + U16) + U16 * dq.abs() + SUB16),
            "dk": (dk, (e_dk1 + (T + 4) * U_ACC * a_dk) * (1 + U16) + U16 * dk.abs() + SUB16),
            "dv": (dv, (e_dv1 + (T + 4) * U_ACC * a_dv) * (1 + U16) + U16 * dv.abs() + SUB16)}


# ------------------------------------------------------------------------------------------------ softmax
def _softmax_depth(cols):
    return -(-cols // 256) + 5 + 8


def softmax_rows_ref_bound(s, scale, store=True):
    """softmax(scale s) over the last dim of fp32 s [rows, cols] -> (ref, bound) fp64."""
    sd = s.double()
    c = scale * LOG2E
    m = sd.amax(-1, keepdim=True)
    ref = torch.softmax(sd * scale, -1)
    E = U32 * c * (2 * sd.abs() + 2 * m.abs()) + 3 * U32 * c * (sd - m).abs()
    eps = LN2 * E + EXP2F
    g = _softmax_depth(sd.shape[-1]) * U32
    emax = eps.amax(-1, keepdim=True)
    bound = ref * (eps + (ref * eps).sum(-1, keepdim=True) + g + 2 * U32) * (1 + 2 * emax)
    return ref, _store(bound, ref, store)


def softmax_groups_ref_bound(logits, heads, S, store=True):
    """Per-head softmax of fp32 logits [rows, >= heads*S] (column h*S + s) -> (ref, bound) [rows, heads*S]."""
    x = logits[:, :heads * S].double().unflatten(-1, (heads, S))
    m = x.amax(-1, keepdim=True)
    ref = torch.softmax(x, -1)
    dx = (x - m).abs()
    eps = U32 * dx + (2.0 + 1.173 * dx) * 2.0 ** -23
    emax = eps.amax(-1, keepdim=True)
    bound = ref * (eps + (ref * eps).sum(-1, keepdim=True) + S * U32 + 2 * U32) * (1 + 2 * emax)
    return ref.flatten(-2), _store(bound, ref, store).flatten(-2)


def softmax_bwd_ref_bound(p, dp, scale, store=True):
    """dS = scale P (dP - sum_k P_k dP_k) from the fp16 P and fp32 dP the kernel reads ([rows, cols])."""
    pd, dd = p.double(), dp.double()
    dot = (pd * dd).sum(-1, keepdim=True)
    ref = scale * pd * (dd - dot)
    e_dot = (_softmax_depth(pd.shape[-1]) + 1) * U32 * (pd * dd).abs().sum(-1, keepdim=True)
    bound = scale * pd * e_dot + 4 * U32 * scale * pd * (dd - dot).abs()
    return ref, _store(bound, ref, store)


# ------------------------------------------------------------------------------------------------ norms
def layer_norm_ref_bound(x, gamma, beta, eps, store=True):
    """LayerNorm over the last dim of x [rows, C] (fp16 or fp32) with fp32 gamma / beta -> (ref, bound) fp64."""
    xd, g, b = x.double(), gamma.double(), beta.double()
    C = xd.shape[-1]
    NV = -(-C // 256)
    mean = xd.mean(-1, keepdim=True)
    d = xd - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    ref = d * rstd * g + b
    e_mean = (8 * NV + 6) * U32 * xd.abs().sum(-1, keepdim=True) / C
    e_var = e_mean ** 2 + 2 * e_mean * d.abs().mean(-1, keepdim=True) + (8 * NV + 9) * U32 * var
    rel_rstd = e_var / (2 * (var + eps)) + RSQRT
    e_y = g.abs() * rstd * (e_mean + d.abs() * (rel_rstd + 3 * U32)) * (1 + rel_rstd) + U32 * ref.abs()
    return ref, _store(e_y, ref, store)


def gn_pixels_per_cta(NB, HW, C, sms=132):
    """(pixels per CTA, pixel rows per pass) of the GroupNorm kernels (norm.cu gn_block / gn_chunks)."""
    V = C // 8
    rpb = max(1, 256 // V)
    target = (sms * 8 + NB - 1) // NB
    return max((HW + target - 1) // target, rpb * 4), rpb


def gn_thread_count(NB, HW, C, sms=132):
    """Most pixels one thread of gn_stats_kernel sums."""
    ppc, rpb = gn_pixels_per_cta(NB, HW, C, sms)
    return -(-ppc // rpb)


def _gn_forward(x, gamma, beta, eps, groups, cnt):
    """The GroupNorm pre-activation t = x a + b and its error e_t, with the group statistics, as [NB, HW, groups, cg]."""
    xd, g, b = x.double(), gamma.double(), beta.double()
    NB, H, W, C = xd.shape
    cg = C // groups
    xg = xd.reshape(NB, H * W, groups, cg)
    mean = xg.mean((1, 3), keepdim=True)
    dev = xg - mean
    var = (dev * dev).mean((1, 3), keepdim=True)
    R = dev.abs().amax((1, 3), keepdim=True)
    e_mean = cnt * U32 * 2 * R
    e_var = cnt * U32 * 12 * R * R + 8 * 2.0 ** -53 * (xg * xg).mean((1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    rel_rstd = e_var / (2 * (var + eps)) + U32
    gg, bb = g.view(1, 1, groups, cg), b.view(1, 1, groups, cg)
    a = rstd * gg
    t = dev * a + bb
    e_t = (a.abs() * ((xg.abs() + mean.abs()) * (rel_rstd + 2 * U32) + e_mean + 2 * U32 * mean.abs())
           + U32 * (bb.abs() + t.abs() + (mean * a).abs()))
    return dict(xg=xg, mean=mean, dev=dev, rstd=rstd, rel_rstd=rel_rstd, e_mean=e_mean, gg=gg, t=t, e_t=e_t)


def group_norm_ref_bound(x, gamma, beta, eps, groups, silu, cnt, store=True):
    """GroupNorm (+ SiLU) of the channel-concatenated x [NB, H, W, C] (fp16 or fp32 values) -> (ref, bound) fp64.
    `cnt`: most pixels one statistics thread sums in fp32 (gn_thread_count), 0 when the per-channel sums are exact
    fp64 (the fused `apply_cs` path fed with fp64 sums)."""
    f = _gn_forward(x, gamma, beta, eps, groups, cnt)
    t, e_t = f["t"], f["e_t"]
    if silu:
        ref = t * torch.sigmoid(t)
        e_y = SILU_LIP * e_t + ref.abs() * (_expf_rel(t) + U32 + FDIV)
    else:
        ref, e_y = t, e_t
    return ref.reshape(x.shape), _store(e_y, ref, store).reshape(x.shape)


def _store_out(bound, ref, out_f32, store):
    """The store of a backward result: exact for fp32 (the add, when there is one, is in `bound`), fp16 as _store."""
    return bound if out_f32 else _store(bound, ref, store)


def group_norm_bwd_ref_bound(x, dy, gamma, beta, eps, groups, silu, cnt, add=None, out_f32=True, store=True):
    """ops.group_norm_bwd over the channel-concatenated x [NB, H, W, C] with fp16 dy and optional `add` (the dx
    dtype).  Returns {"dx": (ref, bound) [NB, H, W, C], "dgamma": ..., "dbeta": ... [C]}, fp64."""
    NB, H, W, C = x.shape
    HW = H * W
    f = _gn_forward(x, gamma, beta, eps, groups, cnt)
    t, e_t, rstd, rel, gg = f["t"], f["e_t"], f["rstd"], f["rel_rstd"], f["gg"]
    cg = C // groups
    dyg = dy.double().reshape(NB, HW, groups, cg)
    xhat = f["dev"] * rstd
    e_xh = rstd * (f["dev"].abs() * (rel + U32) + f["e_mean"] * (1 + rel) + 2 * U32 * f["mean"].abs()) + U32 * xhat.abs()
    if silu:
        sg = torch.sigmoid(t)
        dsil = sg * (1 + t * (1 - sg))
        e_sg = 0.5 * e_t + sg * (1 + t.abs()) * (_expf_rel(t) + 6 * U32)
    else:
        dsil, e_sg = torch.ones_like(t), torch.zeros_like(t)
    dz = dyg * dsil
    e_dz = dyg.abs() * e_sg + U32 * dz.abs()
    # pass 1: per-channel fp32 sums over the HW pixels (thread sums, shared and global atomics: depth <= HW + 2)
    S0, S1 = dz.sum(1), (dz * xhat).sum(1)                                 # [NB, groups, cg]
    e_S0 = e_dz.sum(1) + (HW + 2) * U32 * dz.abs().sum(1)
    e_S1 = (e_dz * xhat.abs() + dz.abs() * e_xh).sum(1) + (HW + 3) * U32 * (dz * xhat).abs().sum(1)
    # pass 2: A, B = fp32 sums over the group's cg channels of gamma S, times fp32(1 / (HW cg))
    g2 = gg[0]
    A, B = (g2 * S0).sum(-1, keepdim=True) / (HW * cg), (g2 * S1).sum(-1, keepdim=True) / (HW * cg)
    e_A = ((g2.abs() * e_S0).sum(-1, keepdim=True) + (cg + 2) * U32 * (g2 * S0).abs().sum(-1, keepdim=True)) / (HW * cg)
    e_B = ((g2.abs() * e_S1).sum(-1, keepdim=True) + (cg + 2) * U32 * (g2 * S1).abs().sum(-1, keepdim=True)) / (HW * cg)
    A, B, e_A, e_B = A[:, None], B[:, None], e_A[:, None], e_B[:, None]
    k0, k1, k2 = rstd * gg, rstd * A, rstd * B
    e_k0 = k0.abs() * (rel + U32)
    e_k1 = rstd * (A.abs() * (rel + U32) + e_A)
    e_k2 = rstd * (B.abs() * (rel + U32) + e_B)
    dx = dz * k0 - k1 - xhat * k2
    e_dx = (e_dz * k0.abs() + dz.abs() * e_k0 + e_k1 + e_xh * k2.abs() + xhat.abs() * e_k2
            + 3 * U32 * ((dz * k0).abs() + k1.abs() + (xhat * k2).abs()))
    dx, e_dx = dx.reshape(x.shape), e_dx.reshape(x.shape)
    if add is not None:
        dx = dx + add.double()
        e_dx = e_dx + U32 * dx.abs()
    # dgamma / dbeta: the [NB, C] sums added over the images in fp32
    dg, db = S1.sum(0).flatten(), S0.sum(0).flatten()
    e_dg = e_S1.sum(0).flatten() + NB * U32 * S1.abs().sum(0).flatten()
    e_db = e_S0.sum(0).flatten() + NB * U32 * S0.abs().sum(0).flatten()
    return {"dx": (dx, _store_out(e_dx, dx, out_f32, store)), "dgamma": (dg, e_dg), "dbeta": (db, e_db)}


def layer_norm_bwd_ref_bound(x, dy, gamma, eps, add=None, out_f32=True, store=True):
    """layer_norm_bwd_kernel: x [rows, C] (fp16 / fp32), fp16 dy, fp32 gamma, optional `add`.  Returns
    {"dx": (ref, bound) [rows, C], "dgamma": ..., "dbeta": ... [C]}, fp64."""
    xd, dyd, g = x.double(), dy.double(), gamma.double()
    rows, C = xd.shape
    NV = -(-C // 256)
    mean = xd.mean(-1, keepdim=True)
    d = xd - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    e_mean = (8 * NV + 6) * U32 * xd.abs().sum(-1, keepdim=True) / C
    e_var = e_mean ** 2 + 2 * e_mean * d.abs().mean(-1, keepdim=True) + (8 * NV + 9) * U32 * var
    rel = e_var / (2 * (var + eps)) + RSQRT
    xhat = d * rstd
    e_xh = rstd * (e_mean + d.abs() * (rel + 2 * U32)) * (1 + rel)
    t = dyd * g
    m1, m2 = t.mean(-1, keepdim=True), (t * xhat).mean(-1, keepdim=True)
    e_m1 = (8 * NV + 7) * U32 * t.abs().sum(-1, keepdim=True) / C
    e_m2 = ((t.abs() * e_xh).sum(-1, keepdim=True) + (8 * NV + 8) * U32 * (t * xhat).abs().sum(-1, keepdim=True)) / C
    inner = t - m1 - xhat * m2
    dx = rstd * inner
    e_dx = (rstd * inner.abs() * rel * (1 + rel)
            + rstd * (1 + rel) * (U32 * t.abs() + e_m1 + e_xh * m2.abs() + xhat.abs() * e_m2
                                  + 3 * U32 * (t.abs() + m1.abs() + (xhat * m2).abs()))
            + U32 * dx.abs())
    if add is not None:
        dx = dx + add.double()
        e_dx = e_dx + U32 * dx.abs()
    dg, db = (dyd * xhat).sum(0), dyd.sum(0)
    e_dg = (dyd.abs() * e_xh).sum(0) + (rows + 3) * U32 * (dyd * xhat).abs().sum(0)
    e_db = (rows + 2) * U32 * dyd.abs().sum(0)
    return {"dx": (dx, _store_out(e_dx, dx, out_f32, store)), "dgamma": (dg, e_dg), "dbeta": (db, e_db)}


# ------------------------------------------------------------------------------------------------ checks / inputs
def bound_ratio(got, ref, bound):
    """max |got - ref| / bound (an exact element counts 0 even where its bound is 0; NaN anywhere gives inf)."""
    err = (got.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    if torch.isnan(r).any():
        return float("inf")
    return r.max().item()


def attention_inputs(B, heads, D, Lq, Lk, regime, seed=0, device="cpu", kv_segments=1):
    """q [B, Lq, C] and k, v [B, Lk, C] as head slices of fused [B, L, 3C] projection buffers whose other columns are
    non-zero, and the scale, for the input regimes of the bound tests:
      gauss    logits of std ~2
      ramp_up / ramp_down   key norms grow / shrink along the keys: the row maximum moves tile after tile
      jump     (kv_segments = 2) the second segment's keys scaled x4: the maximum moves at the segment boundary
      peaked   each query aligned with one key: one dominant weight, the rest far below the fp16 normal range
      uniform  logits of std ~0.01"""
    C = heads * D
    g = torch.Generator(device="cpu").manual_seed(seed)
    qb = torch.randn(B, Lq, 3 * C, generator=g)
    kvb = torch.randn(B, Lk, 3 * C, generator=g)
    kk = kvb[..., C:2 * C].unflatten(-1, (heads, D))
    scale = D ** -0.5
    if regime == "gauss":
        scale *= 2.0
    elif regime in ("ramp_up", "ramp_down"):
        r = torch.linspace(0.05, 6.0, Lk)
        kk *= (r if regime == "ramp_up" else r.flip(0))[None, :, None, None]
    elif regime == "jump":
        assert kv_segments == 2 and B % 2 == 0
        kk[B // 2:] *= 4.0
    elif regime == "peaked":
        j = (torch.arange(Lq) * 7919) % Lk
        qq = qb[..., :C].unflatten(-1, (heads, D))
        qq.copy_(kk[:, j] * 1.5 + 0.1 * qq)
    elif regime == "uniform":
        scale *= 0.01
    else:
        raise ValueError(regime)
    qb, kvb = qb.half().to(device), kvb.half().to(device)
    return qb[..., :C], kvb[..., C:2 * C], kvb[..., 2 * C:], scale


def split_heads(t, heads, kv_segments=1):
    """[B, L, C] -> [B * heads, L', D] fp64, with the joint key concatenation of kv_segments = 2 applied
    (batch b attends to the keys of b % (B/2) then b % (B/2) + B/2)."""
    B, L, C = t.shape
    x = t.double().unflatten(-1, (heads, C // heads)).transpose(1, 2)
    if kv_segments == 2:
        h = B // 2
        x = torch.cat([torch.cat([x[:h], x[h:]], 2)] * 2, 0)
    return x.flatten(0, 1)
