"""fp64 references and per-element error bounds for the kernels between the decoder output and the parameter update:
the task losses and their backward (csrc/loss.cu, backward.cu), the training decode_post and its backward
(elementwise.cu, backward.cu), the bias-gradient / upsample backward sums (backward.cu) and the optimizer (optim.cu).
Every function takes exactly the values the kernel reads and returns (reference, bound), fp64 and of the output's
shape, so that a test asserts |got - ref| <= bound element by element.  Where the reference is an autograd graph
(the SSI and angular losses, decode_post's clamps) the reference gradient is fp64 autograd of the reference
expression, not the kernel's closed form.

Units and instruction errors
----------------------------
* U32 = 2^-24, U64 = 2^-53: unit roundoff of fp32 / fp64 round-to-nearest; U16 / SUB16 as in numerics_bounds.py.
  The library is built without fast-math: fp32 `/` and `sqrtf` are correctly rounded, and nvcc may contract a
  product and a sum into one fma, which never rounds more often than the unfused pair, so each bound below counts
  the unfused roundings.
* `rsqrtf`: RSQRT = 2^-22 relative (2 ulp, CUDA programming guide).  `acosf`: ACOSF = 2 ulp of the result, taken
  as 2^-22 relative (CUDA programming guide, full range).  fp64 `pow`: 2 ulp (CUDA programming guide), so
  |pow - beta^step| <= 2^-51 beta^step.  ASSUMPTIONS, not measured: the guide's figures are the only ones used.
* A fp64 sum of n terms in any order is off by <= depth U64 sum |terms|, depth <= n.  It is EXACT when every term
  is an integer multiple of some q = 2^e and sum |terms| < 2^52 q: then every partial sum is representable
  (`sum_is_exact`).  The dyadic cases use that, so that their moments, fits and residuals are exactly 0 where the
  mathematics says so and the sign / clamp decisions at 0 and +-1 are checked exactly.
* An fp32 expression whose every exact intermediate is representable in fp32 (checked with fp64 error-free
  transformations, `_f32_exact_*`) is exact however nvcc contracts it.

SSI loss (loss.cu ssi_moments_kernel, ssi_l1_kernel; backward.cu ssi_bwd_*)
--------------------------------------------------------------------------
Per image, moments A = (sum p^2, sum p, n, sum p y, sum y) in fp64 over the mask.  p^2 and p y of fp32 values are
exact in fp64, so each moment is off by delta_k <= 2 n U64 sum|term_k| (kernel and reference sum in different orders;
0 when `sum_is_exact`).  det = a00 a11 - a01^2, Ns = a11 b0 - a01 b1, Nt = a00 b1 - a01 b0 to first order in delta:
    e_det = a11 d00 + 2 |a01| d01 + 4 U64 (a00 a11 + a01^2)
    e_Ns  = a11 db0 + |b1| d01 + |a01| db1 + 4 U64 (|a11 b0| + |a01 b1|),  e_Nt alike
    e_s   = (e_Ns + |s| e_det) / det (1 + 2 e_det / det) + 4 U64 |s|,   e_t alike
(0 when the moments are exact and every exact intermediate of the solve is a double, `_solve_exact`).  The kernel
rounds s, t to fp32 for the residual: e_sf = e_s + U32 |s| (0 if additionally s is an fp32 value).
Residual r = fl(fl(sf p) + tf) - y in fp32:  e_r = |p| e_sf + e_tf + U32 (2 |s p| + 2 |t| + |y|)(1 + 3 U32)
(the rounding part 0 where `_f32_exact_residual` holds).
* Forward: loss = fp32(sum |r| / N), the sum in fp64:  bound = (sum e_r + 2 N U64 sum |r|) / N + U32 |loss| + U64.
  All masks empty: NaN, like torch's mean of an empty tensor.
* Backward (ssi_bwd_grad_kernel, fp64 with the fp64 s, t; only sgn(r) uses the fp32 residual):
      g = sgn(r) s / N + (G1 (dns - s ddet) + G0 (dnt - t ddet)) / det
  G0 = sum sgn(r) / N, G1 = sum sgn(r) p / N, dns = a11 y - b1, ddet = 2 p a11 - 2 a01, dnt = 2 p b1 - b0 - a01 y.
  A pixel whose fp64 residual r64 lies within its residual band (e_r plus the reference's own |p| e_s + e_t) may take
  either sign in the kernel: its own term may move by 2 |s| / N and G0, G1 by 2 / N and 2 |p| / N.  The moment
  errors enter dns, ddet, dnt as above (delta_k times their coefficients, plus 3 U64 of each product), s and t with
  e_s, e_t, and det with e_det:
      e_g2 = (|G1| eX1 + dG1 |X1| + |G0| eX0 + dG0 |X0| + 4 U64 (|G1 X1| + |G0 X0|) + |g2| e_det) / det (1 + 2 e_det/det)
  The stored value fp32(grad_out g):  bound = grad_out (e_g1 + e_g2)(1 + U32) + U32 |ref| + 2^-149.
  With sgn(0) = 0 (torch's abs backward gives 0 at 0): a target explained exactly gives a gradient of exactly 0.

Angular loss (loss.cu angular_kernel, backward.cu angular_bwd_kernel)
--------------------------------------------------------------------
d = fp32 dot of 3 products:  e_d = 3.01 U32 sum_c |p_c y_c| (0 where `_f32_exact_dot`); the fp64 reference adds
3 U64 of the same.  acos is monotone, so the forward term is bounded by the exact interval
|acos(clamp(d +- e_d)) - acos(clamp(d))| plus ACOSF |acos|; the fp64 sum and fp32 division as for SSI.
Backward: w = 1 - d d in fp32 (the cancellation: d d rounds by U32 d^2, so w is off by U32 (d^2 + w), i.e. by the
relative U32 d^2 / (1 - d^2) near |d| = 1).  The kernel returns g = -k rsqrtf(w) for -1 < d < 1 and 0 otherwise,
k = fp32(grad_out / N).  Over the interval d +- e_d: the largest w gives the smallest |g|, the smallest positive w
(at least 2^-24 for an fp32 |d| < 1) the largest, and 0 is reachable when the interval touches |d| >= 1.  The bound is
the distance from the fp64 autograd value to that range, times |y_c|, with RSQRT, U32 for k and 2 U32 for the
products.  At |d| = 1 exactly, torch's inclusive clamp passes the gradient and acos' gives -inf / NaN; the kernel
returns 0 there, and the bound pins that exactly 0.

decode_post training modes (elementwise.cu decode_post_kernel modes 2 / 3, backward.cu decode_post_bwd_kernel)
------------------------------------------------------------------------------------------------------------
Mode 2: m = ((a + b) + c) / 3 in fp32:  e_m = U32 (1.01 |a + b| + |a + b + c|) / 3 + 1.01 U32 |m| (0 where exact);
    forward clamp(m) is 1-Lipschitz: e_m.  Backward: dout / 3 (one rounding) where -1 <= m <= 1 (torch's clamp
    backward is inclusive), 0 outside; within e_m of +-1 either is allowed.
Mode 3: u_c = x_c / (|x| + 1e-5):  |x|^2 3.01 U32, sqrtf 2.51 U32, + 1e-5f 3.52 U32 (the constant 1e-5f is itself
    off by U32 1e-5), 1 / den 4.53 U32, x_c inv 5.54 U32 relative:  e_u = 5.6 U32 |u| + 2^-149.  |u_c| < 1 exactly,
    but reaches 1 in fp32 once 1e-5 is lost against |x|; where |u| + e_u >= 1 the clamp may drop the channel.
    Backward dx_c = g_c inv - x_c k, k = (sum g_j x_j) inv^2 / |x| (k = 0 at x = 0, where torch's norm backward adds
    nothing either, so dx = dout / 1e-5):
      e_dx = |g_c inv| 5.6 U32 + |x_c| e_k + 2 U32 (|x_c k| + |dx|),  e_k = (3.01 U32 sum |g x| + |dot| 15.6 U32) inv^2/|x|
    plus, for every channel j that may be dropped, |dout_j| (delta_cj inv + |x_c x_j| inv^2 / |x|).

Masked latent MSE (loss.cu masked_latent_mse_kernel / _bwd_kernel)
-----------------------------------------------------------------
latent_mask = ~max_pool2d(~val_mask, 8, 8), exact.  Forward: d = fp32(pred) - tgt in fp64 (U64 |d|), d^2 (U64), fp64
sum of n terms, count exact:  bound = (n + 3) U64 sum d^2 / cnt + U32 |ref| + U64; empty mask: exactly 0.
Backward: fp32(fp32(2 go / cnt) fl(pred - tgt)): 3.01 U32 |ref|, then the store in pred's dtype (fp16: U16 |ref| +
SUB16).

act_bwd / geglu_bwd (backward.cu silu_grad, gelu_fwd, gelu_grad; fp16 in and out)
-------------------------------------------------------------------------------
`__expf(x)`: relative EXPF(x) = (2 + 1.173 |x|) 2^-23 (numerics_bounds.py); `erff`: 2 ulp, ERFF = 2^-22 relative
(CUDA programming guide; ASSUMPTION, not measured).  x is an exact fp16 value.
* silu'(z) = s (1 + z (1 - s)), s = 1 / (1 + __expf(-z)):  an error de / e of the exponential moves s by s (1 - s)
  de / e; with the add and the division  e_s = s (1 - s) EXPF(z) + 2 U32 s.  d silu' / ds = 1 + z (1 - 2 s), so
      e_act = |1 + z (1 - 2 s)| e_s + s (U32 |z (1 - s)| + 2 U32 |z (1 - s)| + U32 |1 + z (1 - s)|) + U32 |silu'|
* erf term: the argument x c (c = fp32(1 / sqrt 2)) is off by 2 U32 |x c|, erf' <= 2 / sqrt(pi) exp(-(x c)^2):
      e_erf = 1.13 exp(-(x c)^2) 2 U32 |x c| (1.01) + ERFF |erf|
  gelu'(x) = Phi + x phi:  e_cdf = 0.5 e_erf + U32 |Phi|;  phi = fp32(1/sqrt(2 pi)) __expf(-0.5 x x): its argument is
  off by U32 x^2, so e_phi = phi (U32 x^2 (1.01) + EXPF(x^2 / 2) + 2 U32);  e_act = e_cdf + |x| e_phi + U32 |x phi|
  + U32 |gelu'|.  gelu(g) = 0.5 g (1 + erf):  e_gelu = 0.5 |g| (e_erf + U32 |1 + erf|) + 2 U32 |gelu|.
* dx = fp16(dy act'): |dy| e_act + U32 |dy act'|, then the fp16 store; dh = fp16(dy gelu(g)) alike;
  dg = fp16(dy h gelu'(g)): |dy h| e_act + 2 U32 |dy h gelu'|, then the store.

col_sum (backward.cu col_sum_kernel), upsample_nearest_bwd
---------------------------------------------------------
fp32 sums:  bound = depth U32 (sum |x| + |out0|)(1 + depth U32), depth = the longest chain of additions a term goes
through: ceil(ceil(rows / R) / Y) thread-sequential + Y row threads + R ranks + 1 for the old value (col_sum), the
number of summed pixels + 1 (upsample).

sumsq (optim.cu sumsq_kernel)
-----------------------------
fp64 sum of the exact fp64 squares; depth = 4 per float4 + float4s per thread + the tail (3) + 5 (xor butterfly)
+ 31 (warps) + 15 (ranks) + 1:  bound = depth U64 sum x^2 (1 + depth U64) + the reference's own error (a pairwise
long-double sum, 64 2^-64 sum x^2, then U64 to double).

AdamW (optim.cu optim_prepare_kernel + adamw_state_kernel; adamw_kernel of the legacy scaled entry point)
--------------------------------------------------------------------------------------------------------
The reference is the header's update in fp64, with the fp32 hyperparameters widened to fp64:
    c = (1 / (S W)) min(1, max_norm / (sqrt(nsq) / (S W) + 1e-6))     (c = 1 / (S W) without clipping)
    m' = b1 m + (1 - b1) g c,  v' = b2 v + (1 - b2) (g c)^2,  bc_k = 1 - b_k^step (computed as -expm1(step log b_k))
    p' = p (1 - lr wd) - (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps)
Kernel roundings: c rel E_C = 7.1 U32 (+ U32 1e-6 / |g|, the fp32 1e-6); bc_k = fp32(1 - pow64): rel U32 + 2^-51
b^step / bc_k (+ the reference's 4 U64 (1 + step |log b|) b^step); 1 - b exact (Sterbenz);
    e_m = (1 - b1) |g c| (E_C + U32) + U32 (b1 |m| + (1 - b1) |g c|) + U32 |m'|
    e_v = (1 - b2) (g c)^2 (2 E_C + 4 U32) + U32 b2 v + U32 |v'|
    denom: sqrt over the interval v' +- e_v, then sqrtf U32, rsqrtf(bc2) RSQRT + E_bc2 / 2, product U32, + eps U32
    ratio = m' / denom: (e_m + |ratio| e_den) / denom (1 + 2 e_den / denom) + U32 |ratio|
    p' = p decay - step ratio:  |p| (U32 lr wd + U32 decay) + U32 |p decay| + step e_ratio
         + step |ratio| (2 U32 + E_bc1) + U32 |p'|
bc1 / bc2 in the state block are bounded by their own term; an fp32 1 - powf(b, step) is not within it (at step 2,
1 - b2^2 cancels 110 U32 away).
"""
import math
from fractions import Fraction

import numpy as np
import torch
import torch.nn.functional as F

from numerics_bounds import RSQRT, SUB16, U16, U32, bound_ratio  # noqa: F401  (bound_ratio: the tests' check)

U64 = 2.0 ** -53
ACOSF = 2.0 ** -22
POW64 = 2.0 ** -51
F32_TINY = 2.0 ** -149
W_MIN = 2.0 ** -24          # smallest positive fp32 1 - d*d for an fp32 |d| < 1 is 2^-23 - 2^-48
E_C = 7.1 * U32

F32, F64 = torch.float32, torch.float64

# launch geometry the depth-based bounds follow (loss.cu kLossThreads, backward.cu kLossBwdThreads, cluster_reduce.cuh)
LOSS_THREADS = 512
MAX_CLUSTER, MAX_SINGLE_SLOT = 8, 16


def cluster_ctas(work, per_cta, max_ctas=MAX_CLUSTER):
    """cluster_reduce.cuh cluster_ctas."""
    r = -(-work // per_cta)
    return max(1, min(max_ctas, r))


def cluster_share(n, ranks, rank):
    """cluster_reduce.cuh cluster_share: [lo, hi) of rank."""
    per = -(-n // ranks)
    lo = min(n, rank * per)
    return lo, min(n, lo + per)


# ------------------------------------------------------------------------------------------------ exactness
def _lowbit(t):
    """Exponent of the lowest set bit over the nonzero entries of fp64 t, or None if t is all zero."""
    t = t[t != 0]
    if t.numel() == 0:
        return None
    mant, ex = torch.frexp(t)
    mi = (mant.abs() * 2.0 ** 53).to(torch.int64)
    tz = torch.log2((mi & -mi).double()).round().to(torch.int64)
    return int((ex.to(torch.int64) - 53 + tz).min())


def sum_is_exact(t):
    """True when a fp64 sum of the terms t is exact in every order."""
    lb = _lowbit(t.reshape(-1))
    return lb is None or t.abs().sum().item() < 2.0 ** (52 + lb)


def _is_f32(x):
    return x.to(F32).double() == x


def _two_sum_exact(a, b):
    """(a + b in fp64, True where that sum is exact and an fp32 value) for fp32-valued fp64 tensors a, b."""
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)
    return s, (err == 0) & _is_f32(s)


def _f32_exact_residual(sf, tf, p, y):
    """True where fl(fl(sf p) + tf) - y is computed without rounding in fp32 (sf, tf, p, y fp32 values in fp64)."""
    sp = sf * p                                                    # exact in fp64
    u, ok1 = _two_sum_exact(sp, tf + torch.zeros_like(sp))
    _, ok2 = _two_sum_exact(u, -y)
    return _is_f32(sp) & ok1 & ok2


def _f32_exact_dot(p, y):
    """p, y [B, 3, HW] fp32 values in fp64: True where the 3-term fp32 dot is exact."""
    pr = p * y
    ok = _is_f32(pr).all(1)
    s1, ok1 = _two_sum_exact(pr[:, 0], pr[:, 1])
    _, ok2 = _two_sum_exact(s1, pr[:, 2])
    return ok & ok1 & ok2


def _solve_exact(a):
    """a = (a00, a01, a11, b0, b1) exact doubles: True when every exact intermediate of the 2x2 solve is a double."""
    a00, a01, a11, b0, b1 = (Fraction(float(v)) for v in a)
    det = a00 * a11 - a01 * a01
    if det <= 0:
        return det == 0 and all(Fraction(float(v)) == v for v in (a00 * a11, a01 * a01))
    vals = [a11 * b0, a01 * b1, a11 * b0 - a01 * b1, a01 * b0, a00 * b1, a00 * b1 - a01 * b0, a00 * a11, a01 * a01,
            det, (a11 * b0 - a01 * b1) / det, (a00 * b1 - a01 * b0) / det]
    return all(Fraction(float(v)) == v for v in vals)


# ------------------------------------------------------------------------------------------------ SSI
def _ssi_loss64(p, y, m):
    """oracle/pipeline.py's restatement of training/util/loss.py:17-47 on [B, HW] fp64 (the oracle casts to fp32)."""
    from oracle.pipeline import compute_scale_and_shift_masked
    s, t = compute_scale_and_shift_masked(p[:, None], y[:, None], m[:, None])
    scaled = s.view(-1, 1) * p + t.view(-1, 1)
    return F.l1_loss(scaled[m], y[m]), s, t


def _ssi_fit_bounds(p, y, m):
    """Per-image fit and its error terms (module docstring).  p, y [B, HW] fp64 of fp32 values, m bool."""
    B = p.shape[0]
    mf = m.double()
    terms = [mf * p * p, mf * p, mf, mf * p * y, mf * y]
    out = []
    for b in range(B):
        n = int(m[b].sum())
        A = [t[b].sum().item() for t in terms]
        exact = all(sum_is_exact(t[b]) for t in terms)
        d = [0.0 if exact else 2 * n * U64 * t[b].abs().sum().item() for t in terms]
        a00, a01, a11, b0, b1 = A
        det = a00 * a11 - a01 * a01
        solve_exact = exact and _solve_exact(A)
        if solve_exact:
            e_det = 0.0
        else:
            e_det = a11 * d[0] + 2 * abs(a01) * d[1] + 4 * U64 * (a00 * a11 + a01 * a01)
        if det > 0 and not solve_exact and det <= 2 * e_det:
            raise ValueError(f"image {b}: det {det:.3g} within its error {e_det:.3g}: the fit's branch is ambiguous")
        s = t = 0.0
        e_s = e_t = 0.0
        if det > 0:
            s = (a11 * b0 - a01 * b1) / det
            t = (-a01 * b0 + a00 * b1) / det
            if not solve_exact:
                e_ns = a11 * d[3] + abs(b1) * d[1] + abs(a01) * d[4] + 4 * U64 * (abs(a11 * b0) + abs(a01 * b1))
                e_nt = abs(b0) * d[1] + abs(a01) * d[3] + abs(b1) * d[0] + a00 * d[4] \
                    + 4 * U64 * (abs(a01 * b0) + abs(a00 * b1))
                grow = 1 + 2 * e_det / det
                e_s = (e_ns + abs(s) * e_det) / det * grow + 4 * U64 * abs(s)
                e_t = (e_nt + abs(t) * e_det) / det * grow + 4 * U64 * abs(t)
        sf, tf = float(np.float32(s)), float(np.float32(t))
        e_sf = e_s + abs(sf - s)
        e_tf = e_t + abs(tf - t)
        out.append(dict(n=n, A=A, d=d, det=det, e_det=e_det, s=s, t=t, e_s=e_s, e_t=e_t, sf=sf, tf=tf, e_sf=e_sf,
                        e_tf=e_tf))
    return out


def _ssi_residual_band(p, y, fit):
    """Per-pixel bound on |r_kernel - r_exact| for one image (fp64 [HW])."""
    sf, tf = fit["sf"], fit["tf"]
    rnd = U32 * (2 * abs(sf) * p.abs() + 2 * abs(tf) + y.abs()) * (1 + 3 * U32)
    if fit["e_sf"] == 0 and fit["e_tf"] == 0:
        rnd = torch.where(_f32_exact_residual(torch.tensor(sf, dtype=F64), tf, p, y), torch.zeros_like(rnd), rnd)
    return p.abs() * fit["e_sf"] + fit["e_tf"] + rnd


def ssi_loss_ref_bound(pred, tgt, mask):
    """b200_ssi_loss: pred, tgt fp32 [B, ...], mask bool [B, ...] -> (ref, bound) 0-d; ref NaN for an empty batch."""
    B = pred.shape[0]
    p, y, m = pred.reshape(B, -1).double().cpu(), tgt.reshape(B, -1).double().cpu(), mask.reshape(B, -1).bool().cpu()
    N = int(m.sum())
    if N == 0:
        return torch.tensor(float("nan"), dtype=F64), torch.tensor(0.0, dtype=F64)
    ref, s, t = _ssi_loss64(p, y, m)
    fits = _ssi_fit_bounds(p, y, m)
    e_sum = 0.0
    abs_sum = 0.0
    for b, fit in enumerate(fits):
        mb = m[b]
        if not mb.any():
            continue
        band = _ssi_residual_band(p[b][mb], y[b][mb], fit)
        r = (fit["s"] * p[b][mb] + fit["t"] - y[b][mb]).abs()
        e_sum += band.sum().item()
        abs_sum += r.sum().item()
    bound = (e_sum + 2 * N * U64 * abs_sum) / N + U32 * abs(ref.item()) + U64
    return ref.detach(), torch.tensor(bound, dtype=F64)


def ssi_bwd_ref_bound(pred, tgt, mask, grad_out):
    """b200_ssi_loss_bwd: -> (ref, bound) of pred's shape.  grad_out a python float (the fp32 upstream gradient)."""
    B = pred.shape[0]
    shape = pred.shape
    p, y, m = pred.reshape(B, -1).double().cpu(), tgt.reshape(B, -1).double().cpu(), mask.reshape(B, -1).bool().cpu()
    N = int(m.sum())
    if N == 0:
        z = torch.zeros(shape, dtype=F64)
        return z, z.clone()
    pg = p.clone().requires_grad_(True)
    loss, _, _ = _ssi_loss64(pg, y, m)
    (loss * grad_out).backward()
    ref = pg.grad.detach()
    fits = _ssi_fit_bounds(p, y, m)
    bound = torch.zeros_like(p)
    for b, fit in enumerate(fits):
        mb = m[b]
        if not mb.any():
            continue
        pb, yb = p[b][mb], y[b][mb]
        s, t, det = fit["s"], fit["t"], fit["det"]
        r64 = s * pb + t - yb
        band = _ssi_residual_band(pb, yb, fit) + pb.abs() * fit["e_s"] + fit["e_t"]
        if fit["e_s"] or fit["e_t"]:
            band = band + 3 * U64 * (abs(s) * pb.abs() + abs(t) + yb.abs())
        amb = (band > 0) & (r64.abs() <= band)                   # band 0: r64 is the kernel's exact residual
        sg = torch.sign(r64)
        e_g = amb.double() * 2 * abs(s) / N + fit["e_s"] / N
        if det > 0:
            a00, a01, a11, b0, b1 = fit["A"]
            d00, d01, _, db0, db1 = fit["d"]
            G0, G1 = sg.sum().item() / N, (sg * pb).sum().item() / N
            dG0 = 2 * amb.sum().item() / N
            dG1 = (2 * (amb.double() * pb.abs()).sum().item() + 2 * fit["n"] * U64 * pb.abs().sum().item()) / N
            dns = a11 * yb - b1
            ddet = 2 * pb * a11 - 2 * a01
            dnt = -b0 - a01 * yb + 2 * pb * b1
            X1, X0 = dns - s * ddet, dnt - t * ddet
            e_dns = db1 + 3 * U64 * (a11 * yb.abs() + abs(b1))
            e_ddet = 2 * d01 + 3 * U64 * (2 * pb.abs() * a11 + 2 * abs(a01))
            e_dnt = db0 + yb.abs() * d01 + 2 * pb.abs() * db1 + 3 * U64 * (abs(b0) + abs(a01) * yb.abs()
                                                                          + 2 * pb.abs() * abs(b1))
            eX1 = e_dns + abs(s) * e_ddet + fit["e_s"] * ddet.abs() + 2 * U64 * (dns.abs() + abs(s) * ddet.abs())
            eX0 = e_dnt + abs(t) * e_ddet + fit["e_t"] * ddet.abs() + 2 * U64 * (dnt.abs() + abs(t) * ddet.abs())
            g2 = (G1 * X1 + G0 * X0) / det
            num_e = abs(G1) * eX1 + dG1 * X1.abs() + abs(G0) * eX0 + dG0 * X0.abs() \
                + 4 * U64 * (abs(G1) * X1.abs() + abs(G0) * X0.abs())
            e_g = e_g + (num_e + g2.abs() * fit["e_det"]) / det * (1 + 2 * fit["e_det"] / det) + 2 * U64 * g2.abs()
        e_g = e_g + 4 * U64 * (abs(s) / N)
        bb = torch.zeros(p.shape[1], dtype=F64)
        bb[mb] = grad_out * e_g * (1 + U32)
        bound[b] = bb
    bound = bound + U32 * ref.abs() + F32_TINY * m.double()
    return ref.reshape(shape), bound.reshape(shape)


# ------------------------------------------------------------------------------------------------ angular
def _angular_d(p, y):
    """fp64 dot and its kernel error band e_d (0 where the fp32 dot is exact).  p, y [B, 3, HW] fp64."""
    d = (p * y).sum(1)
    e_d = 3.01 * U32 * (p * y).abs().sum(1)
    e_d = torch.where(_f32_exact_dot(p, y), torch.zeros_like(e_d), e_d + 3 * U64 * (p * y).abs().sum(1))
    return d, e_d


def angular_loss_ref_bound(pred, tgt, mask):
    """b200_angular_loss: pred, tgt fp32 [B, 3, H, W], mask bool [B, 1, H, W] -> (ref, bound) 0-d."""
    B = pred.shape[0]
    p, y = pred.reshape(B, 3, -1).double().cpu(), tgt.reshape(B, 3, -1).double().cpu()
    m = mask.reshape(B, -1).bool().cpu()
    N = int(m.sum())
    if N == 0:
        return torch.tensor(float("nan"), dtype=F64), torch.tensor(0.0, dtype=F64)
    d, e_d = _angular_d(p, y)
    a = torch.acos(d.clamp(-1, 1))
    e_a = torch.maximum(torch.acos((d - e_d).clamp(-1, 1)) - a, a - torch.acos((d + e_d).clamp(-1, 1)))
    e_a = e_a + ACOSF * a
    ref = a[m].mean()
    bound = (e_a[m].sum().item() + 2 * N * U64 * a[m].sum().item()) / N + U32 * ref.item() + U64
    return ref, torch.tensor(bound, dtype=F64)


def angular_bwd_ref_bound(pred, tgt, mask, grad_out):
    """b200_angular_loss_bwd -> (ref, bound) [B, 3, H, W].  Where fp64 autograd is not finite (|d| = 1 exactly) the
    reference is the kernel's 0 and the bound admits only what the kernel's fp32 d can reach."""
    B = pred.shape[0]
    shape = pred.shape
    p, y = pred.reshape(B, 3, -1).double().cpu(), tgt.reshape(B, 3, -1).double().cpu()
    m = mask.reshape(B, -1).bool().cpu()
    N = int(m.sum())
    if N == 0:
        z = torch.zeros(shape, dtype=F64)
        return z, z.clone()
    pg = p.clone().requires_grad_(True)
    dd = torch.clamp((pg * y).sum(1), -1.0, 1.0)
    (torch.acos(dd)[m].mean() * grad_out).backward()
    ref = pg.grad.detach()
    d, e_d = _angular_d(p, y)
    lo, hi = d - e_d, d + e_d
    x_min = torch.where((lo <= 0) & (hi >= 0), torch.zeros_like(d), torch.minimum(lo.abs(), hi.abs()))
    x_max = torch.minimum(torch.maximum(lo.abs(), hi.abs()), torch.full_like(d, 1 - 2.0 ** -24))
    can_zero = (hi >= 1) | (lo <= -1)
    can_live = x_min < 1
    w_hi = 1 - x_min ** 2 + U32 * (x_min ** 2 + 1)
    w_lo = (1 - x_max ** 2 - U32 * (x_max ** 2 + 1)).clamp(min=W_MIN)
    k = grad_out / N
    mag_hi = k * (1 + U32 + U64) * (1 + RSQRT) * (1 + 2 * U32) / torch.sqrt(w_lo)
    mag_lo = k * (1 - U32 - U64) * (1 - RSQRT) * (1 - 2 * U32) / torch.sqrt(w_hi)
    mag_lo = torch.where(can_zero, torch.zeros_like(mag_lo), mag_lo)
    mag_hi = torch.where(can_live, mag_hi, torch.zeros_like(mag_hi))
    w64 = 1 - d * d
    inside = d.abs() < 1
    ref_mag = torch.where(inside, k / torch.sqrt(torch.where(inside, w64, torch.ones_like(w64))), torch.zeros_like(d))
    ref_err = torch.where(inside, ref_mag * (4 * U64 + 2 * U64 / torch.where(inside, w64, torch.ones_like(w64))),
                          torch.zeros_like(d))
    mag_b = torch.maximum(mag_hi - ref_mag, ref_mag - mag_lo).clamp(min=0) + ref_err
    mag_b = torch.where(m, mag_b, torch.zeros_like(mag_b))
    bound = mag_b[:, None] * y.abs() + F32_TINY * m[:, None].double()
    ref = torch.where(torch.isfinite(ref), ref, torch.zeros_like(ref))
    return ref.reshape(shape), bound.reshape(shape)


# ------------------------------------------------------------------------------------------------ decode_post
def _mode2_mean(x):
    """x [NB, 3, HW] fp64 of fp32 values -> (m64, e_m)."""
    a, b, c = x[:, 0], x[:, 1], x[:, 2]
    s1, ok1 = _two_sum_exact(a, b)
    s2, ok2 = _two_sum_exact(s1, c)
    m = s2 / 3
    mf = m.to(F32).double()
    exact = ok1 & ok2 & (mf * 3 == s2)
    e_m = U32 * (1.01 * s1.abs() + s2.abs()) / 3 + 1.01 * U32 * m.abs() + 2 * U64 * m.abs()
    return m, torch.where(exact, torch.zeros_like(e_m), e_m)


def _mode3_u(x):
    nrm = torch.sqrt((x * x).sum(1, keepdim=True))
    inv = 1.0 / (nrm + 1e-5)
    u = x * inv
    return nrm, inv, u, 5.6 * U32 * u.abs() + F32_TINY


def decode_post_ref_bound(x, normals):
    """b200_decode_post modes 2 / 3 (training): x fp32 [NB, 3, H, W] -> (ref, bound) [NB, 1 or 3, H, W]."""
    NB, _, H, W = x.shape
    xd = x.reshape(NB, 3, -1).double().cpu()
    if not normals:
        m, e_m = _mode2_mean(xd)
        return m.clamp(-1, 1).reshape(NB, 1, H, W), e_m.reshape(NB, 1, H, W)
    _, _, u, e_u = _mode3_u(xd)
    return u.clamp(-1, 1).reshape(NB, 3, H, W), e_u.reshape(NB, 3, H, W)


def decode_post_bwd_ref_bound(x, dout, normals):
    """b200_decode_post_bwd: fp64 autograd of clamp(mean_c x) (mode 2) or clamp(x / (|x| + 1e-5)) (mode 3)."""
    NB, _, H, W = x.shape
    xd = x.reshape(NB, 3, -1).double().cpu()
    dd = dout.reshape(NB, 1 if not normals else 3, -1).double().cpu()
    xg = xd.clone().requires_grad_(True)
    if not normals:
        xg.mean(1, keepdim=True).clamp(-1, 1).backward(dd)
        ref = xg.grad.detach()
        m, e_m = _mode2_mean(xd)
        amb = ((e_m > 0) & ((m.abs() - 1).abs() <= e_m))[:, None]    # e_m 0: m is exactly the kernel's
        bound = U32 * (dd.abs() / 3) + amb.double() * dd.abs() / 3 + 2 * U64 * dd.abs()
        return ref.reshape(x.shape), bound.expand(NB, 3, -1).reshape(x.shape)
    (xg / (torch.norm(xg, dim=1, keepdim=True) + 1e-5)).clamp(-1, 1).backward(dd)
    ref = xg.grad.detach()
    nrm, inv, u, e_u = _mode3_u(xd)
    amb = (u.abs() + e_u >= 1)
    g = torch.where(u.abs() <= 1, dd, torch.zeros_like(dd))
    dot = (g * xd).sum(1, keepdim=True)
    safe = torch.where(nrm > 0, nrm, torch.ones_like(nrm))
    q = torch.where(nrm > 0, inv * inv / safe, torch.zeros_like(nrm))
    k = dot * q
    e_k = (3.01 * U32 * (g * xd).abs().sum(1, keepdim=True) + dot.abs() * 15.6 * U32) * q
    dx = g * inv - xd * k
    e = (g * inv).abs() * 5.6 * U32 + xd.abs() * e_k + 2 * U32 * ((xd * k).abs() + dx.abs()) \
        + 8 * U64 * ((g * inv).abs() + (xd * k).abs())
    drop = (amb.double() * dd.abs())
    e = e + drop * inv + xd.abs() * (drop * xd.abs()).sum(1, keepdim=True) * q
    return ref.reshape(x.shape), (e + F32_TINY).reshape(x.shape)


# ------------------------------------------------------------------------------------------------ latent MSE
def latent_mask_ref(val_mask):
    """~max_pool2d(~m, 8, 8) of a bool [B, H, W] (floor cropping) -> bool [B, H // 8, W // 8]."""
    inv = (~val_mask.bool()).float()[:, None]
    return ~(F.max_pool2d(inv, 8, 8)[:, 0] > 0)


def masked_latent_mse_ref_bound(pred, tgt, val_mask):
    """b200_masked_latent_mse: pred [2B, C, h, w] (fp16 / fp32), tgt fp32, val_mask bool [B, H, W]."""
    lm = latent_mask_ref(val_mask.cpu())
    p, t = pred.double().cpu(), tgt.double().cpu()
    mm = torch.cat([lm, lm])[:, None].expand_as(p)
    d2 = ((p - t) ** 2)[mm]
    n = d2.numel()
    if n == 0:
        return torch.tensor(0.0, dtype=F64), torch.tensor(0.0, dtype=F64), lm
    ref = d2.mean()
    bound = (n + 3) * U64 * d2.sum().item() / n + U32 * ref.item() + U64
    assert 2 * pred.shape[1] * int(lm.sum()) == n
    return ref, torch.tensor(bound, dtype=F64), lm


def masked_latent_mse_bwd_ref_bound(pred, tgt, latent_mask, grad_out):
    p, t = pred.double().cpu(), tgt.double().cpu()
    lm = latent_mask.bool().cpu()
    mm = torch.cat([lm, lm])[:, None].expand_as(p)
    cnt = int(mm.sum())
    if cnt == 0:
        z = torch.zeros_like(p)
        return z, z.clone()
    ref = torch.where(mm, 2.0 * grad_out * (p - t) / cnt, torch.zeros_like(p))
    b = 3.01 * U32 * ref.abs() + F32_TINY * mm.double()
    if pred.dtype == torch.float16:
        b = b * (1 + U16) + U16 * ref.abs() + SUB16 * mm.double()
    return ref, b


# ------------------------------------------------------------------------------------------------ activations
ERFF = 2.0 ** -22
INV_SQRT2_F32 = float(np.float32(0.70710678118654752))
INV_SQRT2PI_F32 = float(np.float32(0.3989422804014327))


def _expf_rel(x):
    return (2.0 + 1.173 * x.abs()) * 2.0 ** -23


def _store16(bound, ref):
    return bound * (1 + U16) + U16 * ref.abs() + SUB16


def silu_grad_ref_bound(z):
    """fp64 silu'(z) and the bound of backward.cu silu_grad (fp32 value before any product), z fp64."""
    s = torch.sigmoid(z)
    ref = s * (1 + z * (1 - s))
    e_s = s * (1 - s) * _expf_rel(z) + 2 * U32 * s
    zs = (z * (1 - s)).abs()
    e = (1 + z * (1 - 2 * s)).abs() * e_s + s * (3 * U32 * zs + U32 * (1 + z * (1 - s)).abs()) + U32 * ref.abs()
    return ref, e


def _erf_terms(x):
    xc = x * INV_SQRT2_F32
    erf = torch.erf(x / math.sqrt(2.0))
    e_erf = 1.13 * torch.exp(-xc * xc) * 2 * U32 * xc.abs() * 1.01 + ERFF * erf.abs() \
        + (x * INV_SQRT2_F32 - x / math.sqrt(2.0)).abs() * 1.13 * torch.exp(-xc * xc)
    return erf, e_erf


def gelu_grad_ref_bound(x):
    erf, e_erf = _erf_terms(x)
    cdf = 0.5 * (1 + erf)
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    ref = cdf + x * phi
    e_phi = phi * (U32 * x * x * 1.01 + _expf_rel(0.5 * x * x) + 2 * U32 + abs(INV_SQRT2PI_F32 * math.sqrt(2 * math.pi) - 1))
    e = 0.5 * e_erf + U32 * cdf + x.abs() * e_phi + U32 * (x * phi).abs() + U32 * ref.abs()
    return ref, e


def gelu_ref_bound(x):
    erf, e_erf = _erf_terms(x)
    ref = 0.5 * x * (1 + erf)
    return ref, 0.5 * x.abs() * (e_erf + U32 * (1 + erf).abs()) + 2 * U32 * ref.abs()


def act_bwd_ref_bound(x, dy, silu):
    """b200_act_bwd: fp16 x, dy -> (ref, bound) of dx = fp16(dy act'(x))."""
    xd, dd = x.double().cpu(), dy.double().cpu()
    a, e = silu_grad_ref_bound(xd) if silu else gelu_grad_ref_bound(xd)
    ref = dd * a
    return ref, _store16(dd.abs() * e + U32 * ref.abs(), ref)


def geglu_bwd_ref_bound(h, g, dy):
    """b200_geglu_bwd: fp16 h, g, dy [rows, inner] -> {dh, dg: (ref, bound)}."""
    hd, gd, dd = h.double().cpu(), g.double().cpu(), dy.double().cpu()
    ge, e_ge = gelu_ref_bound(gd)
    gp, e_gp = gelu_grad_ref_bound(gd)
    dh = dd * ge
    dg = dd * hd * gp
    return {"dh": (dh, _store16(dd.abs() * e_ge + U32 * dh.abs(), dh)),
            "dg": (dg, _store16((dd * hd).abs() * e_gp + 2 * U32 * dg.abs(), dg))}


# ------------------------------------------------------------------------------------------------ sums
def col_sum_ref_bound(x, out0):
    """b200_col_sum: out[c] = out0[c] + sum_rows x[row][c], x [rows, C] (fp16 / fp32, any row stride)."""
    rows = x.shape[0]
    R = cluster_ctas(rows, 512)
    Y = 32 if R > 1 else 8
    depth = -(-(-(-rows // R)) // Y) + Y + R + 1
    xd = x.double().cpu()
    o = out0.double().cpu()
    ref = o + xd.sum(0)
    bound = depth * U32 * (xd.abs().sum(0) + o.abs()) * (1 + depth * U32)
    return ref, bound


def upsample_nearest_bwd_ref_bound(dy, in_hw, add=None):
    """b200_upsample_nearest_bwd: fp64 autograd of F.interpolate(x, size, mode='nearest') (NHWC fp32)."""
    NB, OH, OW, C = dy.shape
    H, W = in_hw
    x = torch.zeros(NB, C, H, W, dtype=F64, requires_grad=True)
    dyd = dy.double().cpu().permute(0, 3, 1, 2)
    F.interpolate(x, size=(OH, OW), mode="nearest").backward(dyd)
    ref = x.grad.permute(0, 2, 3, 1)
    ones = torch.zeros(1, 1, H, W, dtype=F64, requires_grad=True)
    F.interpolate(ones, size=(OH, OW), mode="nearest").backward(torch.ones(1, 1, OH, OW, dtype=F64))
    cnt = ones.grad[0, 0][None, :, :, None]
    xabs = torch.zeros(NB, C, H, W, dtype=F64, requires_grad=True)
    F.interpolate(xabs, size=(OH, OW), mode="nearest").backward(dyd.abs())
    mag = xabs.grad.permute(0, 2, 3, 1)
    if add is not None:
        ad = add.double().cpu()
        ref = ref + ad
        mag = mag + ad.abs()
    depth = cnt + 1
    return ref.detach(), (depth * U32 * mag * (1 + depth * U32)).detach()


def sumsq_depth(n):
    n4 = n // 4
    R = cluster_ctas(n4, 1024 * 16, MAX_SINGLE_SLOT)
    per = -(-n4 // R)
    return 4 + -(-per // 1024) + 3 + 5 + 31 + 15 + 1


def sumsq_ref_bound(x):
    """b200_sumsq: sum x^2 of a flat fp32 buffer -> (ref, bound) 0-d.  The reference is a pairwise long-double sum."""
    xs = x.detach().cpu().reshape(-1)
    total = np.longdouble(0)
    for i in range(0, xs.numel(), 1 << 22):
        c = xs[i:i + (1 << 22)].double().numpy()
        total += np.sum(np.square(c), dtype=np.longdouble)
    ref = float(total)
    depth = sumsq_depth(xs.numel())
    bound = depth * U64 * ref * (1 + depth * U64) + 64 * 2.0 ** -64 * ref + U64 * ref
    return torch.tensor(ref, dtype=F64), torch.tensor(bound, dtype=F64)


# ------------------------------------------------------------------------------------------------ AdamW
def f32(v):
    """The fp32 value of a python float, as a python float (the kernel's hyperparameters)."""
    return float(np.float32(v))


def bias_correction_ref_bound(beta, step):
    """1 - beta^step for the fp32 beta: (ref, bound on the kernel's fp32 value)."""
    b = f32(beta)
    ref = -math.expm1(step * math.log(b))
    bp = b ** step
    ref_err = 4 * U64 * (1 + step * abs(math.log(b))) * bp
    return ref, U32 * ref + POW64 * bp + U64 + ref_err


def clip_ref(nsq, max_norm, scale=1.0, inv_world=1.0):
    """The multiplier of the gradient: 1 / (S W) times the clip coefficient (fp64 of the fp32 arguments)."""
    unscale = f32(inv_world) / f32(scale)
    if max_norm > 0:
        nrm = math.sqrt(nsq) * unscale
        return unscale * min(1.0, f32(max_norm) / (nrm + 1e-6))
    return unscale


def adamw_ref_bound(p, g, m, v, step, lr, wd, betas, eps, clip, e_clip=E_C):
    """One AdamW step per element.  p, g, m, v fp32 tensors; lr / wd python floats or per-element fp64 tensors (the
    element's group); clip the fp64 multiplier of the gradient.  -> dict name -> (ref, bound) for param, exp_avg,
    exp_avg_sq."""
    pd, gd, md, vd = (t.double().cpu() for t in (p, g, m, v))
    b1, b2, eps = f32(betas[0]), f32(betas[1]), f32(eps)
    lr = lr if torch.is_tensor(lr) else f32(lr)
    wd = wd if torch.is_tensor(wd) else f32(wd)
    bc1, e_bc1 = bias_correction_ref_bound(betas[0], step)
    bc2, e_bc2 = bias_correction_ref_bound(betas[1], step)
    r_bc1, r_bc2 = e_bc1 / bc1, e_bc2 / bc2
    gc = gd * clip
    e_c = e_clip + U32 * 1e-6
    m1 = b1 * md + (1 - b1) * gc
    v1 = b2 * vd + (1 - b2) * gc * gc
    e_m = (1 - b1) * gc.abs() * (e_c + U32) + U32 * (b1 * md.abs() + (1 - b1) * gc.abs()) + U32 * m1.abs()
    e_v = (1 - b2) * gc * gc * (2 * e_c + 4 * U32) + U32 * b2 * vd.abs() + U32 * v1.abs()
    sq = torch.sqrt(v1)
    e_sq = torch.maximum(torch.sqrt(v1 + e_v) - sq, sq - torch.sqrt((v1 - e_v).clamp(min=0)))
    rb = 1 / math.sqrt(bc2)
    den = sq * rb + eps
    e_den = e_sq * rb * (1 + U32) + sq * rb * (2 * U32 + RSQRT + r_bc2 / 2) * 1.01 + U32 * den
    ratio = m1 / den
    e_ratio = (e_m + ratio.abs() * e_den) / den * (1 + 2 * e_den / den) + U32 * ratio.abs()
    step_size = lr / bc1
    decay = 1 - lr * wd
    p1 = pd * decay - step_size * ratio
    e_p = pd.abs() * (U32 * lr * wd + U32 * decay) + U32 * (pd * decay).abs() + step_size * e_ratio \
        + step_size * ratio.abs() * (2 * U32 + r_bc1) + U32 * p1.abs() + F32_TINY
    return {"param": (p1, e_p), "exp_avg": (m1, e_m + F32_TINY), "exp_avg_sq": (v1, e_v + F32_TINY)}
