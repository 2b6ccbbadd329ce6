"""TEST INFRASTRUCTURE ONLY: a numpy restatement of depth-to-normal-translator/python/gen_vkitti_normals.py's
per-frame arithmetic (VERSION = 'd2nt_v3', utils/myApis.py get_DAG_filter / soft_min / MRF_optim, utils/apis.py
vector_normalization) with soft_min's fp32 np.power(e, -lap) pinned to the correctly rounded fp32 value, plus a CPU
emulation of the device step of diffusion_e2e_ft_b200.data.generate_vkitti_normals.  Never imported by the product."""
from decimal import Decimal, localcontext

import numpy as np
import torch

E32 = np.float32(np.e)                      # soft_min's base after NumPy 2 promotion against a float32 array
with localcontext() as _c:
    _c.prec = 60
    LN_E32 = Decimal(float(E32)).ln()       # ln(float32(e)) to 60 digits
LN_E32_F64 = float(LN_E32)
FX, FY, U0, V0 = (np.float32(v) for v in (725.0087, 725.0087, 620.5, 187))   # the script's float32 torch tensor K
_MARGIN = 2.0 ** -40                        # > the fp64 error of exp(-x * LN_E32_F64) for x <= 104, with room


def pow_e32_decimal(x):
    """float32(e) ** -x for one fp32 x >= 0, correctly rounded to fp32 through `decimal` (60 digits for the power, the
    fp32 midpoint compared exactly)."""
    with localcontext() as c:
        c.prec = 60
        v = (-Decimal(float(x)) * LN_E32).exp()
    f = np.float32(float(v))
    if Decimal(float(f)) <= v:
        lo, hi = f, np.nextafter(f, np.float32(np.inf))
    else:
        lo, hi = np.nextafter(f, np.float32(0)), f
    with localcontext() as c:
        c.prec = 400
        mid = (Decimal(float(lo)) + Decimal(float(hi))) / 2
    if v != mid:
        return hi if v > mid else lo
    return lo if int(lo.view(np.uint32)) % 2 == 0 else hi


def pow_e32_neg(x):
    """float32(e) ** -x elementwise for a float32 array x >= 0, correctly rounded to fp32: fp64 exp, and `decimal`
    wherever the fp64 value is within 2^-40 of an fp32 rounding boundary.  Subnormal results are kept."""
    x = np.asarray(x, np.float32)
    y = np.exp(-x.astype(np.float64) * LN_E32_F64)
    f = y.astype(np.float32)
    near = (y * (1 - _MARGIN)).astype(np.float32) != (y * (1 + _MARGIN)).astype(np.float32)
    for i in np.flatnonzero(near):
        f.flat[i] = pow_e32_decimal(x.flat[i])
    return f


def near_boundary_args(lo=1.0, hi=104.5, margin=2.0 ** -44):
    """Every fp32 x in [lo, hi) whose float32(e) ** -x lies within `margin` (relative) of an fp32 rounding boundary:
    the arguments where a fast fp64 evaluation must hand over to a more precise one."""
    a, b = np.float32(lo).view(np.uint32), np.float32(hi).view(np.uint32)
    found = []
    for s in range(int(a), int(b), 1 << 24):
        x = np.arange(s, min(s + (1 << 24), int(b)), dtype=np.uint32).view(np.float32)
        y = np.exp(-x.astype(np.float64) * LN_E32_F64)
        found.append(x[(y * (1 - margin)).astype(np.float32) != (y * (1 + margin)).astype(np.float32)])
    return np.concatenate(found)


def depth_m100(cm):
    """gen_vkitti_normals.py:63 then :100: float32(cm) / 100 and * 100, each rounded in fp32."""
    return (np.asarray(cm).astype(np.float32) / np.float32(100.0)) * np.float32(100)


def dag_gradients(Z):
    """grad_l, grad_r, grad_u, grad_d of get_DAG_filter: the cv2.filter2D correlations with BORDER_REFLECT_101, one
    fp32 subtraction each."""
    P = np.pad(Z, 1, mode="reflect")        # numpy's 'reflect' is BORDER_REFLECT_101
    c = P[1:-1, 1:-1]
    return c - P[1:-1, :-2], P[1:-1, 2:] - c, c - P[:-2, 1:-1], P[2:, 1:-1] - c


def mrf_laplacian(Z):
    """|cv2.filter2D(depth, lap_ker_alpha)|: the five non-zero taps summed in row-major order in fp32."""
    P = np.pad(Z, 1, mode="reflect")
    s = np.float32(0) - P[:-2, 1:-1]
    s = s - P[1:-1, :-2]
    s = s + np.float32(4) * P[1:-1, 1:-1]
    s = s - P[1:-1, 2:]
    s = s - P[2:, 1:-1]
    return np.abs(s)


def _soft_min(lap, axis, power):
    """soft_min (myApis.py:48-70): fp32 powers, zero-padded neighbours in fp64."""
    p = power(lap).astype(np.float64)
    if axis == 1:
        z = np.zeros((p.shape[0], 1))
        a, b = np.hstack([z, p[:, :-1]]), np.hstack([p[:, 1:], z])
    else:
        z = np.zeros((1, p.shape[1]))
        a, b = np.vstack([z, p[:-1, :]]), np.vstack([p[1:, :], z])
    eps = 1e-8
    return (a + eps * 0.5) / (eps + a + b), (b + eps * 0.5) / (eps + a + b)


def _threshold(la, lb):
    """get_DAG_filter's four sequential in-place updates (myApis.py:112-115), each re-evaluating its ratio."""
    eps, t = 1e-8, np.e
    la[la / (lb + eps) > t] = 1
    lb[la / (lb + eps) > t] = 0
    la[lb / (la + eps) > t] = 0
    lb[lb / (la + eps) > t] = 1


def _soft_min_maps(depth, power):
    """The DAG gradients and soft_min's four weight maps before get_DAG_filter's threshold updates."""
    gl, gr, gu, gd = dag_gradients(depth)
    return (gl, gr, gu, gd), _soft_min(np.abs(gl - gr), 1, power) + _soft_min(np.abs(gu - gd), 0, power)


def _mrf_source(depth):
    """MRF_optim's choice per pixel as source coordinates (ys, xs): argmin of the DLF-alpha laplacian over [left,
    right, up, down, self], off-image candidates +inf, first minimum on ties."""
    h, w = depth.shape
    lap = mrf_laplacian(depth).astype(np.float64)
    inf_c, inf_r = np.full((h, 1), np.inf), np.full((1, w), np.inf)
    stack = np.array((np.hstack((inf_c, lap[:, :-1])), np.hstack((lap[:, 1:], inf_c)),
                      np.vstack((inf_r, lap[:-1, :])), np.vstack((lap[1:, :], inf_r)), lap))
    best = np.argmin(stack, axis=0)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return ys + np.array([0, 0, -1, 1, 0])[best], xs + np.array([-1, 1, 0, 0, 0])[best]


def normals_frame(cm, fx=FX, fy=FY, u0=U0, v0=V0, power=pow_e32_neg):
    """One frame of the script's main loop: uint16 cm [H,W] -> uint16 [H,W,3] in the order handed to cv2.imwrite
    (z, y, x).  `power(lap)` is soft_min's float32(e) ** -lap; the default is the correctly rounded pin."""
    depth = depth_m100(cm)
    h, w = depth.shape
    fx, fy, u0, v0 = (np.float32(v) for v in (fx, fy, u0, v0))
    u_map = np.ones((h, 1)) * np.arange(1, w + 1) - u0
    v_map = np.arange(1, h + 1).reshape(h, 1) * np.ones((1, w)) - v0
    (gl, gr, gu, gd), (l1, l2, l3, l4) = _soft_min_maps(depth, power)
    _threshold(l1, l2)
    _threshold(l3, l4)
    Gu = l1 * gl + l2 * gr
    Gv = l3 * gu + l4 * gd
    n = np.stack([Gu * fx, Gv * fy, -(depth + v_map * Gv + u_map * Gu)], axis=2)
    n = n / (np.sqrt((n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1]) + n[..., 2] * n[..., 2]) + 1e-8)[..., None]
    n = n[_mrf_source(depth)]
    return ((-n + 1) * 32767.5).astype(np.uint16)[..., ::-1].copy()


def threshold_margin(cm):
    """Per output pixel, min |r / e - 1| over the ratios l1 / (l2 + eps), l2 / (l1 + eps) and their vertical pair
    that get_DAG_filter compares with e, at the pixel whose normal the MRF step copies there.  Where it is about
    1e-7 or less, one ulp of a power can flip a comparison and move the whole normal."""
    depth = depth_m100(cm)
    _, (l1, l2, l3, l4) = _soft_min_maps(depth, pow_e32_neg)
    eps = 1e-8
    m = np.min([np.abs(a / (b + eps) / np.e - 1) for a, b in ((l1, l2), (l2, l1), (l3, l4), (l4, l3))], axis=0)
    return m[_mrf_source(depth)]


def normals(cm, **kw):
    """normals_frame over a uint16 [B,H,W] batch (numpy or torch) -> uint16 [B,H,W,3] numpy."""
    cm = cm.numpy() if isinstance(cm, torch.Tensor) else np.asarray(cm)
    return np.stack([normals_frame(c, **kw) for c in cm])


def emulated_normals_on_host(depth, dev):
    """CPU stand-in for data._normals_on_host (the copy to `dev`, b200_data_vkitti_normals and the copy back)."""
    assert depth.dtype == torch.uint16 and depth.dim() == 3
    return normals(depth)
