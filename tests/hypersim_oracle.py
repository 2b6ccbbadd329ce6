"""TEST INFRASTRUCTURE ONLY: a numpy restatement of Marigold's Hypersim preprocessing per frame
(script/dataset_preprocess/hypersim/hypersim_util.py tone_map and dist_2_depth, and the casts of
preprocess_hypersim.py) at any frame size, with np.power correctly rounded, plus a CPU emulation of the device step of
diffusion_e2e_ft_b200.data.preprocess_hypersim.  Never imported by the product."""
from decimal import Decimal, localcontext

import numpy as np

GAMMA = 1.0 / 2.2                     # hypersim_util.tone_map's gamma
INV_GAMMA = 1.0 / GAMMA
FOCAL = 886.81
_LD_MARGIN = np.longdouble(2.0) ** -60   # > the error of x87 powl (1 ulp = 2^-63 relative), with room


def pow_decimal(x, y):
    """x ** y for fp64 x > 0 finite and fp64 y, correctly rounded to fp64 through `decimal` (60 digits; float() of a
    Decimal rounds correctly)."""
    with localcontext() as c:
        c.prec = 60
        return float((Decimal(float(y)) * Decimal(float(x)).ln()).exp())


def pow_cr(x, y):
    """np.power(x, y) for a float64 array (or scalar) x and a float64 scalar y, correctly rounded: x87 extended
    precision powl, and `decimal` wherever that value is within 2^-60 (relative) of an fp64 rounding boundary."""
    scalar = np.ndim(x) == 0
    x = np.atleast_1d(np.asarray(x, np.float64))
    with np.errstate(all="ignore"):
        ld = np.power(x.astype(np.longdouble), np.longdouble(y))
        out = ld.astype(np.float64)
        near = (ld * (1 - _LD_MARGIN)).astype(np.float64) != (ld * (1 + _LD_MARGIN)).astype(np.float64)
    near &= np.isfinite(x) & (x > 0)
    for i in np.flatnonzero(near):
        out.flat[i] = pow_decimal(x.flat[i], y)
    return np.float64(out[0]) if scalar else out


def wrap_cast(v, bits):
    """NumPy's float64 -> uint8 / uint16 cast on x86: truncation through int32, keeping the low bits; NaN and values
    outside the int32 range give 0."""
    v = np.asarray(v, np.float64)
    with np.errstate(invalid="ignore"):
        ok = (v > -2147483649.0) & (v < 2147483648.0)
        t = np.trunc(np.where(ok, v, 0.0)).astype(np.int64)
    return (t & ((1 << bits) - 1)).astype(np.uint8 if bits == 8 else np.uint16)


def percentile90(values):
    """np.percentile(values, 90) (method 'linear', NumPy 2.3.5's _quantile), restated with a full sort."""
    s = np.sort(np.asarray(values, np.float64))       # NaN sorts last
    n = s.size
    v = (n - 1) * 0.9
    prev = -1 if v >= n - 1 else int(np.floor(v))
    a, b = (s[-1], s[-1]) if prev == -1 else (s[prev], s[prev + 1])
    gamma = np.float64(v) - np.float64(prev)
    with np.errstate(invalid="ignore"):
        diff = np.float64(b) - np.float64(a)
        r = np.float64(a) + diff * gamma
        if gamma >= 0.5:
            r = np.float64(b) - diff * (1 - gamma)
    return np.float64(np.nan) if np.isnan(s[-1]) else r


def tone_scale(rgb, valid):
    """tone_map's scale: 1 with no valid pixel, 0 below eps, else pow(0.8, inv_gamma) / p90 (NaN for a NaN p90)."""
    if not valid.any():
        return 1.0
    with np.errstate(invalid="ignore", over="ignore"):
        br = 0.3 * rgb[..., 0] + 0.59 * rgb[..., 1] + 0.11 * rgb[..., 2]
    p = percentile90(br[valid])
    return 0.0 if p < 0.0001 else pow_cr(0.8, INV_GAMMA) / p


def plane_norm(H, W, focal=FOCAL):
    """||(x, y, f)|| of dist_2_depth's float32 image plane, fp32 squares summed in order, fp32 sqrt."""
    x = (np.arange(W, dtype=np.float64) + (-0.5 * W + 0.5)).astype(np.float32)[None, :]
    y = (np.arange(H, dtype=np.float64) + (-0.5 * H + 0.5)).astype(np.float32)[:, None]
    f = np.float32(focal)
    return np.sqrt((x * x + y * y) + f * f).astype(np.float32)


def frame(rgb, dist, entity_id, focal=FOCAL):
    """One frame: radiance [H,W,3], distance [H,W], render_entity_id [H,W] -> (bgr uint8 [H,W,3], depth uint16 [H,W])
    as preprocess_hypersim.py writes them.  An entity id of 0 raises ValueError (the script's assert)."""
    entity_id = np.asarray(entity_id)
    if (entity_id == 0).any():
        raise ValueError("render_entity_id holds 0")
    rgb = np.asarray(rgb).astype(np.float64)
    dist = np.asarray(dist).astype(np.float64)
    valid = entity_id != -1
    scale = tone_scale(rgb, valid)
    with np.errstate(invalid="ignore", over="ignore"):
        p = pow_cr(np.maximum(scale * rgb, 0), GAMMA)
        u8 = wrap_cast(np.clip(p, 0, 1) * 255, 8)
        d = dist / plane_norm(*dist.shape, focal).astype(np.float64) * focal
    d[~valid] = 0
    d *= 1000.0
    return np.ascontiguousarray(u8[..., ::-1]), wrap_cast(d, 16)


def level_decimal(m):
    """The uint8 level of pow(m, gamma) for fp64 m >= 0, the power correctly rounded through `decimal`."""
    p = 0.0 if m == 0 else pow_decimal(m, GAMMA)
    return int(wrap_cast(np.clip(p, 0, 1) * 255, 8))


def boundary_args(count=None):
    """fp64 m whose pow(m, gamma) lies within a few ulp of k / 255 for every k = 1 .. 255 (the clip point at k = 255):
    m = (k / 255) ** 2.2 and its neighbours, where a fast fp64 power may land on the wrong side of a level."""
    out = []
    for k in range(1, 256):
        with localcontext() as c:
            c.prec = 60
            m = float((Decimal(k) / 255).ln().__mul__(Decimal(INV_GAMMA)).exp())
        for j in range(-3, 4):
            out.append(m + j * np.spacing(m))
    return np.array(out[:count], np.float64)


def emulated_frames_on_host(rgb, dist, entity_id, focal, dev):
    """CPU stand-in for data._hypersim_on_host (the copies to `dev`, b200_data_hypersim_frames and the copies back)."""
    eid = entity_id.numpy()
    bad = [i for i in range(eid.shape[0]) if (eid[i] == 0).any()]
    if bad:
        from diffusion_e2e_ft_b200.data import HypersimEntityIdError
        raise HypersimEntityIdError(f"hypersim_frames: render_entity_id holds 0 in frame(s) {bad}", bad)
    outs = [frame(r, d, e, focal) for r, d, e in zip(rgb.numpy(), dist.numpy(), eid)]
    return np.stack([o[0] for o in outs]), np.stack([o[1] for o in outs])
