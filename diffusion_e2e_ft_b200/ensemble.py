"""Test-time ensembling and the pipelines' pre/post-processing on the device (SURVEY.md §8 a11, f2).

    ensemble_normals   <- Marigold/marigold/marigold_pipeline.py:59-71 == GeoWizard/geowizard/utils/normal_ensemble.py:6-22
    ensemble_depths    <- Marigold/marigold/util/ensemble.py:40-132
    resize_bilinear_aa / normalise_rgb / minmax_normalise <- marigold_pipeline.py:237-247,300-321
    resize_bicubic_aa / resize_nearest_exact <- the other two resample_method choices (:219,237-242,315-321)
    colorize_depth / colorize_normals <- marigold_pipeline.py:327-343, geowizard_pipeline.py:211-219

Signatures, argument meaning and return values are the reference's.  The arithmetic runs in libb200_e2eft.so
(csrc/postproc.cu); torch only allocates.  `ensemble_depths` keeps the reference's optimiser — scipy's BFGS driven
from the host with a float32 parameter vector, `maxiter` 2 — and evaluates its objective (pairwise RMS distance +
near/far regulariser of the median / mean map) with one kernel per call, reading back three numbers exactly where
the reference does `err.detach().cpu().numpy()`.
"""
import ctypes

import numpy as np
import torch

from . import lib as _lib
from .ops import _ck, _need_cuda, _p, _stream

F32 = torch.float32
MAX_ENSEMBLE = 32


def ensemble_normals_with_index(input_images: torch.Tensor):
    """[E,3,H,W] (any float dtype, CUDA) -> (normalised prediction [3,H,W] of the selected member, index tensor).
    The index is a 0-d int32 device tensor (no host sync)."""
    _need_cuda(input_images)
    E, d, H, W = input_images.shape
    assert d == 3
    if E > MAX_ENSEMBLE:
        raise ValueError(f"ensemble_size {E} > {MAX_ENSEMBLE} supported by the device kernel")
    x = input_images.detach().to(F32).contiguous()
    out = torch.empty((3, H, W), dtype=F32, device=x.device)
    err = torch.empty(E, dtype=torch.float64, device=x.device)
    idx = torch.empty((), dtype=torch.int32, device=x.device)
    _ck(_lib.load().b200_ensemble_normals(_p(x), E, H * W, _p(err), _p(out), _p(idx), _stream()), "b200_ensemble_normals")
    return out.to(input_images.dtype), idx


def ensemble_normals(input_images: torch.Tensor):
    """Reference signature: returns (normal_preds[normal_idx], None)."""
    pred, _ = ensemble_normals_with_index(input_images)
    return pred, None


def minmax_rows(x2d: torch.Tensor):
    """[rows, cols] fp32 -> [rows, 2] (min, max)."""
    _need_cuda(x2d)
    assert x2d.dtype == F32 and x2d.is_contiguous() and x2d.dim() == 2
    rows, cols = x2d.shape
    ws = torch.empty(2 * rows, dtype=torch.int32, device=x2d.device)
    out = torch.empty((rows, 2), dtype=F32, device=x2d.device)
    _ck(_lib.load().b200_minmax_rows(_p(x2d), rows, cols, _p(ws), _p(out), _stream()), "b200_minmax_rows")
    return out


def minmax_normalise_(x: torch.Tensor):
    """In place x = (x - min) / (max - min) (marigold_pipeline.py:305-312); returns (x, [min, max] device tensor).
    max == min gives 0/0 = nan on the device; the pipeline handles that case as the reference does (zeros)."""
    _need_cuda(x)
    assert x.dtype == F32 and x.is_contiguous()
    ws = torch.empty(2, dtype=torch.int32, device=x.device)
    mm = torch.empty(2, dtype=F32, device=x.device)
    _ck(_lib.load().b200_minmax_normalise(_p(x), x.numel(), _p(ws), _p(mm), _stream()), "b200_minmax_normalise")
    return x, mm


def normalise_rgb(rgb: torch.Tensor, round_u8=False):
    """uint8 / float [0,255] image -> fp32 x / 255 * 2 - 1.  `round_u8`: round to the nearest integer first (the
    reference resizes a uint8 tensor with torchvision, which rounds its float result back to uint8)."""
    _need_cuda(rgb)
    x = rgb.contiguous() if rgb.dtype == torch.uint8 else rgb.to(F32).contiguous()
    out = torch.empty(x.shape, dtype=F32, device=x.device)
    _ck(_lib.load().b200_rgb_normalise(_p(x), int(x.dtype == torch.uint8), x.numel(), int(round_u8), _p(out), _stream()),
        "b200_rgb_normalise")
    return out


def resize_bicubic_aa(x: torch.Tensor, size):
    """torchvision `resize(x, size, BICUBIC, antialias=True)` of a [..., H, W] CUDA tensor (geowizard_pipeline.py:239-243)."""
    return resize_bilinear_aa(x, size, _fn="b200_resize_bicubic_aa")


def resize_bilinear_aa(x: torch.Tensor, size, _fn="b200_resize_bilinear_aa"):
    """torchvision `resize(x, size, BILINEAR, antialias=True)` of a [..., H, W] fp32 CUDA tensor."""
    _need_cuda(x)
    xf = x.to(F32).contiguous()
    H, W = xf.shape[-2:]
    OH, OW = int(size[0]), int(size[1])
    planes = xf.numel() // (H * W)
    tmp = torch.empty((planes, H, OW), dtype=F32, device=x.device)
    out = torch.empty((*xf.shape[:-2], OH, OW), dtype=F32, device=x.device)
    _ck(getattr(_lib.load(), _fn)(_p(xf), planes, H, W, OH, OW, _p(tmp), _p(out), _stream()), _fn)
    return out


def resize_nearest(x: torch.Tensor, size):
    _need_cuda(x)
    xf = x.to(F32).contiguous()
    H, W = xf.shape[-2:]
    OH, OW = int(size[0]), int(size[1])
    planes = xf.numel() // (H * W)
    out = torch.empty((*xf.shape[:-2], OH, OW), dtype=F32, device=x.device)
    _ck(_lib.load().b200_resize_nearest(_p(xf), planes, H, W, OH, OW, _p(out), _stream()), "b200_resize_nearest")
    return out


def resize_nearest_exact(x: torch.Tensor, size):
    """torch `interpolate(x, size, mode="nearest-exact")` of a [..., H, W] CUDA tensor: the reference's
    resample_method="nearest" (torchvision NEAREST_EXACT, Marigold/marigold/util/image_util.py:111-116)."""
    _need_cuda(x)
    xf = x.to(F32).contiguous()
    H, W = xf.shape[-2:]
    OH, OW = int(size[0]), int(size[1])
    planes = xf.numel() // (H * W)
    out = torch.empty((*xf.shape[:-2], OH, OW), dtype=F32, device=x.device)
    _ck(_lib.load().b200_resize_nearest_exact(_p(xf), planes, H, W, OH, OW, _p(out), _stream()),
        "b200_resize_nearest_exact")
    return out


# ------------------------------------------------------------------------------------ colour maps
# matplotlib is not a dependency, so the one colour map the reference pipelines default to ("Spectral") is derived
# here the way matplotlib builds and applies it, in numpy float64:
#   * matplotlib/_cm.py `_Spectral_data`: the 11 ColorBrewer control colours, each component k / 255;
#   * matplotlib/colors.py `LinearSegmentedColormap.from_list(name, colors, N=256)`: the colours sit at
#     np.linspace(0, 1, 11), each channel a segment table [x, y0, y1] with y0 == y1;
#   * `_create_lookup_table(N, data, gamma=1)`: x * (N - 1), searchsorted of (N - 1) * linspace(0, 1, N) over it for
#     the interior entries, linear interpolation, the two end entries copied from the table ends, clipped to [0, 1];
#   * `Colormap.__call__(X, bytes=False)` returns lut[index] as float64, and the reference pipelines store
#     `(colored * 255).astype(np.uint8)` (Marigold/marigold/marigold_pipeline.py:331-336,
#     GeoWizard/geowizard/models/geowizard_pipeline.py:211-216): that truncation is folded into the uint8 table, so
#     the device kernel only clips, indexes and gathers.
SPECTRAL_CONTROL_RGB = ((158, 1, 66), (213, 62, 79), (244, 109, 67), (253, 174, 97), (254, 224, 139), (255, 255, 191),
                        (230, 245, 152), (171, 221, 164), (102, 194, 165), (50, 136, 189), (94, 79, 162))
COLOR_MAPS = ("Spectral",)
_LUT_SIZE = 256


def _create_lookup_table(N, x, y0, y1):
    """matplotlib.colors._create_lookup_table(N, np.column_stack([x, y0, y1]), gamma=1.0) for N > 1."""
    x = x * (N - 1)
    xind = (N - 1) * np.linspace(0, 1, N)
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


def spectral_lut(N=_LUT_SIZE):
    """matplotlib's "Spectral" lookup table: float64 [N, 3] in [0, 1]."""
    rgb = np.array(SPECTRAL_CONTROL_RGB, dtype=np.float64) / 255
    vals = np.linspace(0, 1, len(rgb))
    return np.stack([_create_lookup_table(N, vals, rgb[:, c], rgb[:, c]) for c in range(3)], axis=1)


def check_color_map(cmap):
    """None (no depth colouring) or a built-in colour map name; anything else raises before any launch."""
    if cmap is not None and cmap not in COLOR_MAPS:
        raise ValueError(f"color_map={cmap!r}: only {' / '.join(repr(c) for c in COLOR_MAPS)} is built in "
                         "(or None for no depth colouring)")


_TABLES = {}


def _color_table(cmap, device):
    """The uint8 [N, 3] table of `cmap` (a name in COLOR_MAPS) on `device`, built once per device."""
    key = (cmap, device)
    t = _TABLES.get(key)
    if t is None:
        table = (spectral_lut() * 255).astype(np.uint8)
        t = _TABLES[key] = torch.from_numpy(np.ascontiguousarray(table)).to(device)
    return t


def colorize_depth(x: torch.Tensor, cmap="Spectral"):
    """[H, W] (or [1, H, W]) fp32 depth in [0, 1] -> uint8 [H, W, 3] CUDA tensor: the reference's
    `colorize_depth_maps(pred, 0, 1, cmap)` -> `(colored * 255).astype(np.uint8)` -> `chw2hwc`
    (marigold_pipeline.py:327-338).  Values are clipped to [0, 1]; NaN gives (0, 0, 0)."""
    check_color_map(cmap)
    _need_cuda(x)
    xf = x.to(F32).contiguous()
    H, W = xf.shape[-2:]
    assert xf.numel() == H * W, f"colorize_depth takes one [H, W] map, got {tuple(x.shape)}"
    table = _color_table(cmap, xf.device)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=xf.device)
    _ck(_lib.load().b200_colorize_depth(_p(xf), H * W, _p(table), table.shape[0], _p(out), _stream()),
        "b200_colorize_depth")
    return out


def colorize_normals(x: torch.Tensor):
    """[3, H, W] fp32 normals -> uint8 [H, W, 3] CUDA tensor: ((clip(x, -1, 1) + 1) / 2 * 255).astype(np.uint8) in
    HWC (marigold_pipeline.py:339-343, geowizard_pipeline.py:218-219).  NaN gives 0."""
    _need_cuda(x)
    xf = x.to(F32).contiguous()
    assert xf.dim() == 3 and xf.shape[0] == 3, f"colorize_normals takes [3, H, W], got {tuple(x.shape)}"
    H, W = xf.shape[-2:]
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=xf.device)
    _ck(_lib.load().b200_colorize_normals(_p(xf), H * W, _p(out), _stream()), "b200_colorize_normals")
    return out


def ensemble_depths(input_images: torch.Tensor, regularizer_strength: float = 0.02, max_iter: int = 2,
                    tol: float = 1e-3, reduction: str = "median", max_res: int = None):
    """Marigold/marigold/util/ensemble.py:40-132 — align E affine-invariant depth maps [E,H,W] by per-map scale and
    shift (scipy BFGS on the host, objective on the device), reduce with the median (uncertainty = MAD) or the mean
    (uncertainty = std), rescale to [0, 1].  Returns (aligned [H,W], uncertainty [H,W])."""
    from scipy.optimize import minimize
    _need_cuda(input_images)
    if reduction not in ("median", "mean"):
        raise ValueError(f"Unknown reduction method: {reduction}")
    red = 0 if reduction == "median" else 1
    dtype, dev = input_images.dtype, input_images.device
    n_img = input_images.shape[0]
    if n_img > MAX_ENSEMBLE:
        raise ValueError(f"ensemble_size {n_img} > {MAX_ENSEMBLE} supported by the device kernel")
    original = input_images.detach().to(F32).contiguous()
    work = original
    if max_res is not None:                                            # :61-65 nearest down-scaling for the optimisation
        H, W = original.shape[-2:]
        sf = min(max_res / H, max_res / W)
        if sf < 1:
            work = resize_nearest(original, (int(np.floor(H * sf)), int(np.floor(W * sf))))
    E = n_img
    flat = work.reshape(E, -1)
    HW = flat.shape[1]
    L = _lib.load()

    mm = minmax_rows(flat).cpu().numpy()                               # :67-71 init guess (the reference's .cpu() too)
    _min, _max = mm[:, 0].astype(np.float32), mm[:, 1].astype(np.float32)
    s_init = (1.0 / (_max - _min)).reshape((-1, 1, 1))
    t_init = (-1 * s_init.flatten() * _min.flatten()).reshape((-1, 1, 1))
    x = np.concatenate([s_init, t_init]).reshape(-1).astype(np.float32)

    ws = torch.empty(2, dtype=torch.float64, device=dev)
    out3 = torch.empty(3, dtype=F32, device=dev)
    st_dev = torch.empty(2 * E, dtype=F32, device=dev)
    n_pairs = E * (E - 1) // 2

    def closure(xv):
        st_dev.copy_(torch.from_numpy(np.ascontiguousarray(xv, dtype=np.float32)))
        _ck(L.b200_ensemble_depths_objective(_p(flat), _p(st_dev[:E]), _p(st_dev[E:]), E, HW, red, _p(ws), _p(out3),
                                             _stream()), "b200_ensemble_depths_objective")
        sumsq = float(ws[0])                                           # device sync, where the reference has .cpu()
        lo, hi = float(out3[1]), float(out3[2])
        sqrt_dist = np.sqrt(np.float32(sumsq / max(1, n_pairs * HW)), dtype=np.float32) if n_pairs else np.float32(np.nan)
        near_err = np.sqrt(np.float32((0 - lo) ** 2), dtype=np.float32)
        far_err = np.sqrt(np.float32((1 - hi) ** 2), dtype=np.float32)
        return np.float32(sqrt_dist + (near_err + far_err) * np.float32(regularizer_strength))

    res = minimize(closure, x, method="BFGS", tol=tol, options={"maxiter": max_iter, "disp": False})
    x = np.asarray(res.x, dtype=np.float32)
    st_dev.copy_(torch.from_numpy(x))
    aligned = torch.empty(original.shape[1:], dtype=F32, device=dev)
    unc = torch.empty_like(aligned)
    ws2 = torch.empty(2, dtype=torch.float64, device=dev)
    _ck(L.b200_ensemble_depths_reduce(_p(original.reshape(E, -1)), _p(st_dev[:E]), _p(st_dev[E:]), E,
                                      aligned.numel(), red, _p(ws2), _p(aligned), _p(unc), _stream()),
        "b200_ensemble_depths_reduce")
    return aligned.to(dtype), unc.to(dtype)
