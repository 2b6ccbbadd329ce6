"""TEST INFRASTRUCTURE ONLY: numpy / torchvision restatements of the reference pipelines' output post-processing
(Marigold/marigold/marigold_pipeline.py:237-247,298-343, Marigold/marigold/util/image_util.py:29-67) and of the
matplotlib code they call, shared by tests/test_outputs_cpu.py and tests/test_outputs_gpu.py.  matplotlib is not a
dependency of the project, so its "Spectral" colour map and Colormap.__call__ are written out here independently of the product's
table derivation (diffusion_e2e_ft_b200/ensemble.py)."""
import numpy as np
import torch

SPECTRAL_11 = ((158, 1, 66), (213, 62, 79), (244, 109, 67), (253, 174, 97), (254, 224, 139), (255, 255, 191),
               (230, 245, 152), (171, 221, 164), (102, 194, 165), (50, 136, 189), (94, 79, 162))


# ------------------------------------------------------------------------------------------------ matplotlib, restated
def mpl_spectral_lut(N=256):
    """matplotlib's LinearSegmentedColormap.from_list("Spectral", colours, N) lookup table, written out entry by entry:
    _create_lookup_table(N, [x, y0, y1], gamma=1) with searchsorted (side="left") over x * (N - 1)."""
    x = np.linspace(0, 1, len(SPECTRAL_11)) * (N - 1)
    xind = (N - 1) * np.linspace(0, 1, N)
    lut = np.zeros((N, 3))
    for c in range(3):
        y = [k[c] / 255 for k in SPECTRAL_11]
        lut[0, c], lut[N - 1, c] = y[0], y[-1]
        for j in range(1, N - 1):
            i = next(i for i in range(len(x)) if x[i] >= xind[j])
            d = (xind[j] - x[i - 1]) / (x[i] - x[i - 1])
            lut[j, c] = min(max(d * (y[i] - y[i - 1]) + y[i - 1], 0.0), 1.0)
    return lut


def mpl_colorize_depth(depth, lut):
    """Marigold's colorize_depth_maps(depth, 0, 1, cmap) -> (colored * 255).astype(np.uint8) -> chw2hwc, with
    matplotlib's Colormap.__call__(X, bytes=False) restated (under / over / bad = lut[0] / lut[-1] / (0, 0, 0, 0))."""
    depth = np.array(depth, copy=True).squeeze()[None]
    depth = ((depth - 0) / (1 - 0)).clip(0, 1)
    N = lut.shape[0]
    rgba = np.concatenate([lut, np.ones((N, 1))], axis=1)
    rgba = np.concatenate([rgba, rgba[:1], rgba[-1:], np.zeros((1, 4))])      # _i_under, _i_over, _i_bad
    xa = np.array(depth, copy=True)
    xa *= N
    xa[xa == N] = N - 1
    under, over, bad = xa < 0, xa >= N, np.isnan(xa)
    with np.errstate(invalid="ignore"):
        xa = xa.astype(int)
    xa[under], xa[over], xa[bad] = N, N + 1, N + 2
    colored = rgba.take(xa, axis=0, mode="clip")[:, :, :, 0:3]
    colored = np.rollaxis(colored, 3, 1).squeeze()
    colored = (colored * 255).astype(np.uint8)
    return np.moveaxis(colored, 0, -1)


def np_colorize_normals(normal_chw):
    """marigold_pipeline.py:340-343 on a [3, H, W] float32 array: clip, ((n + 1) / 2 * 255).astype(uint8), HWC."""
    n = normal_chw.clip(-1.0, 1.0)
    with np.errstate(invalid="ignore"):
        return np.moveaxis((((n + 1) / 2) * 255).astype(np.uint8), 0, -1)


def special_depths():
    """0, 1, every k/256 boundary and its float32 neighbours, values outside [0, 1], NaN."""
    k = np.arange(257, dtype=np.float32) / np.float32(256)
    vals = [k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)),
            np.array([0, 1, -0.0, -1e-30, -3, 1 + 1e-7, 7, np.inf, -np.inf, np.nan, 0.5, 0.999999], np.float32)]
    return np.concatenate(vals).astype(np.float32)



def tv_mode(method):
    from torchvision.transforms import InterpolationMode
    return {"bilinear": InterpolationMode.BILINEAR, "bicubic": InterpolationMode.BICUBIC,
            "nearest": InterpolationMode.NEAREST_EXACT}[method]


def ref_marigold_post(pred, input_hw, method, normals, color_map, lut):
    """marigold_pipeline.py:298-343 on the host: normalise, torchvision resize back, numpy clip and colouring."""
    from torchvision.transforms.functional import resize
    if normals:
        pred = pred / (torch.norm(pred, p=2, dim=0, keepdim=True) + 1e-5)
    else:
        lo, hi = torch.min(pred), torch.max(pred)
        pred = torch.zeros_like(pred) if hi == lo else (pred - lo) / (hi - lo)
    pred = resize(pred if normals else pred.unsqueeze(0), list(input_hw), interpolation=tv_mode(method),
                  antialias=True).squeeze().cpu().numpy()
    if normals:
        pred = pred.clip(-1.0, 1.0)
        return pred, np_colorize_normals(pred)
    pred = pred.clip(0, 1)
    return pred, (mpl_colorize_depth(pred, lut) if color_map is not None else None)


def ref_marigold_pre(img_u8, processing_res, method):
    """marigold_pipeline.py:237-247: resize_max_res on the uint8 tensor (torchvision), then [0,255] -> [-1,1]."""
    from torchvision.transforms.functional import resize
    _, h, w = img_u8.shape
    s = min(processing_res / w, processing_res / h)
    r = resize(img_u8, [int(h * s), int(w * s)], tv_mode(method), antialias=True)
    return r / 255.0 * 2.0 - 1.0
