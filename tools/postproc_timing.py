"""Time the resampling / colouring kernels and the post-processing tail of MarigoldPipeline.__call__.

    python tools/postproc_timing.py [--out FILE] [--reps N]

At output sizes 768x768 and 3840x2160 (4K UHD):
* each new kernel: `resize_nearest_exact` of a 3-plane fp32 map from half resolution up to the output size,
  `colorize_depth` of an fp32 [H, W] map, `colorize_normals` of an fp32 [3, H, W] map.  CUDA-event time per call
  (median over --iters back-to-back launches per rep, median of --reps), bytes from shapes (each element read once,
  each output written once; the 768-byte colour table is not counted), GB/s = bytes / time;
* the tail of `__call__` (MarigoldPipeline._postprocess): from the ensembled fp32 prediction at processing
  resolution (max edge 768) to the returned numpy arrays and PIL images, depth and normals, colouring on and off,
  each resample method.  CUDA events around a call that ends in its device-to-host copies;
* for context only, the HOST time of the numpy restatement of the reference's colouring (matplotlib's
  Colormap.__call__ on float64, * 255, astype(uint8), chw2hwc) on the same map, labelled as host time.

The device name, power limit and SM clocks come from a read-only nvidia-smi query in the same process.  Prints one
JSON object.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from vae_attention_timing import _gpu_info  # noqa: E402

SIZES = ((768, 768), (2160, 3840))


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def _time_kernel(fn, reps, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    return _median(ts)


def _time_call(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return _median(ts)


def _host_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return _median(ts)


@torch.no_grad()
def time_kernels(H, W, reps, iters):
    from diffusion_e2e_ft_b200.ensemble import colorize_depth, colorize_normals, resize_nearest_exact
    g = torch.Generator(device="cuda").manual_seed(0)
    src = torch.rand(3, H // 2, W // 2, device="cuda", generator=g)
    depth = torch.rand(H, W, device="cuda", generator=g)
    normal = torch.rand(3, H, W, device="cuda", generator=g) * 2 - 1
    out = {}
    for name, fn, nbytes in (
            ("resize_nearest_exact", lambda: resize_nearest_exact(src, (H, W)), 4 * (src.numel() + 3 * H * W)),
            ("colorize_depth", lambda: colorize_depth(depth), 4 * H * W + 3 * H * W),
            ("colorize_normals", lambda: colorize_normals(normal), 4 * 3 * H * W + 3 * H * W)):
        ms = _time_kernel(fn, reps, iters)
        out[name] = dict(ms=ms, bytes=nbytes, gb_per_s=nbytes / (ms * 1e-3) / 1e9)
    return out


@torch.no_grad()
def time_tail(H, W, reps):
    from diffusion_e2e_ft_b200 import MarigoldPipeline
    from diffusion_e2e_ft_b200.pipelines import _max_res_size
    pipe = MarigoldPipeline(None, None, None)
    h, w = _max_res_size(H, W, 768)
    g = torch.Generator(device="cuda").manual_seed(1)
    preds = dict(depth=torch.rand(h, w, device="cuda", generator=g),
                 normals=torch.randn(3, h, w, device="cuda", generator=g))
    out = []
    for kind, pred in preds.items():
        normals = kind == "normals"
        for method in ("bilinear", "bicubic", "nearest"):
            # normals are always coloured (the reference does so whatever color_map is); depth with and without
            for cmap in (("Spectral",) if normals else ("Spectral", None)):
                fn = lambda: pipe._postprocess(pred, None, (H, W), normals=normals, resample_method=method,  # noqa: E731
                                               color_map=cmap)
                ms = _time_call(fn, reps)
                out.append(dict(pred=kind, processing_hw=[h, w], resample_method=method, coloured=cmap is not None,
                                ms=ms))
    return out


def time_host_colouring(H, W, reps):
    from outputs_reference import mpl_colorize_depth, mpl_spectral_lut, np_colorize_normals
    rng = np.random.default_rng(0)
    depth = rng.random((H, W), dtype=np.float32)
    normal = rng.random((3, H, W), dtype=np.float32) * 2 - 1
    lut = mpl_spectral_lut()
    return dict(depth_host_ms=_host_ms(lambda: mpl_colorize_depth(depth, lut), reps),
                normals_host_ms=_host_ms(lambda: np_colorize_normals(normal), reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON here")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("postproc_timing needs a CUDA device")
    res = dict(gpu=_gpu_info(), sizes={})
    for H, W in SIZES:
        r = dict(kernels=time_kernels(H, W, a.reps, a.iters), tail=time_tail(H, W, a.reps),
                 host_time_numpy_reference_colouring=time_host_colouring(H, W, 3))
        res["sizes"][f"{W}x{H}"] = r
        print(json.dumps({f"{W}x{H}": r}), flush=True)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
