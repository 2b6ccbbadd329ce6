"""Time the device evaluators against the reference's evaluation loops as they run on a CUDA machine, in one run.

    depth, per sample   Marigold/eval.py:172-220: host np.linalg.lstsq (alignment.py), numpy clipping, then the ten
                        metric.py calls on CUDA tensors, each ending in .item() (threshold_percentage also does a
                        .cpu()), against DepthEvaluator.update.  NYU 480x640, and ETH3D 4032x6048 at max_res 1024.
    normals, pooled     DSINE/projects/dsine/test.py:100-130: compute_normal_error, torch.cat growth of the masked
                        errors, then compute_normal_metrics (host np.median etc.), against NormalEvaluator.

The reference loops are restated here (the reference is not importable on the GPU machine) with the same torch / numpy
calls.  Inputs are seeded; predictions start on the host as the reference loads them (.npy) and are copied to the
device for the evaluators, and that copy is inside the timed region of both.  Each number is wall time of the whole
loop (host clock around a final synchronise) and CUDA-event time of the same window; the card name and power limit are
printed with the results.

    python tools/eval_timing.py [--samples 200] [--eth3d-samples 10] [--normal-samples 654]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffusion_e2e_ft_b200 import evaluation as ev  # noqa: E402

DEV = "cuda"


# ---- the reference's metric.py calls, restated with the same torch operations
def _masked_mean(x, m):
    x[~m] = 0
    return torch.sum(x, (-1, -2)) / m.sum((-1, -2))


def ref_metrics(p, g, m):
    out = []
    out.append(_masked_mean(torch.abs(p - g) / g, m).mean())
    out.append(_masked_mean(torch.pow(torch.abs(p - g), 2) / g, m).mean())
    out.append(torch.sqrt(_masked_mean(torch.pow(p - g, 2), m)).mean())
    out.append(torch.sqrt(_masked_mean(torch.pow(torch.log(p) - torch.log(g), 2), m)).mean())
    out.append(torch.abs(torch.log10(p[m]) - torch.log10(g[m])).mean())
    for t in (1.25, 1.25 ** 2, 1.25 ** 3):
        mx = torch.max(p / g, g / p)
        bit = torch.where(mx.cpu() < t, torch.ones(*p.shape), torch.zeros(*p.shape))
        bit[~m.cpu()] = 0
        out.append((torch.sum(bit, (-1, -2)) / m.sum((-1, -2)).cpu()).mean())
    out.append(torch.sqrt(_masked_mean(torch.pow(1.0 / p - 1.0 / g, 2), m)).mean())
    d = torch.log(p) - torch.log(g)
    d[~m] = 0
    n = m.sum((-1, -2))
    out.append(torch.sqrt(torch.mean(torch.sum(d * d, (-1, -2)) / n - torch.pow(torch.sum(d, (-1, -2)), 2) / n ** 2)) * 100)
    return [o.item() for o in out]


def ref_align(gt, pred, mask, max_res):
    H, W = pred.shape
    g, p, m = gt, pred, mask
    if max_res is not None:
        s = np.min(max_res / np.array(pred.shape[-2:]))
        if s < 1:
            up = torch.nn.Upsample(scale_factor=s, mode="nearest")
            g = up(torch.as_tensor(g).unsqueeze(0)).numpy()
            p = up(torch.as_tensor(p).unsqueeze(0)).numpy()
            m = up(torch.as_tensor(m).unsqueeze(0).float()).bool().numpy()
    A = np.concatenate([p[m].reshape(-1, 1), np.ones((int(m.sum()), 1), np.float32)], -1)
    scale, shift = np.linalg.lstsq(A, g[m].reshape(-1, 1), rcond=None)[0]
    return pred * scale + shift


def depth_samples(n, H, W, seed):
    rs = np.random.RandomState(seed)
    base = (0.5 + 9.5 * rs.rand(H, W)).astype(np.float32)
    for i in range(n):
        gt = np.roll(base, i, 1)
        pred = ((gt - 0.5) / 9.5 * 0.9 + 0.05 + 0.02 * rs.randn(1, W)).astype(np.float32)
        mask = gt > 0.6 + 0.001 * (i % 50)
        yield gt, pred, mask


def time_loop(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, e0.elapsed_time(e1) / 1e3


def bench_depth(name, n, H, W, max_res):
    data = list(depth_samples(n, H, W, 1))
    gts = [torch.from_numpy(g).to(DEV) for g, _, _ in data]      # ground truth lives on the device in both loops
    masks = [torch.from_numpy(m).to(DEV) for _, _, m in data]

    def reference(k=n):
        for (g, p, m), gd, md in zip(data[:k], gts, masks):
            a = np.clip(np.clip(ref_align(g, p, m, max_res), 0.5, 10.0), 1e-6, None)
            ref_metrics(torch.from_numpy(a).to(DEV), gd, md)

    def device(k=n):
        e = ev.DepthEvaluator(0.5, 10.0, "least_square", max_res)
        for (g, p, m), gd, md in zip(data[:k], gts, masks):
            e.update(torch.from_numpy(p).to(DEV), gd, md)
        e.result()

    reference(2)                                                   # warm-up: library load, allocator, kernels
    device(2)
    r_wall, r_ev = time_loop(reference)
    d_wall, d_ev = time_loop(device)
    print(f"depth {name} {H}x{W} max_res={max_res} samples={n}: reference {r_wall / n * 1e3:.3f} ms/sample "
          f"(events {r_ev / n * 1e3:.3f}), DepthEvaluator {d_wall / n * 1e3:.3f} ms/sample (events {d_ev / n * 1e3:.3f}),"
          f" ratio {r_wall / d_wall:.1f}x")


def bench_normals(n, H, W):
    g = torch.Generator(device=DEV).manual_seed(2)
    gt = torch.nn.functional.normalize(torch.randn(1, 3, H, W, generator=g, device=DEV), dim=1)
    preds = [gt + 0.3 * torch.randn(1, 3, H, W, generator=g, device=DEV) for _ in range(8)]
    mask = torch.rand(1, 1, H, W, generator=g, device=DEV) > 0.1

    def reference():
        total = None
        for i in range(n):
            e = torch.acos(torch.clamp(torch.cosine_similarity(preds[i % 8], gt, dim=1), -1.0, 1.0)) * 180.0 / np.pi
            sel = e.unsqueeze(1)[mask]
            total = sel if total is None else torch.cat((total, sel), dim=0)
        t = total.detach().cpu().numpy()
        npx = t.shape[0]
        return dict(mean=np.average(t), median=np.median(t), rmse=np.sqrt(np.sum(t * t) / npx),
                    **{f"a{k + 1}": 100.0 * (np.sum(t < v) / npx) for k, v in enumerate((5, 7.5, 11.25, 22.5, 30))})

    res = {}

    def device():
        e = ev.NormalEvaluator()
        for i in range(n):
            e.update(preds[i % 8], gt, mask)
        res["dev"] = e.result()

    device()                                                       # warm-up
    r_wall, r_ev = time_loop(reference)
    d_wall, d_ev = time_loop(device)
    print(f"normals pooled {n} x {H}x{W}: reference {r_wall:.3f} s (events {r_ev:.3f}), NormalEvaluator {d_wall:.3f} s "
          f"(events {d_ev:.3f}), ratio {r_wall / d_wall:.1f}x; median {res['dev']['median']:.4f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=200)
    ap.add_argument("--eth3d-samples", type=int, default=10)
    ap.add_argument("--normal-samples", type=int, default=654)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_timing.py measures on a GPU; none is visible")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(), "|", q)
    bench_depth("NYU", args.samples, 480, 640, None)
    bench_depth("ETH3D", args.eth3d_samples, 4032, 6048, 1024)
    bench_normals(args.normal_samples, 480, 640)


if __name__ == "__main__":
    main()
