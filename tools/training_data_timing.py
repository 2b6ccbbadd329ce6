"""Device time of diffusion_e2e_ft_b200.data.prepare_batch at bs 2 and full size, for Hypersim (768x1024 -> 480x640)
and Virtual KITTI 2 (375x1242 -> 352x1216 crop): per call from CUDA events around many calls after warm-up (kernels
plus the gaps between launches), and the summed kernel time per call from torch.profiler in a separate run.  Also the host CPU
time per sample of the same transforms done the reference's way (numpy / PIL / torch, tests/data_oracle.py), as a
CPU number.  Prints one JSON line and writes it to out/training_data_timing.json.

    python tools/training_data_timing.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.utils.data import default_collate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from diffusion_e2e_ft_b200 import data  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def batch(domain, H, W, B=2, seed=0):
    rng = np.random.default_rng(seed)
    samples = []
    for b in range(B):
        d = rng.integers(300, 9000, (H, W)).astype(np.uint16)
        d[rng.random((H, W)) < 0.05] = 0
        d[: H // 6] = 65535
        samples.append(data._sample(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), d,
                                    rng.integers(0, 256, (H, W, 3), dtype=np.uint8), b % 2 == 0, True, 1e-5,
                                    65.0 if domain == "indoor" else 80.0, domain))
    return samples


def kernel_time_ms(batch, iters):
    """Device time of prepare_batch's kernels and copies per call (total in ms, and per kernel name in us), from
    torch.profiler in a run of its own."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            data.prepare_batch(batch)
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = t if t is not None else e.cuda_time_total
        if t > 0:
            per_kernel[e.key.split("(")[0][:48]] = round(t / iters, 2)
    return sum(per_kernel.values()) / 1e3, per_kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    import data_oracle as oracle
    res = {"card": card(), "batch": 2}
    for domain, (H, W), (OH, OW) in (("indoor", (768, 1024), data.HYPERSIM_SIZE),
                                     ("outdoor", (375, 1242), data.KB_CROP)):
        samples = batch(domain, H, W)
        raw = default_collate(samples)
        # the images and flip flags already resident; the per-sample settings stay on the host, as collated
        dev = {k: v.cuda() if k in ("rgb", "depth", "normals", "flip") else v for k, v in raw.items()}
        for _ in range(5):
            data.prepare_batch(dev)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            data.prepare_batch(dev)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        kernel_ms, per_kernel = kernel_time_ms(dev, args.iters)
        # bytes that must cross HBM at least: the decoded inputs (3 + 2 + 3 B per source pixel) and the fp32 / bool
        # outputs (3 + 3 + 1 + 3 floats + 1 byte = 41 B per output pixel)
        essential = 2 * (8 * H * W + 41 * OH * OW)
        t0 = time.perf_counter()
        for s in samples:
            oracle.sample_from_raw(s)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / len(samples)
        name = "hypersim" if domain == "indoor" else "vkitti"
        res[name] = {"call_ms_per_batch": round(ms, 4), "kernel_ms_per_batch": round(kernel_ms, 4),
                     "essential_bytes": essential, "essential_GBps_over_kernel_time": round(essential / kernel_ms / 1e6, 1),
                     "kernel_us_per_batch": per_kernel, "host_cpu_ms_per_sample_reference_way": round(cpu_ms, 1)}
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
    open(os.path.join(ROOT, "out", "training_data_timing.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
