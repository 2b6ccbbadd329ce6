"""Time the Virtual KITTI 2 normal generation (diffusion_e2e_ft_b200.data.vkitti_normals / generate_vkitti_normals).

    python tools/vkitti_normals_timing.py [--frames 200] [--out out/vkitti_normals_timing.json]

- Kernel time per 375x1242 frame at B = 1 and B = 16: the kernel's duration from torch.profiler, and CUDA events around
  many raw C-ABI calls on preallocated buffers, both after warm-up.  Against it: the essential bytes per second over
  the H100 SXM data sheet's 3.35 TB/s, and an ESTIMATE of the fp64 work (operations counted from the kernel source,
  with assumed instruction costs for exp, division and sqrt) over the data sheet's 34 TFLOP/s fp64 (non-tensor).
- generate_vkitti_normals frames/s over `--frames` synthetic frames in a temporary directory on local disk, end to end
  and split into its three stages run on their own: decode (DataLoader workers), kernel + copies, encode + write.
- The CPU time per frame of the numpy oracle (tests/vkitti_normals_oracle.py) on the same host, as a stand-in for the
  reference script's arithmetic.
Reads the card's name and power limit in the same run.  Prints one JSON line and writes it to --out.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from diffusion_e2e_ft_b200 import data  # noqa: E402

H, W = 375, 1242
HBM_BPS = 3.35e12
FP64_FLOPS = 34e12
# An ESTIMATE of the fp64 work per pixel on the common path of data_vkitti_normals_kernel.  Counted from the source:
# 4 exp, 15 divisions, 1 square root and 66 adds / multiplies / FMAs.  The instruction costs of exp (15), division
# (10) and square root (10) are assumptions, not counts; each instruction is taken as 2 flops, like an FMA.
FP64_FLOP_PER_PIXEL = 2 * (4 * 15 + 15 * 10 + 10 + 66)
BYTES_PER_PIXEL = 2 + 6


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def frames(n):
    import make_vkitti_normals_pins as mk
    base = [mk.case_depth(c) for c in mk.FULL_CASES]
    return [np.clip(base[i % len(base)].astype(np.int64) + (i // len(base)) * 7, 0, 65535).astype(np.uint16)
            for i in range(n)]


def kernel_us_per_frame(depths, B, iters):
    """Per 375x1242 frame: (1) CUDA events around `iters` raw b200_data_vkitti_normals calls on preallocated buffers
    (no Python wrapper between launches), (2) the kernel's own duration from torch.profiler in a separate run."""
    from torch.profiler import ProfilerActivity, profile
    L = data._lib.load()
    d = torch.from_numpy(np.stack([depths[i % len(depths)] for i in range(B)])).cuda()
    out = torch.empty((B, H, W, 3), dtype=torch.uint16, device=d.device)
    st = data._stream()
    args = (data._p(d), B, H, W, data.VKITTI_FX, data.VKITTI_FY, data.VKITTI_U0, data.VKITTI_V0, data._p(out), st)
    for _ in range(5):
        data._ck(L.b200_data_vkitti_normals(*args), "b200_data_vkitti_normals")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.b200_data_vkitti_normals(*args)
    e1.record()
    torch.cuda.synchronize()
    us_events = e0.elapsed_time(e1) * 1e3 / iters / B
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            L.b200_data_vkitti_normals(*args)
        torch.cuda.synchronize()
    kern = [e for e in prof.key_averages() if "vkitti_normals_kernel" in e.key]
    t = getattr(kern[0], "device_time_total", None) if kern else None
    t = t if t is not None else (kern[0].cuda_time_total if kern else float("nan"))
    us = t / iters / B
    px = H * W
    floor_mem, floor_fp64 = BYTES_PER_PIXEL * px / HBM_BPS * 1e6, FP64_FLOP_PER_PIXEL * px / FP64_FLOPS * 1e6
    return {"us_per_frame_kernel_profiler": round(us, 2), "us_per_frame_events_raw_calls": round(us_events, 2),
            "GBps": round(BYTES_PER_PIXEL * px / us / 1e3, 1), "share_of_3.35TBps": round(floor_mem / us, 4),
            "fp64_TFLOPs_estimated": round(FP64_FLOP_PER_PIXEL * px / us / 1e6, 2),
            "share_of_34TFLOPs_fp64_estimated": round(floor_fp64 / us, 3),
            "bound_estimated": "fp64" if floor_fp64 > floor_mem else "HBM"}


def write_tree(root, depths):
    import cv2
    for i, d in enumerate(depths):
        scene = data.VKITTI_SCENES[i % 5]
        variant = data.VKITTI_NORMAL_VARIANTS[(i // 5) % 10]
        for sub, kind in (("vkitti_2.0.3_rgb", "rgb"), ("vkitti_2.0.3_depth", "depth")):
            os.makedirs(os.path.join(root, sub, scene, variant, "frames", kind, "Camera_0"), exist_ok=True)
        open(os.path.join(root, "vkitti_2.0.3_rgb", scene, variant, "frames", "rgb", "Camera_0", f"rgb_{i:05d}.jpg"),
             "wb").close()
        cv2.imwrite(os.path.join(root, "vkitti_2.0.3_depth", scene, variant, "frames", "depth", "Camera_0",
                                 f"depth_{i:05d}.png"), d)


def end_to_end(depths, batch_size, workers):
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "virtual_kitti_2")
        write_tree(root, depths)
        n = len(depths)
        loader = torch.utils.data.DataLoader(data._VKITTIDepthFrames(root), batch_size=None, num_workers=workers)
        t0 = time.perf_counter()
        decoded = list(data._equal_size_batches(loader, batch_size))
        t_decode = time.perf_counter() - t0
        dev = torch.device("cuda", torch.cuda.current_device())
        data._normals_on_host(decoded[0][1], dev)        # warm-up
        t0 = time.perf_counter()
        outs = [(paths, data._normals_on_host(d, dev)) for paths, d in decoded]
        t_kernel = time.perf_counter() - t0
        t0 = time.perf_counter()
        with ThreadPoolExecutor(workers) as pool:
            list(pool.map(lambda a: data._write_png(*a), [(p, o) for paths, b in outs for p, o in zip(paths, b)]))
        t_write = time.perf_counter() - t0
        t0 = time.perf_counter()
        written = data.generate_vkitti_normals(root, batch_size=batch_size, num_workers=workers)
        t_all = time.perf_counter() - t0
        assert written == n
    return {"frames": n, "batch_size": batch_size, "workers": workers, "frames_per_s": round(n / t_all, 1),
            "stage_frames_per_s": {"decode": round(n / t_decode, 1), "kernel_and_copies": round(n / t_kernel, 1),
                                   "encode_and_write": round(n / t_write, 1)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "vkitti_normals_timing.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    import vkitti_normals_oracle as oracle
    depths = frames(args.frames)
    res = {"card": card(), "cpus": os.cpu_count(),
           "kernel": {"B1": kernel_us_per_frame(depths, 1, 500), "B16": kernel_us_per_frame(depths, 16, 100)},
           "generate": end_to_end(depths, 8, 4)}
    t0 = time.perf_counter()
    for d in depths[:4]:
        oracle.normals_frame(d)
    res["cpu_oracle_ms_per_frame"] = round((time.perf_counter() - t0) * 1e3 / 4, 1)
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
