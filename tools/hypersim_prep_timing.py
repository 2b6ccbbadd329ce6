"""Time the Hypersim preprocessing (diffusion_e2e_ft_b200.data.hypersim_frames / preprocess_hypersim).

    python tools/hypersim_prep_timing.py [--frames 48] [--out out/hypersim_prep_timing.json]

- Kernel time per 768x1024 frame at B = 1 and B = 8 on typical frames, and at B = 1 on the worst case (every level
  exactly on a boundary): the summed device time of the call's kernels from
  torch.profiler, and CUDA events around many raw C-ABI calls on preallocated buffers, both after warm-up.  Against
  it: the essential bytes (fp16 radiance and distance, int32 entity ids in; uint8 BGR and uint16 depth out) per
  second, over the H100 SXM data sheet's 3.35 TB/s.
- preprocess_hypersim frames/s over `--frames` synthetic frames (an in-memory h5py stand-in) written to a temporary
  directory on local disk, end to end and split into its stages run on their own: read (DataLoader workers), kernel +
  copies, encode + write (with the metadata).
- The CPU time per frame of the numpy oracle (tests/hypersim_oracle.py) on the same host: a CPU number.
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
from diffusion_e2e_ft_b200 import lib as _lib  # noqa: E402

H, W = 768, 1024
HBM_BPS = 3.35e12
BYTES_PER_PIXEL = 3 * 2 + 2 + 4 + 3 + 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def typical_frames(n):
    """n seeded Hypersim-like frames: lognormal HDR fp16 radiance, fp16 distances, 7 % invalid pixels."""
    rng = np.random.default_rng(2024)
    out = []
    for _ in range(n):
        eid = rng.integers(1, 400, (H, W)).astype(np.int32)
        eid[rng.random((H, W)) < 0.07] = -1
        out.append((np.exp(rng.normal(-1.5, 1.5, (H, W, 3))).astype(np.float16),
                    (1.0 + 20.0 * rng.random((H, W))).astype(np.float16), eid))
    return out


def kernel_us_per_frame(frames, B, iters):
    dev = torch.device("cuda", 0)
    rgb, dist, eid = (torch.from_numpy(np.stack([f[k] for f in frames[:B]])).to(dev) for k in range(3))
    L = _lib.load()
    bgr = torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev)
    depth = torch.empty((B, H, W), dtype=torch.uint16, device=dev)
    err = torch.empty(B, dtype=torch.int32, device=dev)
    ws = torch.empty(L.b200_data_hypersim_workspace_bytes(B, H, W) // 8 + 1, dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def call():
        _lib.check(L.b200_data_hypersim_frames(rgb.data_ptr(), 1, dist.data_ptr(), 1, eid.data_ptr(), B, H, W, 886.81,
                                               data._tone_map_numerator(), bgr.data_ptr(), depth.data_ptr(),
                                               err.data_ptr(), None, ws.data_ptr(), ws.numel() * 8, st),
                   "b200_data_hypersim_frames")
    for _ in range(10):
        call()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    ev_us = a.elapsed_time(b) * 1e3 / iters / B
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            call()
        torch.cuda.synchronize()
    dev_us = sum(e.device_time_total for e in prof.key_averages()
                 if e.key.startswith(("void b200::hs_", "b200::hs_")) or "hs_" in e.key) / 20 / B
    per_kernel = {e.key.split("(")[0].replace("void ", "")[:40]: round(e.device_time_total / 20 / B, 2)
                  for e in prof.key_averages() if "hs_" in e.key}
    return {"events_us": round(ev_us, 2), "profiler_us": round(dev_us, 2), "per_kernel_us": per_kernel,
            "essential_GBps": round(H * W * BYTES_PER_PIXEL / (ev_us * 1e-6) / 1e9, 1),
            "share_of_3.35TBps": round(H * W * BYTES_PER_PIXEL / (ev_us * 1e-6) / HBM_BPS, 4)}


def end_to_end(n, batch_size, workers):
    import make_hypersim_pins as mk
    cases = ["random_hdr", "nan_invalid", "nan_dist", "index_integral"]
    base = {c: mk.case_arrays(c) for c in cases}
    frames = tuple((cases[i % 4], f"ai_{i // 16:03d}_001", "cam_00", i, "train", True) for i in range(n))
    orig = mk.case_arrays
    mk.case_arrays = lambda name: base[name]
    with tempfile.TemporaryDirectory() as tmp:
        raw, csv = os.path.join(tmp, "raw"), os.path.join(tmp, "split.csv")
        registry = mk.write_raw_tree(raw, csv, frames)
        mk.case_arrays = orig
        sys.modules["h5py"] = mk.h5py_stub(registry)
        dev = torch.device("cuda", 0)
        ds = data._HypersimRawFrames(raw, [(i, mk.input_paths(*f[1:4])) for i, f in enumerate(frames)])
        loader = torch.utils.data.DataLoader(ds, batch_size=None, num_workers=workers)
        t0 = time.perf_counter()
        decoded = list(data._equal_size_batches(loader, batch_size))
        t_read = time.perf_counter() - t0
        data._hypersim_on_host(*decoded[0][1], 886.81, dev)           # warm-up
        t0 = time.perf_counter()
        outs = [(idx, data._hypersim_on_host(*t, 886.81, dev), t[2].numpy()) for idx, t in decoded]
        t_kernel = time.perf_counter() - t0
        os.makedirs(os.path.join(tmp, "stage"))
        t0 = time.perf_counter()
        with ThreadPoolExecutor(workers) as pool:
            jobs = [(os.path.join(tmp, "stage"), i, f"s/rgb_{i}.png", f"s/depth_{i}.png", b, d, e != -1)
                    for idx, (bgr, dep), eid in outs for i, b, d, e in zip(idx, bgr, dep, eid)]
            list(pool.map(lambda a: data._write_hypersim_frame(*a), jobs))
        t_write = time.perf_counter() - t0
        t0 = time.perf_counter()
        written = data.preprocess_hypersim(csv, raw, os.path.join(tmp, "out"), batch_size=batch_size,
                                           num_workers=workers, device=dev)
        t_all = time.perf_counter() - t0
        assert written == n
    return {"frames": n, "batch_size": batch_size, "workers": workers, "frames_per_s": round(n / t_all, 1),
            "stage_frames_per_s": {"read": round(n / t_read, 1), "kernel_and_copies": round(n / t_kernel, 1),
                                   "encode_write_and_metadata": round(n / t_write, 1)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "hypersim_prep_timing.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    import hypersim_oracle as oracle
    import make_hypersim_pins as mk
    frames = typical_frames(8)
    # the constant frame puts every channel on the 90th-percentile brightness, so every level sits exactly on the
    # 204 boundary and takes the double-double power: the worst case, timed on its own
    res = {"card": card(), "cpus": os.cpu_count(),
           "kernel": {"B1": kernel_us_per_frame(frames, 1, 200), "B8": kernel_us_per_frame(frames, 8, 50),
                      "B1_constant_worst_case": kernel_us_per_frame([mk.case_arrays("constant")], 1, 50)},
           "preprocess": end_to_end(args.frames, 8, 4)}
    t0 = time.perf_counter()
    for f in frames[:2]:
        oracle.frame(*f)
    res["cpu_oracle_ms_per_frame"] = round((time.perf_counter() - t0) * 1e3 / 2, 1)
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
