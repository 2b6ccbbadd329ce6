"""Time the grouped fused AdamW (`b200_adamw_step_state_groups`, GeoWizard's 3-run / 2-group table) against the
one-group `b200_adamw_step_state` on the flat buffers of the SD-2-sized GeoWizard UNet, the two alternating in one
session, and time `FlatTrainer.save_state` / `load_state` with and without the EMA.  Prints the device name and power
limit of the card it ran on.

    python tools/training_state_timing.py --rounds 5 --reps 20 --out /tmp/training_state.json

Kernel time: CUDA events around `reps` back-to-back steps (sum-of-squares excluded; the per-step prepare kernel
included in both).  Bytes: 16 B read + 12 B written per parameter (the run table is a few bytes per block).
Checkpoint time: host clock around the call, which ends with every buffer on the host / device (a sync); the
checkpoint is written under --dir and deleted afterwards."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from diffusion_train_timing import HBM_BYTES_PER_S, events_ms, power_limit     # noqa: E402


def folder_bytes(d):
    return sum(os.path.getsize(os.path.join(r, f)) for r, _, fs in os.walk(d) for f in fs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "training_state_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU timing")
    from diffusion_e2e_ft_b200 import B200UNet2DConditionModel, ops, training
    dev = "cuda:0"
    out = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit())
    print(json.dumps(out), flush=True)
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = B200UNet2DConditionModel(class_embed_type="projection", projection_class_embeddings_input_dim=10,
                                        cross_attention_dim=768, joint_attention=True)
    unet.train().requires_grad_(True)
    groups = training.geowizard_param_groups(10)
    tr = training.FlatTrainer(unet, lr=3e-5, param_groups=groups)
    n = tr.flat_param.numel()
    out.update(params=sum(p.numel() for p in unet.parameters()), flat_elements=n, runs=len(tr._runs))
    g = torch.Generator(device=dev).manual_seed(5)
    tr.flat_grad.copy_(torch.randn(n, device=dev, generator=g) * 1e-3 * tr.loss_scale())
    nsq = ops.grad_norm_sq(tr.flat_grad)
    args = (tr.flat_param, tr.flat_grad, tr.exp_avg, tr.exp_avg_sq, tr.state, nsq)
    lrs, wds = tr.get_last_lr(), [gd["weight_decay"] for gd in tr._group_def]

    def single():
        ops.adamw_step_state(*args, lr=lrs[0], weight_decay=wds[0], max_grad_norm=1.0, growth_interval=10 ** 9)

    def grouped():
        ops.adamw_step_state_groups(*args, *tr._run_table, lrs, wds, max_grad_norm=1.0, growth_interval=10 ** 9)

    for fn in (single, grouped):
        fn()
    times = dict(single=[], grouped=[])
    for _ in range(a.rounds):
        for name, fn in (("single", single), ("grouped", grouped)):
            times[name].append(events_ms(fn, a.reps))
    bytes_per_step = 28 * n
    for name, ts in times.items():
        med = statistics.median(ts)
        out[f"adamw_{name}_ms"] = dict(median=med, min=min(ts), max=max(ts), all=ts,
                                       tb_per_s=bytes_per_step / (med * 1e-3) / 1e12,
                                       share_of_hbm_peak=bytes_per_step / (med * 1e-3) / HBM_BYTES_PER_S)
    print(json.dumps({k: v for k, v in out.items() if k.startswith("adamw")}), flush=True)

    # save / load of the whole training state
    for use_ema in (False, True):
        if use_ema:
            del tr
            torch.cuda.empty_cache()
            tr = training.FlatTrainer(unet, lr=3e-5, param_groups=groups, use_ema=True)
            tr.flat_grad.copy_(torch.randn(n, device=dev, generator=g) * 1e-3 * tr.loss_scale())
            tr._micro, tr._synced = 0, True
            tr.step()
        d = tempfile.mkdtemp(prefix="training_state_", dir=a.dir)
        key = "with_ema" if use_ema else "without_ema"
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.save_state(os.path.join(d, "checkpoint-1"))
            t1 = time.perf_counter()
            size = folder_bytes(os.path.join(d, "checkpoint-1"))
            tr.load_state(os.path.join(d, "checkpoint-1"))
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            out[key] = dict(save_s=t1 - t0, load_s=t2 - t1, bytes=size, save_gb_per_s=size / (t1 - t0) / 1e9,
                            load_gb_per_s=size / (t2 - t1) / 1e9)
        except OSError as e:                     # e.g. no room for the ~10-14 GB folder under --dir
            out[key] = dict(error=f"not measured: {e}")
        finally:
            shutil.rmtree(d, ignore_errors=True)
        print(json.dumps({key: out[key]}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
