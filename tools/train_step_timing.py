"""Time the engine's fine-tuning iteration (training/train.py:469-568: VAE encode -> UNet -> decode -> SSI loss ->
backward -> clip -> AdamW) at the full SD-2 model size on one GPU.  Random-init weights, synthetic batch.
Not the headline metric (that is inference images/s, bench.py) — a first measurement of row a10.

    python tools/train_step_timing.py --batch 2 --height 512 --width 640 --steps 2 --warmup 1
    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/train_step_timing.py   # SURVEY §8(d) config 3:
        data parallel, bs 2 per rank, one NCCL all-reduce of the flat gradient per step; max over ranks, all-reduce timed
        separately on the device
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--breakdown", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "train_step.json"))
    a = ap.parse_args()
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler, ops
    from diffusion_e2e_ft_b200.training import FlatTrainer, e2e_ft_loss
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = f"cuda:{local}"
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl")
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = B200UNet2DConditionModel()
        vae = B200AutoencoderKL()
    vae.eval().requires_grad_(False)
    unet.train().requires_grad_(True)
    tr = FlatTrainer(unet, lr=3e-5)
    g = torch.Generator(device=dev).manual_seed(5 + rank)                      # different images per rank
    rgb = torch.rand(a.batch, 3, a.height, a.width, device=dev, generator=g) * 2 - 1
    gt = torch.rand(a.batch, 1, a.height, a.width, device=dev, generator=g) * 9.9 + 0.1
    mask = torch.rand(a.batch, 1, a.height, a.width, device=dev, generator=g) > 0.2
    ete = torch.randn(1, 77, 1024, device=dev, generator=g) * 0.5
    sched = DDIMScheduler()
    losses, times, ar_ms = [], [], []
    for it in range(a.warmup + a.steps):
        torch.cuda.synchronize()
        ops.STATS.reset()
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        loss, _ = e2e_ft_loss(unet, vae, sched, rgb, gt, mask, ete, "depth")
        e1.record()
        tr.backward(loss)
        tr.step()
        e2.record()
        torch.cuda.synchronize()
        losses.append(loss.item())
        if it >= a.warmup:
            times.append((e0.elapsed_time(e1), e1.elapsed_time(e2)))
            if world > 1:                                   # the exchange alone, on the same buffer
                from diffusion_e2e_ft_b200.training import allreduce_mean_
                a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                dist.barrier()
                a0.record()
                allreduce_mean_(tr.flat_grad)
                a1.record()
                torch.cuda.synchronize()
                ar_ms.append(a0.elapsed_time(a1))
    # per-op-kind GPU time of one more iteration (CUDA events around every op: adds launch gaps, so the sums
    # are kernel time, not wall time)
    breakdown = {}
    if a.breakdown:
        ops.STATS.time_all, ops.STATS.op_events = True, []
        loss, _ = e2e_ft_loss(unet, vae, sched, rgb, gt, mask, ete, "depth")
        n_fwd = len(ops.STATS.op_events)
        tr.backward(loss)
        tr.step()
        torch.cuda.synchronize()
        ops.STATS.time_all = False
        for i, (name, e0, e1) in enumerate(ops.STATS.op_events):
            k = ("fwd." if i < n_fwd else "bwd.") + name
            breakdown[k] = breakdown.get(k, 0.0) + e0.elapsed_time(e1)
        breakdown = {k: round(v, 2) for k, v in sorted(breakdown.items(), key=lambda kv: -kv[1])}
    fwd = sum(t[0] for t in times) / len(times)
    bwd = sum(t[1] for t in times) / len(times)
    if world > 1:                                           # max over ranks of the device times
        t = torch.tensor([fwd, bwd, sum(ar_ms) / len(ar_ms)], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        fwd, bwd, ar = (float(v) for v in t)
    else:
        ar = 0.0
    res = dict(what="fine-tuning iteration, full SD-2 UNet + VAE, depth recipe", batch=a.batch, height=a.height,
               width=a.width, steps=a.steps, warmup=a.warmup, forward_ms=fwd, backward_optimizer_ms=bwd,
               ms_per_step=fwd + bwd, images_per_s=world * a.batch / ((fwd + bwd) / 1e3), n_gpus=world,
               allreduce_ms=ar, grad_bytes=int(tr.flat_grad.numel()) * 4, losses=losses,
               launches_last_step=ops.STATS.launches, peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30,
               breakdown_ms=breakdown, breakdown_sum_ms=round(sum(breakdown.values()), 1),
               finite=all(l == l and abs(l) < 1e9 for l in losses), time=time.strftime("%Y-%m-%d %H:%M:%S"))
    if rank == 0:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
