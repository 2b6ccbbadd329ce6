"""Time and size one Marigold E2E micro-step (forward, loss, backward; no optimizer step) with the VAE decoder's
gradient checkpointing off and on (`vae.enable_gradient_checkpointing()`), alternated in one process.  The UNet
checkpoints its blocks in both (the recipes' --gradient_checkpointing, bench.py's training leg).  SD-2 widths, seeded
weights.  Shapes: 768^2 bs 2 (the recipe), 1024^2 bs 2, 1536^2 bs 1 and 2048^2 bs 1, the last with the memory-efficient
VAE attention (the unfused path cannot index one 2048^2 image's scores).  Reports ms per micro-step (the min over 3
rounds of the mean of 5 steps; every round is listed) and the peak allocated memory of each mode.

At 768^2 bs 2 it also measures the granularity the decoder does not use: diffusers' segments (the mid-block, each up
block with its upsampler), each kept as its input only and re-run as a whole in its backward, for the comparison in
DESIGN.md §7.

A shape and mode run only when their estimated need fits the device: the peak measured at 768^2 bs 2 in the same mode,
scaled by the pixel count, plus the L^2 buffers of the unfused mid-block attention (S and P in its forward, dP and dS
per image in its backward), with a 10 % margin.  No shape is run to find out whether it fits.  Reads the card name,
power limit and max SM clock in the same run.

    python tools/vae_checkpoint_timing.py --out /tmp/vae_checkpoint_timing.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diffusion_e2e_ft_b200 import autograd_blocks as ab  # noqa: E402
from diffusion_e2e_ft_b200.ops import F32  # noqa: E402

GB = 1024 ** 3
SHAPES = [(768, 2, False), (1024, 2, False), (1536, 1, False), (2048, 1, True)]     # (res, batch, memory-efficient)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip()


def quadratic_bytes(res, batch, memory_efficient):
    """The unfused mid-block attention's L^2 buffers at their largest: S fp32 + P fp16 for the batch in the forward,
    or the saved P plus one image's dP fp32 and dS fp16 in the backward.  The d=512 flash path has none."""
    if memory_efficient:
        return 0
    L = (res // 8) ** 2
    return max(6 * batch, 2 * batch + 6) * L * ((L + 7) // 8 * 8)


class _SegmentFn(torch.autograd.Function):
    """One decoder segment checkpointed as a whole: the forward walks its blocks on their inference forward and keeps
    the input; the backward re-runs their training forward from it (with the producer extras `_cs` / `_h16` the first
    block reads re-attached) and back-propagates through the re-run."""

    @staticmethod
    def forward(ctx, walk, x):
        ctx.walk, ctx.x = walk, x
        return walk(x, False)

    @staticmethod
    def backward(ctx, dout):
        x = ctx.x.detach().requires_grad_(True)
        for k in ("_cs", "_h16"):
            if getattr(ctx.x, k, None) is not None:
                setattr(x, k, getattr(ctx.x, k))
        with torch.enable_grad():
            out = ctx.walk(x, True)
        torch.autograd.backward(out, dout)
        return None, x.grad


def segment_forward(decoder):
    """Decoder.forward with diffusers' segments checkpointed (training only)."""
    def walk(seg, x, train):
        if train:
            resnet = lambda r, h, f16_copy=False: ab.resnet(r, h, f16_copy=f16_copy)               # noqa: E731
            attention, upsample = ab.vae_attention, ab.upsample
        else:
            resnet = lambda r, h, f16_copy=False: r.run(h, None, None, F32, f16_copy)              # noqa: E731
            attention = lambda m, h: m.run(h, F32)                                                  # noqa: E731
            upsample = lambda m, h: m.run(h, None, F32)                                             # noqa: E731
        if seg is decoder.mid_block:
            return seg.run(x, resnet, attention)
        for i, r in enumerate(seg.resnets):
            x = resnet(r, x, i == len(seg.resnets) - 1 and seg.upsamplers is not None)
        return x if seg.upsamplers is None else upsample(seg.upsamplers[0], x)

    def forward(z):
        h = ab.conv_in(decoder._in, z)
        for seg in (decoder.mid_block, *decoder.up_blocks):
            # apply() hands back the tensor walk() made, with its producer extras for the next segment
            h = _SegmentFn.apply(lambda x, train, seg=seg: walk(seg, x, train), h)
        return ab.conv_out(decoder._out, h)
    return forward


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "vae_checkpoint_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_checkpoint_timing.py needs a GPU")
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss
    res_all = dict(card=card(), shapes=[])
    print(json.dumps(res_all), flush=True)
    torch.manual_seed(1234)
    with torch.device("cuda"):
        unet = B200UNet2DConditionModel()
        vae = B200AutoencoderKL()
    vae.eval().requires_grad_(False)
    unet.train().requires_grad_(True)
    unet.enable_gradient_checkpointing()
    sched = DDIMScheduler()
    dec = vae.decoder

    def set_mode(mode):
        dec.__dict__.pop("forward", None)
        (vae.enable_gradient_checkpointing if mode == "on" else vae.disable_gradient_checkpointing)()
        if mode == "segment":
            dec.forward = segment_forward(dec)

    peak_768 = {}
    for res, batch, me in SHAPES:
        (vae.enable_xformers_memory_efficient_attention if me else vae.disable_xformers_memory_efficient_attention)()
        modes = ["off", "on"] + (["segment"] if (res, batch) == (768, 2) else [])
        r = dict(res=res, batch=batch, memory_efficient_attention=me)
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        avail = free + torch.cuda.memory_reserved()
        run = []
        for m in modes:
            if m in peak_768:
                px = res * res * batch / (768 * 768 * 2)
                need = 1.1 * ((peak_768[m] - quadratic_bytes(768, 2, False)) * px + quadratic_bytes(res, batch, me))
                r[f"need_gib_{m}"] = need / GB
                if need > avail:
                    r[f"skipped_{m}"] = f"estimated {need / GB:.1f} GiB > {avail / GB:.1f} GiB available"
                    continue
            run.append(m)
        g = torch.Generator(device="cuda").manual_seed(3)
        data = (torch.rand(batch, 3, res, res, device="cuda", generator=g) * 2 - 1,
                torch.rand(batch, 1, res, res, device="cuda", generator=g) * 9.9 + 0.1,
                torch.rand(batch, 1, res, res, device="cuda", generator=g) > 0.001,
                torch.randn(1, 77, 1024, device="cuda", generator=g) * 0.5)

        def step():
            (e2e_ft_loss(unet, vae, sched, *data, "depth")[0] * LOSS_SCALE).backward()
            unet.zero_grad(set_to_none=True)

        ms = {m: [] for m in run}
        peak = {m: 0 for m in run}
        for m in run:                                      # warm-up, one step per mode
            set_mode(m)
            step()
        for _ in range(a.rounds):
            for m in run:
                set_mode(m)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e0.record()
                for _ in range(a.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                ms[m].append(e0.elapsed_time(e1) / a.steps)
                peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        set_mode("off")
        for m in run:
            r[m] = dict(ms_min=min(ms[m]), ms_rounds=ms[m], peak_gib=peak[m] / GB)
            if (res, batch) == (768, 2):
                peak_768[m] = peak[m]
        if "off" in run and "on" in run:
            r["recompute_ms"] = r["on"]["ms_min"] - r["off"]["ms_min"]
            r["recompute_share"] = r["recompute_ms"] / r["off"]["ms_min"]
        print(json.dumps(r), flush=True)
        res_all["shapes"].append(r)
        del data
    vae.disable_xformers_memory_efficient_attention()
    res_all["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res_all, f, indent=1)
    print(json.dumps({k: res_all[k] for k in ("card", "card_after")}), flush=True)


if __name__ == "__main__":
    main()
