"""Time GeoWizard's SD-1-shaped UNet (8 heads of width 40 / 80 / 160, 1x1-conv projections, context 768) on the GPU:
the flash kernel at the SD-1 GeoWizard shapes beside the head-width-64 kernel at the same channel count (equal FLOPs),
DepthNormalEstimationPipeline inference at SD-1 and SD-2 widths (alternating), and the E2E fine-tuning micro-step at
SD-1 widths.  Prints the card's name, power limit and maximum SM clock with the numbers.

    python tools/geowizard_sd1_timing.py --out /tmp/geowizard_sd1_timing.json

Times are CUDA events around work that ends in a device synchronise; kernel times average --kernel-reps launches after
warm-up.  Peak memory is torch's max_memory_allocated over each leg.  Weights are seeded random (the timing does not
depend on their values)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP16_DENSE = 989e12          # H100 SXM data sheet, dense fp16 / bf16 tensor core rate


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip()


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attention_leg(reps):
    from diffusion_e2e_ft_b200 import ops
    out = []
    # (level, channels, UNet batch, tokens): GeoWizard at 768^2 = latent 96^2, batch 8 = 4 images x (depth, normal)
    for level, C, B, L in ((0, 320, 8, 9216), (1, 640, 8, 2304), (2, 1280, 8, 576)):
        qkv = torch.randn(B, L, 3 * C, device="cuda", dtype=torch.float16)
        for D in (C // 8, 64):
            heads = C // D
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            o = torch.empty(B, L, C, device="cuda", dtype=torch.float16)
            fn = lambda: ops.attention(q, k, v, heads, D ** -0.5, kv_segments=2, out=o)
            for _ in range(3):
                fn()
            ms = events_ms(fn, reps)
            flops = 4 * B * heads * L * (2 * L) * D
            r = dict(level=level, C=C, heads=heads, head_dim=D, B=B, Lq=L, Lk=2 * L, ms=ms,
                     tflops=flops / ms / 1e9, share_of_989=flops / ms / 1e-3 / PEAK_FP16_DENSE)
            print(json.dumps(r), flush=True)
            out.append(r)
        del qkv
    return out


def build_unet(sd1, **kw):
    from diffusion_e2e_ft_b200 import B200UNet2DConditionModel
    cfg = dict(class_embed_type="projection", projection_class_embeddings_input_dim=10, cross_attention_dim=768,
               joint_attention=True, **kw)
    if sd1:
        cfg.update(attention_head_dim=8, use_linear_projection=False)
    return B200UNet2DConditionModel(**cfg)


@torch.no_grad()
def inference_leg(images, res, rounds):
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, DDIMScheduler, DepthNormalEstimationPipeline
    torch.manual_seed(1234)
    pipes = {}
    with torch.device("cuda"):
        vae = B200AutoencoderKL()
        for name, sd1 in (("sd1", True), ("sd2", False)):
            pipes[name] = DepthNormalEstimationPipeline(build_unet(sd1).half().eval(), vae, DDIMScheduler())
    vae.half().eval()
    rgb = torch.rand(images, 3, res, res, device="cuda") * 2 - 1
    emb = (torch.randn(images, 1, 768, device="cuda") * 0.5).half()
    run = lambda p: p.single_infer(rgb, 1, "indoor", noise="zeros", img_embed=emb)
    res_ = {n: dict(ms=[]) for n in pipes}
    for p in pipes.values():
        run(p)
        run(p)
    for _ in range(rounds):                                      # alternate the two widths
        for n, p in pipes.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            ms = events_ms(lambda: run(p), 1)
            res_[n]["ms"].append(ms)
            res_[n]["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    for n, r in res_.items():
        r["images_per_s"] = images / (min(r["ms"]) / 1e3)
        print(json.dumps({f"inference_{n}": r}), flush=True)
    return res_


def training_leg(batch, res, steps):
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss_geowizard
    torch.manual_seed(1234)
    with torch.device("cuda"):
        unet = build_unet(True)
        vae = B200AutoencoderKL()
    vae.eval().requires_grad_(False)
    unet.train().requires_grad_(True)
    unet.enable_gradient_checkpointing()
    g = torch.Generator(device="cuda").manual_seed(3)
    rgb = torch.rand(batch, 3, res, res, device="cuda", generator=g) * 2 - 1
    depth_gt = torch.rand(batch, 1, res, res, device="cuda", generator=g) * 9.9 + 0.1
    normals = torch.nn.functional.normalize(torch.randn(batch, 3, res, res, device="cuda", generator=g), dim=1)
    mask = torch.rand(batch, 1, res, res, device="cuda", generator=g) > 0.001
    emb = torch.randn(batch, 1, 768, device="cuda", generator=g) * 0.5
    sched = DDIMScheduler()

    def step():
        loss, _, _ = e2e_ft_loss_geowizard(unet, vae, sched, rgb, depth_gt, normals, mask, emb)
        (loss * LOSS_SCALE).backward()
        unet.zero_grad(set_to_none=True)

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = [events_ms(step, 1) for _ in range(steps)]
    r = dict(batch=batch, res=res, ms=times, ms_min=min(times), peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(json.dumps({"e2e_ft_step_sd1": r}), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--train-batch", type=int, default=2)
    ap.add_argument("--train-steps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "geowizard_sd1_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU timing")
    out = dict(card=card())
    print(json.dumps(out), flush=True)
    out["attention"] = attention_leg(a.kernel_reps)
    out["inference"] = inference_leg(a.images, a.res, a.rounds)
    torch.cuda.empty_cache()
    try:
        out["training"] = training_leg(a.train_batch, a.res, a.train_steps)
    except torch.cuda.OutOfMemoryError as e:
        out["training"] = dict(error=f"out of memory: {e}"[:400])
        print(json.dumps({"e2e_ft_step_sd1": out["training"]}), flush=True)
    out["card_after"] = card()
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
