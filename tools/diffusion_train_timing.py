"""Time GeoWizard's diffusion-objective micro-step (train_depth_normal.py:600-717, `training.diffusion_loss_geowizard`)
against its E2E fine-tuning micro-step (`training.e2e_ft_loss_geowizard`) on the same inputs, at SD-2 widths
(GeoWizard-shaped UNet, seeded weights), and the three kernels the diffusion objective added (ABI 10) against the HBM
bandwidth of the data sheet.  Prints the device name and power limit of the card it ran on.

    python tools/diffusion_train_timing.py --batch 2 --res 768 --steps 3 --warmup 1 --out /tmp/diffusion_train.json

Micro-step = forward + loss + backward (gradient checkpointing on for both), no optimizer step; timed with CUDA events
around work that ends in a device synchronise.  Peak memory is torch's max_memory_allocated over each leg."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or None
    except Exception:
        return None


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--kernel-reps", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "diffusion_train_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU timing")
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler, ops
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, diffusion_loss_geowizard, e2e_ft_loss_geowizard
    dev = "cuda:0"
    out = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), batch=a.batch, res=a.res)
    print(json.dumps(dict(device=out["device"], power_limit=out["power_limit"])), flush=True)
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = B200UNet2DConditionModel(class_embed_type="projection", projection_class_embeddings_input_dim=10,
                                        cross_attention_dim=768, joint_attention=True)
        vae = B200AutoencoderKL()
    vae.eval().requires_grad_(False)
    unet.train().requires_grad_(True)
    unet.enable_gradient_checkpointing()
    n_params = sum(p.numel() for p in unet.parameters())
    g = torch.Generator(device=dev).manual_seed(3)
    B, H = a.batch, a.res
    rgb = torch.rand(B, 3, H, H, device=dev, generator=g) * 2 - 1
    depth_gt = torch.rand(B, 1, H, H, device=dev, generator=g) * 9.9 + 0.1
    depth = (torch.rand(B, 1, H, H, device=dev, generator=g) * 2 - 1).expand(-1, 3, -1, -1).contiguous()
    normals = torch.nn.functional.normalize(torch.randn(B, 3, H, H, device=dev, generator=g), dim=1)
    mask = torch.rand(B, 1, H, H, device=dev, generator=g) > 0.001
    emb = torch.randn(B, 1, 768, device=dev, generator=g) * 0.5
    sched = DDIMScheduler()
    gen = torch.Generator(device=dev).manual_seed(4)

    def diffusion():
        loss, _, _ = diffusion_loss_geowizard(unet, vae, sched, rgb, depth, normals, mask, emb, generator=gen)
        (loss * LOSS_SCALE).backward()
        return loss

    def e2e():
        loss, _, _ = e2e_ft_loss_geowizard(unet, vae, sched, rgb, depth_gt, normals, mask, emb)
        (loss * LOSS_SCALE).backward()
        return loss

    for name, fn in (("diffusion_step", diffusion), ("e2e_ft_step", e2e)):
        for _ in range(a.warmup):
            fn()
            unet.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        times, losses = [], []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss = fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
            losses.append(loss.item())
            unet.zero_grad(set_to_none=True)
        out[name] = dict(ms=times, ms_min=min(times), loss=losses,
                         peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
        print(json.dumps({name: out[name]}), flush=True)
    out["diffusion_over_e2e"] = out["diffusion_step"]["ms_min"] / out["e2e_ft_step"]["ms_min"]
    del unet, vae
    torch.cuda.empty_cache()

    # ---- the ABI-10 kernels at the shapes of this micro-step; bytes = what each kernel must move
    h = H // 8
    CHW = 4 * h * h
    rgb_l = torch.randn(B, 4, h, h, device=dev)
    x0 = torch.randn(2 * B, 4, h, h, device=dev)
    noise = torch.randn(2 * B, 4, h, h, device=dev)
    t = torch.randint(0, 1000, (B,)).repeat(2)
    t_dev, ac = t.to(dev), sched.alphas_cumprod.to(dev)
    kern = {}
    ms = events_ms(lambda: ops.diffusion_inputs(rgb_l, x0, noise, t_dev, ac, "v_prediction", timesteps_host=t),
                   a.kernel_reps)
    kern["diffusion_inputs"] = (ms, 4 * 2 * B * CHW * 6)            # rgb + x0 + noise in, 2C unet_in + target out
    pred = torch.randn(2 * B, 4, h, h, device=dev)
    target = torch.randn(2 * B, 4, h, h, device=dev)
    res = {}
    kern["masked_latent_mse"] = (events_ms(lambda: res.update(r=ops.masked_latent_mse(pred, target, mask)),
                                           a.kernel_reps), B * H * H + 2 * 4 * 2 * B * CHW + B * h * h)
    _, lm, ws = res["r"]
    go = torch.ones((), device=dev)
    kern["masked_latent_mse_bwd"] = (events_ms(lambda: ops.masked_latent_mse_bwd(pred, target, lm, ws, go), a.kernel_reps),
                                     3 * 4 * 2 * B * CHW + B * h * h)
    n = (n_params + 3) // 4 * 4
    ema = torch.randn(n, device=dev)
    param = torch.randn(n, device=dev)
    kern["ema_update"] = (events_ms(lambda: ops.ema_update(ema, param, 1e-4), max(5, a.kernel_reps // 5)), 12 * n)
    out["kernels"] = {}
    for k, (ms, nbytes) in kern.items():
        out["kernels"][k] = dict(ms=ms, bytes=nbytes, tb_per_s=nbytes / (ms * 1e-3) / 1e12,
                                 of_hbm_peak=nbytes / (ms * 1e-3) / HBM_BYTES_PER_S)
    out["unet_params"] = n_params
    print(json.dumps(out["kernels"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(device=out["device"], power_limit=out["power_limit"],
                          diffusion_ms=out["diffusion_step"]["ms_min"], e2e_ms=out["e2e_ft_step"]["ms_min"],
                          diffusion_peak_gib=out["diffusion_step"]["peak_gib"],
                          e2e_peak_gib=out["e2e_ft_step"]["peak_gib"])))


if __name__ == "__main__":
    main()
