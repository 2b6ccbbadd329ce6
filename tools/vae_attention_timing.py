"""Time the VAE mid-block attention (one head, d = 512) on both paths, and one native-resolution 4K pipeline call.

    python tools/vae_attention_timing.py [--out FILE]

Per (B, L): CUDA-event time of one attention core call, Q, K, V (views of one fused [B, L, 1536] projection) -> O:
  fused    ops.attention_d512 (flash kernel, no L x L buffer)
  unfused  S = Q K^T (fp32 GEMM) -> row softmax (fp16 P) -> O = P V on the GEMM, as VAEAttention runs it by default
           (V^T is prepared outside the timed window; its swapped GEMM is part of the projection, not of the core)
at (8, 9216) (768^2 bs 8), (1, 16384) (1024^2), (1, 32400) (1920x1080), and fused only at (1, 129600) (3840x2160,
where the unfused path cannot index its scores).  Then wall time and peak allocation of one MarigoldPipeline call on a
3840x2160 image with processing_res=0 (random-init SD-2 widths, 1 step, ensemble 1), after one warm-up call.
Device name, power limit and SM clocks are read in the same process and reported with the numbers; no device setting
is changed.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _gpu_info():
    info = dict(name=torch.cuda.get_device_name())
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit, sm_clock, max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return dict(median_ms=ts[len(ts) // 2], min_ms=ts[0], max_ms=ts[-1], reps=reps)


def time_attention(B, L, unfused=True):
    from diffusion_e2e_ft_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = (torch.randn(B, L, 1536, device="cuda", generator=g) * 1.5).half()
    q, k, v = qkv[..., :512], qkv[..., 512:1024], qkv[..., 1024:]
    scale = 512 ** -0.5
    flops = 4 * B * L * L * 512
    reps, warmup = (3, 1) if L > 100000 else (10, 2)
    out = torch.empty((B, L, 512), dtype=torch.float16, device="cuda")
    res = dict(B=B, L=L, flops=flops)
    res["fused"] = _time(lambda: ops.attention_d512(q, k, v, scale, out=out), reps, warmup)
    res["fused"]["tflops"] = flops / res["fused"]["median_ms"] / 1e9
    if unfused:
        Lp = (L + 7) // 8 * 8
        vt_buf = torch.zeros((B, 512, Lp), dtype=torch.float16, device="cuda")
        vt_buf[:, :, :L] = v.transpose(1, 2)
        s_buf = torch.empty((B, L, Lp), dtype=torch.float32, device="cuda")

        def run():
            ops.linear(q, k, out=s_buf[:, :, :L])
            p_buf = ops.softmax_rows(s_buf, scale, cols=L)
            return ops.linear(p_buf[:, :, :L], vt_buf[:, :, :L])
        ref = run()
        res["fused_vs_unfused_rel_l2"] = ((out.float() - ref.float()).norm() / ref.float().norm()).item()
        del ref
        res["unfused"] = _time(run, reps, warmup)
        res["unfused"]["tflops"] = flops / res["unfused"]["median_ms"] / 1e9
        del s_buf, vt_buf
    torch.cuda.empty_cache()
    return res


@torch.no_grad()
def time_pipeline_4k():
    from oracle.unet import UNet2DConditionRef, UNetConfig, seeded_init
    from oracle.vae import AutoencoderKLRef, VAEConfig
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    import engine_checks as EC
    uref = seeded_init(UNet2DConditionRef(UNetConfig()), seed=4321).eval()
    vref = seeded_init(AutoencoderKLRef(VAEConfig()), seed=99).eval()
    unet, vae = EC.engine_from_oracle(uref, vref, "cuda")
    ete = (torch.randn(1, 2, 1024, generator=torch.Generator().manual_seed(7)) * 0.5).cuda()
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=ete)
    pipe.use_cuda_graph = False
    img = torch.randint(0, 256, (3, 2160, 3840), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))

    def call():
        return pipe(img, denoising_steps=1, ensemble_size=1, processing_res=0, noise="zeros",
                    show_progress_bar=False).depth_np
    call()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    d = call()                                   # ends in a device-to-host copy of the depth map: synchronised
    wall = time.perf_counter() - t0
    return dict(input="3840x2160 uint8", processing_res=0, wall_s=wall,
                max_memory_allocated_gb=torch.cuda.max_memory_allocated() / 1024 ** 3,
                depth_shape=list(d.shape), depth_finite=bool((d == d).all()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON here")
    ap.add_argument("--no-pipeline", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_attention_timing needs a CUDA device")
    res = dict(gpu=_gpu_info(), attention=[])
    for B, L in ((8, 9216), (1, 16384), (1, 32400)):
        res["attention"].append(time_attention(B, L))
    res["attention"].append(time_attention(1, 129600, unfused=False))
    if not a.no_pipeline:
        res["pipeline_4k"] = time_pipeline_4k()
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
