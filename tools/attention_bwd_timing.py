"""Time the attention backward: the fused flash kernels (csrc/attention_bwd.cu) against the per-image GEMM composition
with stored P and dS that they replaced (backward._attention_bwd_gemm; for joint attention the depth / normal pairs
concatenated and run one pair at a time, as the UNet block did before), alternated in one process at the UNet's shapes.  Reports kernel
time, TFLOP/s from shapes (5 products of 2 T Tk D per head), peak memory growth, the largest difference between the
two paths' gradients, and E2E fine-tuning micro-steps (Marigold SD-2 and GeoWizard SD-1, bs 2, 768 x 768) with either
backward.  Reads the card name and power limit in the same run.

    python tools/attention_bwd_timing.py --reps 20 --out /tmp/attention_bwd_timing.json
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

from diffusion_e2e_ft_b200 import backward as bw  # noqa: E402
from diffusion_e2e_ft_b200 import ops  # noqa: E402

PEAK_FP16_DENSE = 989e12          # H100 SXM data sheet, dense fp16
HBM = 3.35e12                     # H100 SXM data sheet, HBM3 bytes/s
FUSED = bw.attention_bwd          # the package's entry point (the e2e leg swaps bw.attention_bwd)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip()


def gemm_path(q, k, v, do, heads, scale, outs=None, kv_segments=1):
    """The backward before the fused kernels: backward._attention_bwd_gemm, the per-image GEMM composition with stored
    P and dS (joint pairs concatenated into one 2L x 2L problem), after the same forward re-run and rowdot."""
    C = q.shape[-1]
    dq, dk, dv = outs if outs is not None else (torch.empty_like(q), torch.empty_like(k), torch.empty_like(v))
    if k.shape[1] == 1 and kv_segments == 1:
        return FUSED(q, k, v, do, heads, scale, outs=(dq, dk, dv))           # the exact one-key form
    o, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)
    delta = ops.rowdot_heads_d(do, o, heads, C // heads)
    bw._attention_bwd_gemm(q, k, v, do, heads, scale, lse, delta, dq, dk, dv, kv_segments)
    return dq, dk, dv


def fused_path(q, k, v, do, heads, scale, kv_segments=1):
    C = q.shape[-1]
    o, lse = ops.attention(q, k, v, heads, scale, kv_segments=kv_segments, want_lse=True)
    delta = ops.rowdot_heads_d(do, o, heads, C // heads)
    outs = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    return ops.attention_bwd(q, k, v, do, lse, delta, *outs, heads, scale, kv_segments)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def peak_growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    r = fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e6, r


# (name, B, heads, D, T, Tk, kv_segments): SD-2 levels 0-3 at 768^2 (latent 96^2), B = 2; SD-1 joint pairs (8 heads)
SHAPES = [("sd2_l0_self", 2, 5, 64, 9216, 9216, 1), ("sd2_l1_self", 2, 10, 64, 2304, 2304, 1),
          ("sd2_l2_self", 2, 20, 64, 576, 576, 1), ("sd2_l3_self", 2, 20, 64, 144, 144, 1),
          ("sd2_l0_cross77", 2, 5, 64, 9216, 77, 1), ("sd2_l1_cross77", 2, 10, 64, 2304, 77, 1),
          ("sd2_l3_cross77", 2, 20, 64, 144, 77, 1), ("sd2_l0_cross2", 2, 5, 64, 9216, 2, 1),
          ("sd2_l0_self_640x480", 2, 5, 64, 4800, 4800, 1),
          ("sd1_joint_l0_768", 2, 8, 40, 9216, 9216, 2), ("sd1_joint_l1_768", 2, 8, 80, 2304, 2304, 2),
          ("sd1_joint_l2_768", 2, 8, 160, 576, 576, 2), ("sd1_joint_l0_480x640", 2, 8, 40, 4800, 4800, 2),
          ("sd1_l0_cross77", 2, 8, 40, 9216, 77, 1)]


def kernel_leg(reps, only=None):
    out = []
    for name, B, heads, D, T, Tk, kv in SHAPES:
        if only and name not in only:
            continue
        C = heads * D
        g = torch.Generator(device="cpu").manual_seed(T + Tk + D)
        q = torch.randn(B, T, C, generator=g).half().cuda()
        k, v = ((torch.randn(B, Tk, C, generator=g) * 0.5).half().cuda() for _ in range(2))
        do = torch.randn(B, T, C, generator=g).half().cuda()
        scale = D ** -0.5
        old = lambda: gemm_path(q, k, v, do, heads, scale, kv_segments=kv)
        new = lambda: fused_path(q, k, v, do, heads, scale, kv)
        mem_old, r_old = peak_growth(old)
        mem_new, r_new = peak_growth(new)
        diff = max(((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30)).item()
                   for a, b in zip(r_new, r_old))
        del r_old, r_new
        for _ in range(2):
            old(), new()
        ms = {"gemm": [], "fused": []}
        for _ in range(3):                                   # alternate the two paths
            ms["gemm"].append(timed(old, reps))
            ms["fused"].append(timed(new, reps))
        # the forward re-run and rowdot are common to both: time them alone so the backward proper can be told apart
        fwd = timed(lambda: ops.rowdot_heads_d(do, ops.attention(q, k, v, heads, scale, kv_segments=kv), heads, D),
                    reps)
        useful = 5 * 2 * B * heads * T * (Tk * kv) * D
        t_gemm, t_fused = min(ms["gemm"]), min(ms["fused"])
        pds_bytes = 2 * 2 * B * heads * T * Tk * kv
        r = dict(name=name, B=B, heads=heads, D=D, T=T, Tk=Tk, kv_segments=kv, gemm_ms=t_gemm, fused_ms=t_fused,
                 forward_and_rowdot_ms=fwd, fused_bwd_only_ms=t_fused - fwd, gemm_bwd_only_ms=t_gemm - fwd,
                 fused_bwd_tflops=useful / max(t_fused - fwd, 1e-6) / 1e9,
                 fused_share_of_989=useful / ((t_fused - fwd) / 1e3) / PEAK_FP16_DENSE,
                 gemm_hbm_floor_ms=(pds_bytes + 4 * pds_bytes) / HBM * 1e3,
                 fused_tensor_floor_ms=7 / 5 * useful / PEAK_FP16_DENSE * 1e3,
                 peak_growth_mb_gemm=mem_old, peak_growth_mb_fused=mem_new, max_rel_diff=diff, spread=ms)
        print(json.dumps(r), flush=True)
        out.append(r)
        del q, k, v, do
        torch.cuda.empty_cache()
    return out


def e2e_leg(steps, res):
    """Micro-steps (forward, loss, backward; no optimizer step) with either attention backward, alternated."""
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss, e2e_ft_loss_geowizard
    fused = FUSED
    out = {}
    for name in ("marigold_sd2", "geowizard_sd1"):
        torch.manual_seed(1234)
        with torch.device("cuda"):
            if name == "marigold_sd2":
                unet = B200UNet2DConditionModel()
            else:
                unet = B200UNet2DConditionModel(class_embed_type="projection", projection_class_embeddings_input_dim=10,
                                                cross_attention_dim=768, joint_attention=True, attention_head_dim=8,
                                                use_linear_projection=False)
                unet.enable_gradient_checkpointing()
            vae = B200AutoencoderKL()
        vae.eval().requires_grad_(False)
        unet.train().requires_grad_(True)
        g = torch.Generator(device="cuda").manual_seed(3)
        B = 2
        rgb = torch.rand(B, 3, res, res, device="cuda", generator=g) * 2 - 1
        depth = torch.rand(B, 1, res, res, device="cuda", generator=g) * 9.9 + 0.1
        mask = torch.rand(B, 1, res, res, device="cuda", generator=g) > 0.001
        sched = DDIMScheduler()
        if name == "marigold_sd2":
            ete = torch.randn(1, 77, 1024, device="cuda", generator=g) * 0.5
            loss_fn = lambda: e2e_ft_loss(unet, vae, sched, rgb, depth, mask, ete, "depth")[0]
        else:
            normals = torch.nn.functional.normalize(torch.randn(B, 3, res, res, device="cuda", generator=g), dim=1)
            emb = torch.randn(B, 1, 768, device="cuda", generator=g) * 0.5
            loss_fn = lambda: e2e_ft_loss_geowizard(unet, vae, sched, rgb, depth, normals, mask, emb)[0]

        def step():
            (loss_fn() * LOSS_SCALE).backward()
            unet.zero_grad(set_to_none=True)

        r = {"gemm": dict(ms=[]), "fused": dict(ms=[])}
        for path, fn in (("gemm", gemm_path), ("fused", fused)):
            bw.attention_bwd = fn
            step()
        for _ in range(steps):
            for path, fn in (("gemm", gemm_path), ("fused", fused)):
                bw.attention_bwd = fn
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                r[path]["ms"].append(timed(step, 1))
                r[path]["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        bw.attention_bwd = fused
        for p in r.values():
            p["ms_min"] = min(p["ms"])
        out[name] = r
        print(json.dumps({name: r}), flush=True)
        del unet, vae
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--only", nargs="*", default=None, help="kernel-leg shape names")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "attention_bwd_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attention_bwd_timing.py needs a GPU")
    res = dict(card=card())
    print(json.dumps(res), flush=True)
    res["kernels"] = kernel_leg(a.reps, a.only)
    if not a.no_e2e:
        res["e2e"] = e2e_leg(a.e2e_steps, a.res)
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
