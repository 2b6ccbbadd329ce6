"""Time the backward of the VAE mid-block attention (one head of width 512): the fused flash kernels
(csrc/attention_d512_bwd.cu: delta, then dQ, dK, dV with P recomputed from the saved log-sum-exp) against the unfused
path that training ran before (autograd_blocks._VAEAttentionFn on the GEMMs: per image dP = dO V^T in fp32, the row
softmax backward to fp16 dS, then dQ = dS K, dK = dS^T Q, dV = P^T dO from the P [B, L, Lp] its forward saved).
Both legs start from what their forward saved and produce dQ, dK, dV; they are alternated in one process.  Reports
time, TFLOP/s from shapes (5 products of 2 L^2 512 per image), peak memory growth and the largest difference between
the two paths' gradients, then Marigold E2E micro-steps (bs 2, 768 x 768) with and without
`vae.enable_xformers_memory_efficient_attention()`.  Reads the card name and power limit in the same run.

    python tools/vae_attention_bwd_timing.py --reps 10 --out /tmp/vae_attention_bwd_timing.json
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

from diffusion_e2e_ft_b200 import ops  # noqa: E402
from diffusion_e2e_ft_b200.ops import F16, F32  # noqa: E402

PEAK_FP16_DENSE = 989e12          # H100 SXM data sheet, dense fp16
C = 512


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip()


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


def unfused_forward_p(q, k):
    """The P [B, L, Lp] fp16 the unfused forward saves (S = Q K^T in fp32, then the row softmax)."""
    B, L = q.shape[:2]
    Lp = (L + 7) // 8 * 8
    s_buf = torch.empty((B, L, Lp), dtype=F32, device=q.device)
    ops.linear(q, k, out=s_buf[:, :, :L])
    return ops.softmax_rows(s_buf, C ** -0.5, cols=L)


def unfused_bwd(q, k, v, do, p_buf):
    """The per-image loop of autograd_blocks._VAEAttentionFn._dhn_unfused, up to dQ, dK, dV."""
    B, L = q.shape[:2]
    Lp = p_buf.shape[2]
    dq, dk, dv = (torch.empty((B, L, C), dtype=F16, device=q.device) for _ in range(3))
    for b in range(B):
        dp = torch.zeros((L, Lp), dtype=F32, device=q.device)
        ops.linear(do[b], v[b], out=dp[:, :L], out_dtype=F32)
        ds = ops.softmax_bwd_rows(p_buf[b], dp, C ** -0.5, cols=L)
        del dp
        ops.linear(ds[:, :L], k[b], out=dq[b], w_t=True)
        ops.linear(ds[:, :L], q[b], out=dk[b], a_t=True, w_t=True)
        ops.linear(p_buf[b][:, :L], do[b], out=dv[b], a_t=True, w_t=True)
    return dq, dk, dv


def fused_bwd(q, k, v, do, o, lse):
    delta = ops.rowdot_d512(do, o)
    outs = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    return ops.attention_d512_bwd(q, k, v, do, lse, delta, *outs, C ** -0.5)


# (B, L): 768^2 bs 2 (Marigold), bs 4 (GeoWizard decodes depth and normal), 1024^2, 1536^2; 2048^2 fused only
SHAPES = [(2, 9216, True), (4, 9216, True), (1, 16384, True), (1, 36864, True), (1, 65536, False)]


def kernel_leg(reps):
    out = []
    for B, L, with_unfused in SHAPES:
        g = torch.Generator(device="cpu").manual_seed(L + B)
        qkv = (torch.randn(B, L, 3 * C, generator=g) * 0.5).half().cuda()
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        do = torch.randn(B, L, C, generator=g).half().cuda()
        o, lse = ops.attention_d512(q, k, v, C ** -0.5, want_lse=True)
        new = lambda: fused_bwd(q, k, v, do, o, lse)                     # noqa: E731
        mem_new, r_new = peak_growth(new)
        r = dict(B=B, L=L)
        useful = 5 * 2 * B * L * L * C
        if with_unfused:
            p_buf = unfused_forward_p(q, k)
            old = lambda: unfused_bwd(q, k, v, do, p_buf)                # noqa: E731
            mem_old, r_old = peak_growth(old)
            r["max_rel_diff"] = max(((a.float() - b.float()).abs().max() / b.float().abs().max()).item()
                                    for a, b in zip(r_new, r_old))
            del r_old
            ms = {"unfused": [], "fused": []}
            old(), new()
            for _ in range(3):                                           # alternate the two paths
                ms["unfused"].append(timed(old, reps))
                ms["fused"].append(timed(new, reps))
            r.update(unfused_ms=min(ms["unfused"]), unfused_tflops=useful / min(ms["unfused"]) / 1e9,
                     peak_growth_mb_unfused=mem_old, saved_p_mb=p_buf.numel() * 2 / 1e6)
            del p_buf
        else:
            new()
            ms = {"fused": [timed(new, reps) for _ in range(3)]}
        r.update(fused_ms=min(ms["fused"]), fused_tflops=useful / min(ms["fused"]) / 1e9,
                 fused_share_of_989=useful / (min(ms["fused"]) / 1e3) / PEAK_FP16_DENSE,
                 fused_forward_lse_ms=timed(lambda: ops.attention_d512(q, k, v, C ** -0.5, want_lse=True), reps),
                 peak_growth_mb_fused=mem_new, spread=ms)
        print(json.dumps(r), flush=True)
        out.append(r)
        del qkv, q, k, v, do, o, lse, r_new
        torch.cuda.empty_cache()
    return out


def e2e_leg(steps, res):
    """Marigold micro-steps (forward, loss, backward; no optimizer step), unfused and memory-efficient alternated."""
    from diffusion_e2e_ft_b200 import B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss
    torch.manual_seed(1234)
    with torch.device("cuda"):
        unet = B200UNet2DConditionModel()
        vae = B200AutoencoderKL()
    vae.eval().requires_grad_(False)
    unet.train().requires_grad_(True)
    g = torch.Generator(device="cuda").manual_seed(3)
    B = 2
    rgb = torch.rand(B, 3, res, res, device="cuda", generator=g) * 2 - 1
    depth = torch.rand(B, 1, res, res, device="cuda", generator=g) * 9.9 + 0.1
    mask = torch.rand(B, 1, res, res, device="cuda", generator=g) > 0.001
    ete = torch.randn(1, 77, 1024, device="cuda", generator=g) * 0.5
    sched = DDIMScheduler()

    def step():
        (e2e_ft_loss(unet, vae, sched, rgb, depth, mask, ete, "depth")[0] * LOSS_SCALE).backward()
        unet.zero_grad(set_to_none=True)

    paths = (("unfused", vae.disable_xformers_memory_efficient_attention),
             ("memory_efficient", vae.enable_xformers_memory_efficient_attention))
    r = {p: dict(ms=[]) for p, _ in paths}
    for _, switch in paths:
        switch()
        step()
    for _ in range(steps):
        for p, switch in paths:
            switch()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            r[p]["ms"].append(timed(step, 1))
            r[p]["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    vae.disable_xformers_memory_efficient_attention()
    for p in r.values():
        p["ms_min"] = min(p["ms"])
    print(json.dumps({"marigold_e2e": r}), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "vae_attention_bwd_timing.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_attention_bwd_timing.py needs a GPU")
    res = dict(card=card())
    print(json.dumps(res), flush=True)
    res["kernels"] = kernel_leg(a.reps)
    if not a.no_e2e:
        res["e2e"] = e2e_leg(a.e2e_steps, a.res)
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("card", "card_after")}), flush=True)


if __name__ == "__main__":
    main()
