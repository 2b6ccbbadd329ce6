"""Per-stage error budget of the UNet forward against the fp32 oracle (VERDICT r1 task 1b).

    python tools/error_budget.py [latent=24] > out/error_budget.txt

Full SD-2 widths, batch 1.  For every ResnetBlock2D / Transformer2DModel / Down/Upsample2D output: cumulative rel-L2
of the engine's activation against the oracle's.  Then attribution experiments on the same weights / inputs:
  exact_attention   the flash kernel replaced by an fp32 softmax attention on the same fp16 q/k/v (isolates the
                    kernel's internal rounding: fp16 P, ex2.approx)
  fp16_stream       residual stream in fp16 instead of fp32
  general_path      single-step specialisations off (flash cross-attention over 2 keys instead of the folded GEMMs)
  split_operands    every GEMM / conv activation operand carried as hi + lo fp16 halves (two MMAs per k-block):
                    removes the activation-rounding term, leaves the weight rounding
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import engine_checks as EC  # noqa: E402
import make_golden as MG  # noqa: E402
from diffusion_e2e_ft_b200 import modules as M, ops  # noqa: E402
from oracle.unet import UNet2DConditionRef, UNetConfig, seeded_init  # noqa: E402

DEV = "cuda:0"


def exact_attention(q, k, v, heads, scale, kv_segments=1, out=None):
    B, Lq, _ = q.shape
    def split(t):
        return t.float().reshape(t.shape[0], t.shape[1], heads, 64).permute(0, 2, 1, 3)
    qh, kh, vh = split(q), split(k), split(v)
    if kv_segments == 2:
        h = B // 2
        kh = torch.cat([torch.cat([kh[:h], kh[h:]], 2)] * 2, 0)
        vh = torch.cat([torch.cat([vh[:h], vh[h:]], 2)] * 2, 0)
    if kh.shape[0] == 1 and B > 1:
        kh, vh = kh.expand(B, -1, -1, -1), vh.expand(B, -1, -1, -1)
    o = torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh
    o = o.permute(0, 2, 1, 3).reshape(B, Lq, heads * 64).half()
    if out is not None:
        out.copy_(o)
        return out
    return o


def main():
    latent = int(sys.argv[1]) if len(sys.argv) > 1 else 24
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ref = seeded_init(UNet2DConditionRef(UNetConfig()), seed=4321).eval().to(DEV)
    x = MG.inputs(11, 1, 8, latent, latent).to(DEV)
    ctx = MG.inputs(12, 1, 2, 1024, scale=0.5).to(DEV)
    ref_out = {}
    for name, mod in ref.named_modules():
        if type(mod).__name__ in ("ResnetBlock2D", "Transformer2DModel", "Downsample2D", "Upsample2D"):
            mod.register_forward_hook(lambda m, i, o, name=name: ref_out.__setitem__(name, o.detach()))
    with torch.no_grad():
        want = ref(x, 999, ctx).sample

    def run(stream=torch.float32, spec=True, stages=False):
        eng, _ = EC.engine_from_oracle(ref.cpu(), None, DEV, stream)
        ref.to(DEV)
        eng.single_step_specialisations = spec
        eng_out = {}
        if stages:
            for name, mod in eng.named_modules():
                mod._dbg_name = name
            for cls in (M.ResnetBlock2D, M.Transformer2DModel, M.Downsample2D, M.Upsample2D):
                orig = cls.run
                def wrapped(self, *a, _orig=orig, **k):
                    o = _orig(self, *a, **k)
                    eng_out[self._dbg_name] = o.detach().float()
                    return o
                cls.run = wrapped
                cls._orig_run = orig
        with torch.no_grad():
            got = eng(x, 999, ctx.expand(1, -1, -1)).sample
        if stages:
            for cls in (M.ResnetBlock2D, M.Transformer2DModel, M.Downsample2D, M.Upsample2D):
                cls.run = cls._orig_run
        return got, eng_out

    got, eng_out = run(stages=True)
    print(f"# full-width UNet, latent {latent}x{latent}, batch 1, fp32 stream, specialisations on")
    print(f"final rel-L2 {EC.rel_l2(got, want):.3e}")
    print(f"{'stage':60s} {'cum rel-L2':>10s}  ref_std")
    for name, r in ref_out.items():
        e = eng_out.get(name)
        if e is None:
            continue
        if e.dim() == 4:
            e = e.permute(0, 3, 1, 2)
        print(f"{name:60s} {EC.rel_l2(e, r):10.3e}  {r.std().item():.3f}")

    print("\n# attribution experiments (final rel-L2 vs the fp32 oracle)")
    print(f"baseline                 {EC.rel_l2(got, want):.3e}")
    keep = ops.attention_d64
    ops.attention_d64 = exact_attention
    print(f"exact_attention          {EC.rel_l2(run()[0], want):.3e}")
    ops.attention_d64 = keep
    print(f"fp16_stream              {EC.rel_l2(run(stream=torch.float16)[0], want):.3e}")
    print(f"general_path             {EC.rel_l2(run(spec=False)[0], want):.3e}")
    if hasattr(ops, "SPLIT_OPERANDS"):
        ops.SPLIT_OPERANDS = True
        print(f"split_operands           {EC.rel_l2(run()[0], want):.3e}")
        ops.SPLIT_OPERANDS = False
    y16 = ref.half()(x.half(), 999, ctx.half()).sample
    print(f"torch_fp16_reference     {EC.rel_l2(y16, want):.3e}   (the reference's own fp16 GPU path)")


if __name__ == "__main__":
    main()
