"""Throughput of the other BASELINE.json configs on one GPU (not the bench line):
   config 5: marigold normals, bs=16, processing_res in {384,512,768,1024}
   config 4: GeoWizard joint depth+normals, bs=4 images (UNet batch 8, joint self-attention Lk = 2L), 768x768."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from diffusion_e2e_ft_b200 import (B200AutoencoderKL, B200UNet2DConditionModel, DDIMScheduler, MarigoldPipeline,
                                   DepthNormalEstimationPipeline)
dev = torch.device("cuda", 0)
torch.manual_seed(0)
out = {}

def timeit(fn, n=3):
    fn(); fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

with torch.device(dev):
    unet = B200UNet2DConditionModel().half().eval().requires_grad_(False)
    vae = B200AutoencoderKL().half().eval().requires_grad_(False)
pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=(torch.randn(1, 2, 1024, device=dev) * 0.5).half())
for res in (384, 512, 768, 1024):
    bs = 16
    while bs >= 1:
        try:
            x = (torch.rand(bs, 3, res, res, device=dev) * 2 - 1).half()
            ms = timeit(lambda: pipe.single_infer(x, 1, False, noise="zeros", normals=True))
            out[f"marigold_normals_res{res}"] = dict(batch=bs, ms_per_batch=ms, images_per_s=bs / ms * 1e3)
            break
        except RuntimeError as e:
            out[f"marigold_normals_res{res}_bs{bs}_error"] = str(e)[:120]
            bs //= 2
    print(res, out.get(f"marigold_normals_res{res}"), flush=True)
del pipe, unet
torch.cuda.empty_cache()
with torch.device(dev):
    gunet = B200UNet2DConditionModel(class_embed_type="projection", projection_class_embeddings_input_dim=10,
                                     cross_attention_dim=768, joint_attention=True).half().eval().requires_grad_(False)
gp = DepthNormalEstimationPipeline(gunet, vae, DDIMScheduler())
x = (torch.rand(4, 3, 768, 768, device=dev) * 2 - 1).half()
emb = (torch.randn(4, 1, 768, device=dev) * 0.5).half()
ms = timeit(lambda: gp.single_infer(x, 1, "indoor", img_embed=emb))
out["geowizard_joint_bs4_768"] = dict(batch=4, ms_per_batch=ms, images_per_s=4 / ms * 1e3)
print(out["geowizard_joint_bs4_768"])
os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "out", "extra_configs.json"), "w"), indent=1)
