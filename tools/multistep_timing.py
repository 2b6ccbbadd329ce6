"""Time multi-step DDIM inference of the diffusion-estimator checkpoints (random-init SD-2 widths, fp16 modules, fp32
residual stream: bench.py's headline engine configuration).

    python tools/multistep_timing.py [--out FILE] [--reps N]

* Marigold, one 3x768x768 image as the reference's default call shapes it: ensemble 10 in one batch of 10
  (`single_infer` of [10, 3, 768, 768]), gaussian noise (zeros for 1 step, the E2E-FT setting), steps {1, 4, 10},
  CUDA-graphed and eager;
* GeoWizard, the same image, ensemble 10 in one batch (joint depth + normal: UNet batch 20), 10 gaussian steps,
  eager (the CLIP image embedding is passed in, so the time is the denoising loop + VAE).

Each entry: CUDA-event time of one `single_infer` call after warm-up (graph capture included in the warm-up), median of
--reps, and torch.cuda.max_memory_allocated from the first warm-up call on (graph capture included).  Device name,
power limit and SM clocks are read with a read-only nvidia-smi query in the same process and printed beside the
numbers; no device setting is changed.  Prints one JSON object.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from vae_attention_timing import _gpu_info  # noqa: E402


def _time(fn, reps, warmup):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()           # before the warm-up: a captured graph's private pool counts
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return dict(median_ms=ts[len(ts) // 2], min_ms=ts[0], max_ms=ts[-1], reps=reps,
                max_memory_allocated_gb=torch.cuda.max_memory_allocated() / 1024 ** 3)


def _engine(workload):
    from bench import build_engine
    return build_engine("cuda", torch.float32, torch.float16, workload=workload)


@torch.no_grad()
def time_marigold(res, batch, steps_list, reps):
    pipe = _engine("marigold")
    x = (torch.rand(batch, 3, res, res, generator=torch.Generator().manual_seed(0)) * 2 - 1).cuda().half()
    out = []
    for steps in steps_list:
        noise = "zeros" if steps == 1 else "gaussian"
        for graph in (True, False):
            pipe.use_cuda_graph = graph
            gen = torch.Generator(device="cuda").manual_seed(0)
            r = _time(lambda: pipe.single_infer(x, steps, noise=noise, generator=gen), reps, 2)
            r.update(steps=steps, noise=noise, graphed=graph, images_per_s=batch / (r["median_ms"] / 1e3))
            out.append(r)
            print(json.dumps(dict(marigold=r)), flush=True)
        pipe.__dict__.pop("_graphs", None)
        torch.cuda.empty_cache()
    return out


@torch.no_grad()
def time_geowizard(res, batch, steps, reps):
    pipe = _engine("geowizard")
    x = (torch.rand(batch, 3, res, res, generator=torch.Generator().manual_seed(0)) * 2 - 1).cuda().half()
    emb = (torch.randn(1, 1, 768, generator=torch.Generator().manual_seed(1)) * 0.5).cuda().half()
    r = _time(lambda: pipe.single_infer(x, steps, "indoor", noise="gaussian", img_embed=emb), reps, 2)
    r.update(steps=steps, noise="gaussian", graphed=False, images_per_s=batch / (r["median_ms"] / 1e3))
    print(json.dumps(dict(geowizard=r)), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON here")
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", default="1,4,10")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multistep_timing needs a CUDA device")
    res = dict(gpu=_gpu_info(), res=a.res, batch=a.batch)
    res["marigold"] = time_marigold(a.res, a.batch, [int(s) for s in a.steps.split(",")], a.reps)
    torch.cuda.empty_cache()
    res["geowizard"] = time_geowizard(a.res, a.batch, 10, a.reps)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
