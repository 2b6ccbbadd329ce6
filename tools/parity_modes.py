"""Full-size (768x768, SD-2 widths, batch 1) parity of the three residual-stream modes against the fp32 oracle run with
torch ops on the same GPU -> out/parity_modes.json."""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import engine_checks as EC
out = {}
for name, (s, v) in dict(fp32=(torch.float32, None), mixed=(torch.float32, torch.float16), fp16=(torch.float16, None)).items():
    r = EC.run_full_size(res=768, batch=1, stream_dtype=s, vae_stream_dtype=v)
    out[name] = {k: float(f"{x:.4g}") for k, x in r.items()}
    print(name, out[name], flush=True)
    torch.cuda.empty_cache()
os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "out", "parity_modes.json"), "w"), indent=1)
