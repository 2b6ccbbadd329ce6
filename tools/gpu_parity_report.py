"""Write a parity report (to out/parity.json) from the engine checks."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import engine_checks as EC
rep = {}
rep["marigold_tiny_fp32_stream"] = EC.run_marigold_tiny()
rep["marigold_tiny_fp16_stream"] = EC.run_marigold_tiny(stream_dtype=torch.float16)
rep["geowizard_tiny_fp32_stream"] = EC.run_geowizard_tiny()
rep["unet_fullwidth_latent24_fp32_stream"] = EC.run_unet_fullwidth(latent=24)
rep["unet_fullwidth_latent24_fp16_stream"] = EC.run_unet_fullwidth(latent=24, stream_dtype=torch.float16)
os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
json.dump(rep, open(os.path.join(ROOT, "out", "parity.json"), "w"), indent=1)
print(json.dumps(rep, indent=1))
