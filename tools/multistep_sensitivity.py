"""How much a multi-step DDIM loop amplifies a per-call UNet error, on the fp32 oracle (CPU, tiny config).

    python tools/multistep_sensitivity.py [--eps 1e-3]

Every UNet call's output gets an independent gaussian perturbation of relative L2 size `eps` (a stand-in for the
engine's fp16-operand error per call); the final depth (rel-L2) and normals (mean angle) are compared with the
unperturbed oracle, for zeros- and gaussian-started loops at 1, 2, 4, 10 trailing steps (worst of 3 seeds).  This
attributes the engine-vs-oracle error of multi-step runs (tests/test_multistep_gpu.py) to the UNet rather than to the
DDIM step, whose kernel matches a torch fp32 restatement bit for bit.  Prints one line per case.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import engine_checks as E  # noqa: E402
import make_golden as MG  # noqa: E402
import multistep_oracle as MO  # noqa: E402


class Perturbed(torch.nn.Module):
    def __init__(self, unet, eps, seed):
        super().__init__()
        self.unet, self.eps, self.g = unet, eps, torch.Generator().manual_seed(seed)

    def forward(self, *a, **k):
        out = self.unet(*a, **k)
        y = out.sample
        d = torch.randn(y.shape, generator=self.g)
        out.sample = y + self.eps * y.norm() / d.norm() * d
        return out


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--eps", type=float, default=1e-3)
    a = ap.parse_args()
    unet, vae = MG.build_tiny()
    rgb = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(3)) * 2 - 1
    ete = MG.inputs(5, 1, 2, 128, scale=0.5)
    for noise in ("zeros", "gaussian"):
        for steps in (1, 2, 4, 10):
            init = None if noise == "zeros" else torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(17))
            res = {}
            for normals in (False, True):
                want = MO.marigold_infer(unet, vae, MO.DDIMRef(), rgb, ete, steps, init_latent=init, normals=normals)
                errs = []
                for seed in range(3):
                    got = MO.marigold_infer(Perturbed(unet, a.eps, seed), vae, MO.DDIMRef(), rgb, ete, steps,
                                            init_latent=init, normals=normals)
                    errs.append(E.mean_angle_deg(got, want) if normals else E.rel_l2(got, want))
                res["normals_mean_angle_deg" if normals else "depth_rel_l2"] = max(errs)
            print(f"eps={a.eps:g} noise={noise} steps={steps}", res, flush=True)


if __name__ == "__main__":
    main()
