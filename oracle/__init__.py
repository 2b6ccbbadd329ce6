"""ORACLE — test infrastructure only.

Plain-PyTorch fp32 restatement of the reference's single-step denoising hot path
(`VAE.encode -> UNet2DConditionModel(t=999) -> x0 -> VAE.decode`) used as the CHECKER
for the CUDA engine in `diffusion_e2e_ft_b200`.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl reference`
legs may import this package.  The product path never does.

PARITY UNPINNED: the reference (the reference checkout, pure Python) ships no tests, no golden
vectors and no weights, and its arithmetic lives in `diffusers==0.30.2` /
`xformers==0.0.24` (requirements.txt:2,8) which are not installable here (no network).
The restatement follows the in-tree GeoWizard copies of the diffusers graph
(GeoWizard/geowizard/models/*.py) plus the published diffusers-0.30.2 semantics of the
leaf operators (SURVEY.md App. A); it is pinned structurally (parameter counts
865,910,724 UNet-4ch / 865,922,244 UNet-8ch, 34,163,664 + 49,490,199 VAE — the public SD-2
figures — and the diffusers `state_dict` key layout) and by algebraic known-answer tests
(tests/test_oracle.py), not by reference-run outputs.
"""
