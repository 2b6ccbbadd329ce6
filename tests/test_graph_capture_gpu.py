"""The pipelines' CUDA-graph capture keeps Python's cyclic garbage collector off while it captures: a collection in
the middle could free an unreachable pipeline together with its captured graphs, and destroying a graph while a
stream captures invalidates the capture."""
import gc

import pytest
import torch

DEV = "cuda:0"


@pytest.mark.gpu
def test_capture_runs_with_the_collector_off_and_restores_it():
    import engine_checks as E
    import make_golden as MG
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    unet_ref, vae_ref = MG.build_tiny()
    unet, vae = E.engine_from_oracle(unet_ref, vae_ref, DEV)
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=MG.inputs(5, 1, 2, 128, scale=0.5).to(DEV))
    seen = []

    def fn(x):
        if torch.cuda.is_current_stream_capturing():
            seen.append(gc.isenabled())
        return x * 2.0

    x = torch.arange(8.0, device=DEV)
    assert gc.isenabled()
    out = pipe._graphed("probe", fn, x)
    assert seen == [False] and gc.isenabled()
    assert torch.equal(out, x * 2.0)
    # a replay does not capture again
    assert torch.equal(pipe._graphed("probe", fn, x + 1.0), (x + 1.0) * 2.0) and seen == [False]
    # the caller's setting is kept: with the collector already off it stays off
    gc.disable()
    try:
        pipe._graphed("probe2", fn, x)
        assert seen == [False, False] and not gc.isenabled()
    finally:
        gc.enable()
