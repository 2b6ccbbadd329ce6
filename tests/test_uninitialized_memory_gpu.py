"""The whole engine on NaN-filled allocations.

With torch.utils.deterministic.fill_uninitialized_memory, every torch.empty* returns NaN (floats) or the largest value
(integers, uint8).  The library never allocates, so every buffer the engine hands a kernel starts poisoned: a kernel
that reads an element nobody wrote (a padding column, a K tail, a workspace it expects zeroed) turns the result into
NaN or garbage.  Each test reruns an existing tiny-size driver under the fill and asserts its home test's thresholds
and that every reported metric is finite.
"""
import math

import pytest
import torch

import diffusion_training_checks as DC
import engine_checks as EC
import test_evaluation_gpu as TEV
import test_multistep_gpu as TMS
import test_outputs_gpu as TOUT
import test_training_data_gpu as TDATA

pytestmark = pytest.mark.gpu


@pytest.fixture
def nan_fill():
    prev_det = torch.are_deterministic_algorithms_enabled()
    prev_warn = torch.is_deterministic_algorithms_warn_only_enabled()
    prev_fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        probe = torch.empty(1024, device="cuda")
        assert bool(torch.isnan(probe).all()), "fill_uninitialized_memory does not poison CUDA torch.empty"
        assert bool((torch.empty(64, dtype=torch.int32, device="cuda") == torch.iinfo(torch.int32).max).all())
        yield
    finally:
        torch.utils.deterministic.fill_uninitialized_memory = prev_fill
        torch.use_deterministic_algorithms(prev_det, warn_only=prev_warn)


def _finite(r):
    for k, v in r.items():
        if isinstance(v, float):
            assert math.isfinite(v), (k, r)


def test_marigold_tiny(nan_fill):
    r = EC.run_marigold_tiny()
    _finite(r)
    for k in ("unet_16x16_ctx2", "unet_15x20_ctx77", "vae_encode", "vae_decode", "depth_rel_l2"):
        assert r[k] <= 3e-3, (k, r)
    assert r["normals_mean_angle_deg"] <= 0.5 and r["absrel_delta"] <= 1e-3, r


def test_geowizard_tiny(nan_fill):
    r = EC.run_geowizard_tiny()
    _finite(r)
    assert r["depth"] <= 3e-3 and r["normal_mean_angle_deg"] <= 0.5, r


def test_single_step_specialisations(nan_fill):
    r = EC.run_single_step_specialisations(hw=(16, 16))
    _finite(r)
    assert r["spec_vs_general"] <= 2e-3 and r["repeat_call"] == 0.0, r
    assert r["spec_vs_oracle"] <= 3e-3 and r["per_image_ctx_vs_oracle"] <= 3e-3, r


def test_sd1_single_step_specialisations(nan_fill, monkeypatch):
    import sd1_checks
    sd1_checks.sd1_tiny(monkeypatch)
    r = EC.run_single_step_specialisations(hw=(15, 20))
    _finite(r)
    assert r["general_vs_oracle"] <= 3e-3 and r["spec_vs_oracle"] <= 3e-3 and r["spec_vs_general"] <= 2e-3, r
    assert r["per_image_ctx_vs_oracle"] <= 3e-3 and r["repeat_call"] == 0.0, r


@pytest.mark.parametrize("hw", [(16, 16), (15, 20)])
def test_unet_backward(nan_fill, hw):
    r = EC.run_unet_backward_tiny(hw=hw)
    _finite(r)
    assert not r["missing"] and r["forward"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


@pytest.mark.parametrize("modality,tol", [("depth", 3e-2), ("normals", 6e-2)])
def test_training_step(nan_fill, modality, tol):
    r = EC.run_training_step_tiny(modality=modality)
    _finite(r)
    assert not r["missing"] and r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= tol and r["grad_worst"] <= 3 * tol, r


def test_training_step_geowizard(nan_fill):
    r = EC.run_training_step_geowizard_tiny()
    _finite(r)
    assert not r["missing"] and r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 6e-2 and r["grad_worst"] <= 0.2, r


def test_checkpointing(nan_fill):
    r = EC.run_checkpointing_tiny()
    _finite(r)
    assert r["global_rel_diff"] <= 3e-3 and r["worst_rel_diff"] <= 1e-2 and r["ckpt_vs_oracle_global"] <= 1e-2, r


def test_training_loop(nan_fill):
    r = EC.run_training_loop_tiny()
    _finite(r)
    for a, b in zip(r["loss_engine"], r["loss_oracle"]):
        assert abs(a - b) / abs(b) <= 3e-3, r
    assert r["update_cosine"] >= 0.98 and abs(r["update_norm_ratio"] - 1.0) <= 0.03, r


def test_diffusion_step(nan_fill):
    r = DC.run_diffusion_step_tiny("cuda:0", "v_prediction", "gaussian", timesteps=(311, 42))
    _finite(r)
    assert r["loss_rel"] <= 3e-3 and r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


def test_wgrad_split_k(nan_fill):
    """The split-K weight gradient reads gather_planar's zero tail past the last pixel."""
    import test_engine_gpu as TE
    TE.test_wgrad_variants(True, 296)
    TE.test_wgrad_variants(False, 296)


@pytest.fixture
def tiny_multistep(nan_fill):
    return TMS.tiny.__wrapped__()


@pytest.fixture
def tiny_outputs(nan_fill):
    return TOUT.tiny.__wrapped__()


def test_multistep_tiny(tiny_multistep):
    TMS.test_marigold_tiny_vs_oracle(tiny_multistep, 4, "trailing", "gaussian")
    TMS.test_default_call_returns_depth_and_uncertainty(tiny_multistep)


def test_call_outputs_colourised(tiny_outputs):
    TOUT.test_marigold_call_vs_reference_postprocessing(tiny_outputs, "bilinear", 80)
    TOUT.test_marigold_bilinear_outputs_unchanged_by_colouring(tiny_outputs)


def test_evaluation_end_to_end(nan_fill):
    TEV.test_end_to_end_tiny_pipeline_outputs()
    TEV.test_normal_error_maps_and_pooled_metrics_vs_reference()


def test_training_batch_preparation(nan_fill, tmp_path_factory):
    trees = TDATA.trees.__wrapped__(tmp_path_factory)
    TDATA.test_hypersim_pins_bitwise(trees, True)
    TDATA.test_vkitti_pins_digests(trees, False)
