"""CPU tests of multi-step DDIM inference: the scheduler surface (schedules, prev_timestep, final_alpha_cumprod,
from_pretrained), the host wiring of the Marigold and GeoWizard denoising loops with the kernels emulated, and the
argument errors raised before any launch."""
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

# diffusers 0.30.2 schedules for T = 1000, steps_offset = 1 (from its set_timesteps formulas)
SCHEDULES = {
    ("trailing", 3): [999, 666, 332],
    ("trailing", 10): [999, 899, 799, 699, 599, 499, 399, 299, 199, 99],
    ("leading", 3): [667, 334, 1],
    ("leading", 10): [901, 801, 701, 601, 501, 401, 301, 201, 101, 1],
    ("linspace", 3): [999, 500, 0],
    ("linspace", 4): [999, 666, 333, 0],
    ("linspace", 10): [999, 888, 777, 666, 555, 444, 333, 222, 111, 0],
}


# ------------------------------------------------------------------------------------------------ scheduler
@pytest.mark.parametrize("spacing,n", sorted(SCHEDULES))
def test_schedules_match_diffusers(spacing, n):
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from multistep_oracle import DDIMRef
    s, o = DDIMScheduler(timestep_spacing=spacing), DDIMRef(timestep_spacing=spacing)
    s.set_timesteps(n)
    o.set_timesteps(n)
    assert s.timesteps.tolist() == SCHEDULES[(spacing, n)]
    assert o.timesteps.tolist() == SCHEDULES[(spacing, n)]
    assert s.timesteps.dtype == torch.long


def test_prev_timestep_is_diffusers_t_minus_T_over_n():
    from diffusion_e2e_ft_b200 import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(3)
    # 999 -> 666 -> 332, but the step at 666 uses prev = 333 (diffusers' t - T // n)
    assert [s.coefficients(i)[1] for i in range(3)] == [666, 333, -1]
    s.set_timesteps(10)
    assert [s.coefficients(i)[1] for i in range(10)] == [899, 799, 699, 599, 499, 399, 299, 199, 99, -1]


@pytest.mark.parametrize("set_alpha_to_one", [True, False])
def test_final_alpha_cumprod(set_alpha_to_one):
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from multistep_oracle import DDIMRef
    s = DDIMScheduler(set_alpha_to_one=set_alpha_to_one, timestep_spacing="leading")
    o = DDIMRef(set_alpha_to_one=set_alpha_to_one, timestep_spacing="leading")
    want = 1.0 if set_alpha_to_one else float(s.alphas_cumprod[0])
    assert float(s.final_alpha_cumprod) == want == float(o.final_alpha_cumprod)
    s.set_timesteps(4)                                          # leading 4: [751, 501, 251, 1]; the last prev is -249
    t, prev, a_t, a_prev = s.coefficients(3)
    assert (t, prev) == (1, -249) and a_prev == want and a_t == float(s.alphas_cumprod[1])
    t, prev, a_t, a_prev = s.coefficients(0)
    assert (t, prev) == (751, 501) and a_prev == float(s.alphas_cumprod[501])


_MARIGOLD_CONFIG = {
    "_class_name": "DDIMScheduler", "_diffusers_version": "0.25.0", "beta_end": 0.012,
    "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False, "clip_sample_range": 1.0,
    "dynamic_thresholding_ratio": 0.995, "num_train_timesteps": 1000, "prediction_type": "v_prediction",
    "rescale_betas_zero_snr": False, "sample_max_value": 1.0, "set_alpha_to_one": False, "steps_offset": 1,
    "skip_prk_steps": True, "thresholding": False, "timestep_spacing": "leading", "trained_betas": None,
}


def _write_config(tmp_path, **changes):
    d = tmp_path / "ckpt" / "scheduler"
    d.mkdir(parents=True, exist_ok=True)
    cfg = dict(_MARIGOLD_CONFIG, **changes)
    (d / "scheduler_config.json").write_text(json.dumps(cfg))
    return str(tmp_path / "ckpt")


def test_from_pretrained_reads_scheduler_config(tmp_path):
    from diffusion_e2e_ft_b200 import DDIMScheduler
    ckpt = _write_config(tmp_path)
    s = DDIMScheduler.from_pretrained(ckpt, subfolder="scheduler")
    assert s.config["timestep_spacing"] == "leading" and s.config["prediction_type"] == "v_prediction"
    assert s.config["set_alpha_to_one"] is False and s.config["steps_offset"] == 1
    assert float(s.final_alpha_cumprod) == float(s.alphas_cumprod[0])
    # keys that are not DDIM arguments (the PNDM `skip_prk_steps` of SD-2 configs) change no math and are kept aside
    assert s.config["_extra"] == {"_diffusers_version": "0.25.0", "skip_prk_steps": True}
    s.set_timesteps(3)
    assert s.timesteps.tolist() == [667, 334, 1]
    # the keyword override wins over the file (Marigold/run.py:273, GeoWizard/run_infer.py:194-197)
    s = DDIMScheduler.from_pretrained(ckpt, subfolder="scheduler", timestep_spacing="trailing")
    s.set_timesteps(3)
    assert s.timesteps.tolist() == [999, 666, 332]
    torch.testing.assert_close(s.alphas_cumprod, DDIMScheduler().alphas_cumprod, rtol=0, atol=0)
    # the path may also point at the scheduler directory itself
    s = DDIMScheduler.from_pretrained(os.path.join(ckpt, "scheduler"), timestep_spacing="linspace")
    s.set_timesteps(4)
    assert s.timesteps.tolist() == [999, 666, 333, 0]


@pytest.mark.parametrize("key,value", [("beta_schedule", "linear"), ("beta_schedule", "squaredcos_cap_v2"),
                                       ("trained_betas", [0.1] * 1000), ("clip_sample", True),
                                       ("thresholding", True), ("rescale_betas_zero_snr", True),
                                       ("prediction_type", "flow"), ("timestep_spacing", "karras")])
def test_from_pretrained_rejects_unsupported_config(tmp_path, key, value):
    from diffusion_e2e_ft_b200 import DDIMScheduler
    ckpt = _write_config(tmp_path, **{key: value})
    with pytest.raises(ValueError, match=key):
        DDIMScheduler.from_pretrained(ckpt, subfolder="scheduler")


def test_from_pretrained_missing_keys_take_diffusers_defaults(tmp_path):
    """diffusers' own defaults are `linear` betas and clip_sample=True: a config that omits them is not SD-2 math."""
    from diffusion_e2e_ft_b200 import DDIMScheduler
    d = tmp_path / "s"
    d.mkdir()
    (d / "scheduler_config.json").write_text(json.dumps({"prediction_type": "v_prediction"}))
    with pytest.raises(ValueError, match="beta_schedule"):
        DDIMScheduler.from_pretrained(str(d))


def test_step_rejects_eta_and_unknown_prediction_type():
    from diffusion_e2e_ft_b200 import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(2)
    x = torch.zeros(1, 4, 2, 2)
    with pytest.raises(NotImplementedError, match="eta"):
        s.step(x, 999, x, eta=0.5)
    for t in (-1, 1000, torch.tensor(-5)):                     # no wrap-around into alphas_cumprod
        with pytest.raises(ValueError, match="outside"):
            s.step(x, t, x)
    s.config["prediction_type"] = "flow"
    with pytest.raises(ValueError, match="prediction_type"):
        s.step(x, 999, x)                                       # raised before anything is launched


# ------------------------------------------------------------------------------------------------ emulated kernel
def _ddim_step_emulated(calls):
    """The b200_ddim_step contract in torch fp32 (include/b200_e2eft.h), with the argument checks of ops.ddim_step."""
    from diffusion_e2e_ft_b200 import ops

    def ddim_step(model_out, sample, alpha_prod_t, alpha_prod_t_prev, prediction_type="v_prediction", out=None,
                  want_x0=False, unet_in=None):
        assert model_out.dtype in (torch.float16, torch.float32) and model_out.stride(-1) == 1
        assert sample is None or sample.dtype == torch.float32
        assert prediction_type in ops.PREDICTION_TYPES
        calls.append(dict(sample=sample, out=out, unet_in=unet_in, a=(alpha_prod_t, alpha_prod_t_prev)))
        a_t, a_prev = torch.tensor(alpha_prod_t, dtype=torch.float32), torch.tensor(alpha_prod_t_prev, dtype=torch.float32)
        m = model_out.float()
        x = torch.zeros_like(m) if sample is None else sample
        beta = 1 - a_t
        if prediction_type == "v_prediction":
            x0, eps = a_t.sqrt() * x - beta.sqrt() * m, a_t.sqrt() * m + beta.sqrt() * x
        elif prediction_type == "epsilon":
            x0, eps = (x - beta.sqrt() * m) / a_t.sqrt(), m
        else:
            x0 = m
            eps = (x - a_t.sqrt() * x0) / beta.sqrt()
        prev = a_prev.sqrt() * x0 + (1 - a_prev).sqrt() * eps
        if out is None:
            out = prev
        else:
            assert out.is_contiguous()
            out.copy_(prev)
        if unet_in is not None:
            unet_in.copy_(prev.to(unet_in.dtype))
        return out, (x0 if want_x0 else None)
    return ddim_step


def _install(monkeypatch):
    import cpu_emulation
    from diffusion_e2e_ft_b200 import ops
    cpu_emulation.install(monkeypatch)
    calls = []
    monkeypatch.setattr(ops, "ddim_step", _ddim_step_emulated(calls))
    # b200_conv3x3_small_cout writes a contiguous NCHW tensor; F.conv2d on the NHWC view keeps the channels-last strides
    small = cpu_emulation.conv3x3_small_cout
    monkeypatch.setattr(ops, "conv3x3_small_cout", lambda *a, **k: small(*a, **k).contiguous())
    return calls


def test_scheduler_step_matches_oracle(monkeypatch):
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from multistep_oracle import DDIMRef
    _install(monkeypatch)
    g = torch.Generator().manual_seed(0)
    m, x = torch.randn(2, 4, 3, 5, generator=g), torch.randn(2, 4, 3, 5, generator=g)
    for pt in ("v_prediction", "epsilon", "sample"):
        s, o = DDIMScheduler(prediction_type=pt), DDIMRef(prediction_type=pt)
        s.set_timesteps(3)
        o.set_timesteps(3)
        for t in s.timesteps:                                   # 0-d tensors, as the reference loop passes them
            out = s.step(m, t, x)
            want_prev, want_x0 = o.step(m, t, x)
            torch.testing.assert_close(out.prev_sample, want_prev, rtol=1e-6, atol=1e-6)
            torch.testing.assert_close(out.pred_original_sample, want_x0, rtol=1e-6, atol=1e-6)
        prev, x0 = s.step(m, 332, x, return_dict=False)
        assert prev.dtype == torch.float32 and x0.shape == m.shape


# ------------------------------------------------------------------------------------------------ host wiring
def rel_l2(a, b):
    a, b = a.detach().float(), b.detach().float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def tiny_marigold():
    import make_golden as MG
    torch.manual_seed(0)
    return MG.build_tiny()


def _engine_reference_loop(pipe, rgb, steps, sched, init_latent=None, normals=False):
    """The reference's loop (marigold_pipeline.py:434-478) written out with the ENGINE modules and the oracle
    scheduler: torch.cat per step, scheduler.step in torch, x0 decoded unfused.  Same kernels (emulated) as the
    pipeline, so the two differ only by fp32 rounding: this isolates the pipeline's wiring."""
    import multistep_oracle as MO
    sched.set_timesteps(steps)
    rgb_latent = pipe.encode_rgb(rgb)
    latent = torch.zeros_like(rgb_latent) if init_latent is None else init_latent.float()
    ctx = pipe.empty_text_embed.expand(rgb.shape[0], -1, -1)
    for i, t in enumerate(sched.timesteps):
        pred = pipe.unet(torch.cat([rgb_latent, latent], 1), int(t), encoder_hidden_states=ctx).sample
        prev, x0 = MO.DDIMRef.step(sched, pred, t, latent)
        latent = x0 if i == steps - 1 else prev
    dec = pipe.vae.decoder(pipe.vae.post_quant_conv(latent, scale_in=1 / 0.18215))
    from diffusion_e2e_ft_b200 import ops
    return ops.decode_post(dec.float().contiguous(), normals=normals)


# The emulated GEMMs round their operands to fp16 as the kernels do; on this tiny random-weight model the DDIM loop
# amplifies that rounding step by step, so against the fp32 oracle the gate is looser than the wiring gate.
ORACLE_GATE_EMULATED = 3e-2


@pytest.mark.parametrize("steps", [2, 4])
@pytest.mark.parametrize("spacing", ["trailing", "leading"])
def test_marigold_multistep_host_wiring(monkeypatch, tiny_marigold, steps, spacing):
    import engine_checks as E
    import make_golden as MG
    import multistep_oracle as MO
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    calls = _install(monkeypatch)
    unet_ref, vae_ref = tiny_marigold
    unet, vae = E.engine_from_oracle(unet_ref, vae_ref, "cpu")
    rgb = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(3)) * 2 - 1
    ete = MG.inputs(5, 1, 2, 128, scale=0.5)
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(timestep_spacing=spacing), empty_text_embed=ete)
    got = pipe.single_infer(rgb, steps, noise="gaussian", generator=torch.Generator().manual_seed(11))
    noise = torch.randn((2, 4, 4, 4), generator=torch.Generator().manual_seed(11))   # the draw the engine made
    want = MO.marigold_infer(unet_ref, vae_ref, MO.DDIMRef(timestep_spacing=spacing), rgb, ete, steps, init_latent=noise)
    assert len(calls) == steps - 1
    # every intermediate step updates the fp32 state in place and writes channels 4..7 of ONE persistent UNet input
    assert all(c["out"] is calls[0]["out"] and c["sample"] is c["out"] for c in calls)
    assert len({c["unet_in"].data_ptr() for c in calls}) == 1 and calls[0]["unet_in"].shape == (2, 4, 4, 4)
    assert calls[0]["unet_in"].stride(0) == 8 * 16
    wired = _engine_reference_loop(pipe, rgb, steps, MO.DDIMRef(timestep_spacing=spacing), init_latent=noise)
    assert rel_l2(got, wired) <= 1e-5, rel_l2(got, wired)
    assert rel_l2(got, want) <= ORACLE_GATE_EMULATED, rel_l2(got, want)
    # zeros noise with several steps: the first step runs conv_in on the 4 rgb channels, the sample starts as NULL
    calls.clear()
    got0 = pipe.single_infer(rgb, steps, noise="zeros")
    want0 = MO.marigold_infer(unet_ref, vae_ref, MO.DDIMRef(timestep_spacing=spacing), rgb, ete, steps)
    assert calls[0]["sample"] is None and len(calls) == steps - 1
    wired0 = _engine_reference_loop(pipe, rgb, steps, MO.DDIMRef(timestep_spacing=spacing))
    # (the 4-channel conv_in of the first step sums in another order than the 8-channel one of the written-out loop;
    # the loop amplifies that fp32 rounding difference, to 2e-4 at 4 steps)
    assert rel_l2(got0, wired0) <= 1e-3, rel_l2(got0, wired0)
    assert rel_l2(got0, want0) <= ORACLE_GATE_EMULATED, rel_l2(got0, want0)


def test_marigold_normals_multistep_host_wiring(monkeypatch, tiny_marigold):
    import engine_checks as E
    import make_golden as MG
    import multistep_oracle as MO
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    _install(monkeypatch)
    unet_ref, vae_ref = tiny_marigold
    unet, vae = E.engine_from_oracle(unet_ref, vae_ref, "cpu")
    rgb = torch.rand(1, 3, 32, 32, generator=torch.Generator().manual_seed(4)) * 2 - 1
    ete = MG.inputs(5, 1, 2, 128, scale=0.5)
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=ete)
    got = pipe.single_infer(rgb, 2, noise="gaussian", normals=True, generator=torch.Generator().manual_seed(2))
    noise = torch.randn((1, 4, 4, 4), generator=torch.Generator().manual_seed(2))
    want = MO.marigold_infer(unet_ref, vae_ref, MO.DDIMRef(), rgb, ete, 2, init_latent=noise, normals=True)
    wired = _engine_reference_loop(pipe, rgb, 2, MO.DDIMRef(), init_latent=noise, normals=True)
    assert rel_l2(got, wired) <= 1e-5, rel_l2(got, wired)
    assert E.mean_angle_deg(got, want) <= 0.5 and rel_l2(got, want) <= ORACLE_GATE_EMULATED


def test_geowizard_multistep_host_wiring(monkeypatch):
    import engine_checks as E
    import make_golden as MG
    import multistep_oracle as MO
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline
    calls = _install(monkeypatch)
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = E.engine_from_oracle(gunet_ref, vae_ref, "cpu")
    rgb = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(3)) * 2 - 1
    emb = MG.inputs(6, 2, 1, 96, scale=0.5)
    pipe = DepthNormalEstimationPipeline(unet, vae, DDIMScheduler())
    d, n = pipe.single_infer(rgb, 4, "indoor", noise="gaussian", img_embed=emb,
                             generator=torch.Generator().manual_seed(9))
    noise = torch.randn((2, 4, 4, 4), generator=torch.Generator().manual_seed(9))
    wd, wn = MO.geowizard_infer(gunet_ref, vae_ref, MO.DDIMRef(), rgb, emb, "indoor", 4, init_latent=noise)
    assert len(calls) == 3 and calls[0]["unet_in"].shape == (4, 4, 4, 4)       # the whole [2B] state per step
    assert rel_l2(d, wd) <= ORACLE_GATE_EMULATED and rel_l2(n, wn) <= ORACLE_GATE_EMULATED, (rel_l2(d, wd), rel_l2(n, wn))
    assert E.mean_angle_deg(n, wn) <= 0.5


def test_restated_oracle_reduces_to_the_single_step_oracle():
    """At one step with zeros the multi-step oracle computes what the golden fixtures hold."""
    import engine_checks as E
    import make_golden as MG
    import multistep_oracle as MO
    gold = torch.load(E.GOLD)
    unet, vae = MG.build_tiny()
    rgb = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(3)) * 2 - 1
    ete = MG.inputs(5, 1, 2, 128, scale=0.5)
    d = MO.marigold_infer(unet, vae, MO.DDIMRef(), rgb, ete)
    assert rel_l2(d, gold["marigold_depth_64"]["y"]) <= 1e-5
    gunet, _ = MG.build_tiny("geowizard")
    gd, gn = MO.geowizard_infer(gunet, vae, MO.DDIMRef(), rgb, MG.inputs(6, 2, 1, 96, scale=0.5))
    assert rel_l2(gd, gold["geowizard_64"]["depth"]) <= 1e-5 and rel_l2(gn, gold["geowizard_64"]["normal"]) <= 1e-5


# ------------------------------------------------------------------------------------------------ argument errors
class _NoLaunch(torch.nn.Module):
    """A module that fails the test if anything tries to run it."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.config = {"block_out_channels": (32, 64), "latent_channels": 4}

    def forward(self, *a, **k):
        raise AssertionError("launched before the argument check")

    encoder = decoder = forward

    def encode_scaled_mean(self, *a, **k):
        raise AssertionError("launched before the argument check")


def test_argument_errors_before_any_launch():
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline, MarigoldPipeline
    geo = DepthNormalEstimationPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler())
    x = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="pyramid"):
        geo.single_infer(x, 4, "indoor", noise="pyramid", img_embed=torch.zeros(1, 1, 96))
    with pytest.raises(ValueError, match="pyramid"):
        geo(torch.zeros(3, 16, 16), denoising_steps=2, noise="pyramid", img_embed=torch.zeros(1, 1, 96))
    with pytest.raises(ValueError, match="Unknown noise type"):
        geo.single_infer(x, 1, "indoor", noise="uniform")
    mari = MarigoldPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler(), empty_text_embed=torch.zeros(1, 2, 128))
    with pytest.raises(ValueError, match="Unknown noise type"):
        mari.single_infer(x, 4, noise="uniform")
    with pytest.raises(ValueError, match="Unknown noise type"):
        mari(torch.zeros(3, 16, 16), noise="uniform")
    with pytest.raises(ValueError, match="num_inference_steps"):
        mari.single_infer(x, 0, noise="gaussian")
    s = DDIMScheduler()
    s.set_timesteps(4)
    with pytest.raises(NotImplementedError, match="eta"):
        s.step(torch.zeros(1, 4, 2, 2), 999, torch.zeros(1, 4, 2, 2), eta=1.0)


def test_geowizard_pyramid_noise_is_its_own_variant():
    """geowizard_pipeline.py:33-43: one timestep, unit std, shape of x; more than one timestep cannot broadcast."""
    import numpy as np
    from diffusion_e2e_ft_b200.pipelines import geowizard_pyramid_noise_like
    torch.manual_seed(0)
    np.random.seed(0)
    x = torch.zeros(1, 4, 12, 12)
    n = geowizard_pyramid_noise_like(x, torch.tensor([999]))
    assert n.shape == x.shape and abs(n.std().item() - 1.0) < 1e-5
    with pytest.raises(RuntimeError):
        geowizard_pyramid_noise_like(x, torch.tensor([999, 499]))
