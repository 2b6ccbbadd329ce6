"""GeoWizard's SD-1-shaped UNet on the CPU: 8 heads of width 40 / 80 / 160 and 1x1-conv transformer projections.
Construction, the public SD-1 parameter count and diffusers state_dict layout, config / training-state round trips,
the head-width checks of the C ABI, and the host wiring of forward and backward with the kernels replaced by their
plain-torch contracts (tests/cpu_emulation.py, tests/sd1_checks.py)."""
import json
import os

import pytest
import torch

import engine_checks as EC           # also puts tests/golden on sys.path
import sd1_checks as S
from diffusion_e2e_ft_b200 import B200UNet2DConditionModel, ops

SD1_PARAMS = 859_520_964             # the public SD-1.x UNet (in_channels 4, cross-attention width 768)


@pytest.fixture
def emulated(monkeypatch):
    S.install_emulation(monkeypatch)
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)
    S.sd1_tiny(monkeypatch)


def test_geowizard_sd1_config_constructs():
    with torch.device("meta"):
        unet = B200UNet2DConditionModel(**S.GEOWIZARD_SD1)
    widths = {blk.head_dim for m in unet.modules() for blk in getattr(m, "transformer_blocks", [])}
    assert widths == {40, 80, 160}
    assert tuple(unet.down_blocks[0].attentions[0].proj_in.weight.shape) == (320, 320, 1, 1)
    assert unet.config["attention_head_dim"] == 8 and unet.config["use_linear_projection"] is False


@pytest.mark.parametrize("heads,width", [(10, "32"), (6, "53.3333"), (1, "320")])
def test_unsupported_head_width_raises_at_construction(heads, width):
    with pytest.raises(NotImplementedError, match=f"head width {width}"):
        with torch.device("meta"):
            B200UNet2DConditionModel(block_out_channels=(320, 320, 320, 320), attention_head_dim=heads)


def test_sd1_parameter_count_and_state_dict_match_oracle():
    with torch.device("meta"):
        ref = S.unet_ref(S.sd1_config())
        eng = B200UNet2DConditionModel(in_channels=4, attention_head_dim=8, cross_attention_dim=768,
                                       use_linear_projection=False)
    assert sum(p.numel() for p in ref.parameters()) == SD1_PARAMS
    assert sum(p.numel() for p in eng.parameters()) == SD1_PARAMS
    sr, se = ref.state_dict(), eng.state_dict()
    assert {k: tuple(v.shape) for k, v in sr.items()} == {k: tuple(v.shape) for k, v in se.items()}
    assert tuple(se["mid_block.attentions.0.proj_out.weight"].shape) == (1280, 1280, 1, 1)
    eng.load_state_dict(sr, strict=True)
    ref.load_state_dict(se, strict=True)


def test_save_pretrained_round_trips_scalar_heads_and_conv_projections(tmp_path):
    ref, _ = S.build_tiny_sd1("geowizard")
    unet = B200UNet2DConditionModel(block_out_channels=(320, 320, 320, 320), attention_head_dim=8,
                                    use_linear_projection=False, cross_attention_dim=96, class_embed_type="projection",
                                    projection_class_embeddings_input_dim=10, joint_attention=True)
    torch.manual_seed(0)
    with torch.no_grad():
        for p in unet.parameters():
            p.normal_()
    unet.save_pretrained(str(tmp_path / "unet"))
    cfg = json.load(open(os.path.join(tmp_path, "unet", "config.json")))
    assert cfg["attention_head_dim"] == 8 and cfg["use_linear_projection"] is False
    back = B200UNet2DConditionModel.from_pretrained(str(tmp_path), subfolder="unet")
    assert back.config["attention_head_dim"] == 8 and back.config["use_linear_projection"] is False
    for (k, a), (k2, b) in zip(unet.state_dict().items(), back.state_dict().items()):
        assert k == k2 and torch.equal(a, b), k
    back.save_pretrained(str(tmp_path / "again"))
    assert json.load(open(os.path.join(tmp_path, "again", "config.json"))) == cfg


def test_flat_trainer_resume_with_conv_projections(monkeypatch, tmp_path):
    import test_training_state_cpu as T
    S.install_emulation(monkeypatch)
    monkeypatch.setattr(ops, "adamw_step_state_groups", T.adamw_step_state_groups)
    monkeypatch.setattr(ops, "ema_update", lambda ema, p, omd: ema.sub_(float(omd) * (ema - p)))
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)
    S.sd1_tiny(monkeypatch)
    assert T._unet().down_blocks[0].attentions[0].proj_in.weight.dim() == 4
    T.test_resume_continues_bit_identically(None, tmp_path)


def test_c_abi_rejects_other_head_widths_without_launching():
    from diffusion_e2e_ft_b200 import lib
    L = lib.load()
    for d in (32, 48, 128):
        rc = L.b200_attention(16, 64, 64, 16, 64, 64, 16, 64, 64, 16, 64, 64, 1, 1, d, 8, 8, 1, 0.1, None, None)
        assert rc < 0 and f"head_dim={d}".encode() in L.b200_last_error_string()
        rc = L.b200_rowdot_heads_d(16, 64, 64, 16, 64, 64, 1, 8, 1, d, 16, None)
        assert rc < 0 and f"head_dim={d}".encode() in L.b200_last_error_string()
    q = torch.zeros(1, 8, 96, dtype=torch.float16)
    with pytest.raises(ValueError, match="head width 48"):
        ops.attention(q, q, q, 2, 0.1)


@pytest.mark.parametrize("kind,hw", [("geowizard", (16, 16)), ("geowizard", (15, 20)), ("marigold", (15, 20))])
def test_unet_backward_wiring_matches_oracle_autograd(emulated, kind, hw):
    r = EC.run_unet_backward_tiny(device="cpu", hw=hw, kind=kind)
    assert not r["missing"], r["missing"]
    assert r["forward"] <= 3e-3, r
    assert r["grad_global"] <= 1e-2 and r["grad_worst"] <= 2e-2, r


def test_gradient_checkpointing_wiring(emulated):
    r = EC.run_checkpointing_tiny(device="cpu")
    assert r["global_rel_diff"] <= 1e-6 and r["ckpt_vs_oracle_global"] <= 1e-2, r


def test_constant_context_fold_wiring(emulated):
    r = EC.run_single_step_specialisations(device="cpu", hw=(8, 8))
    assert r["spec_vs_general"] <= 2e-3 and r["spec_vs_oracle"] <= 3e-3 and r["repeat_call"] == 0.0, r
    assert r["per_image_ctx_vs_oracle"] <= 3e-3, r


def test_geowizard_joint_training_step_wiring(emulated):
    r = EC.run_training_step_geowizard_tiny(device="cpu")
    assert not r["missing"], r["missing"]
    assert r["loss_rel"] <= 3e-3, r
    assert r["grad_global"] <= 6e-2 and r["grad_worst"] <= 0.2, r
