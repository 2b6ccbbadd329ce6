"""GPU tests of the resampling choice and colour outputs: the nearest-exact and colour kernels bit for bit against torch
and the numpy restatements, the bicubic input path against torchvision's uint8 resize, and both pipelines' `__call__`
on the tiny models against the reference's post-processing applied to the engine's own `single_infer` output.
Measured values are printed (-s)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from outputs_reference import (mpl_colorize_depth, mpl_spectral_lut, np_colorize_normals,  # noqa: E402
                               ref_marigold_post, special_depths, tv_mode)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("hw,size", [((37, 53), (101, 77)), ((101, 77), (37, 53)), ((3, 7), (25, 29)),
                                     ((480, 640), (333, 999)), ((25, 29), (2, 3)), ((64, 64), (64, 64))])
def test_resize_nearest_exact_bit_exact(hw, size):
    from diffusion_e2e_ft_b200.ensemble import resize_nearest_exact
    x = torch.randn(3, *hw, generator=torch.Generator().manual_seed(0))
    got = resize_nearest_exact(x.to(DEV), size)
    want = F.interpolate(x[None].to(DEV), size=size, mode="nearest-exact")[0]
    assert got.shape == (3, *size) and torch.equal(got, want)
    assert torch.equal(got.cpu(), F.interpolate(x[None], size=size, mode="nearest-exact")[0])      # the CPU rule too
    d = resize_nearest_exact(x[0].to(DEV), size)                                                   # [H, W]
    assert torch.equal(d, want[0])


def test_bicubic_input_path_vs_torchvision_uint8():
    """The engine's bicubic input (fp32 resize, then round and clamp in normalise_rgb) against torchvision's
    resize(uint8, BICUBIC, antialias=True) on the host, as the reference runs it.  The separable fp32 sums run in
    another order than torch's, so a value that lands within the last bit of x.5 can round the other way: any
    difference must be exactly one uint8 level, on a small fraction of the pixels (printed).  Measured on an H100:
    at most 0.08 % of the values (576x768), none at 97x131 and 480x640."""
    from torchvision.transforms.functional import resize
    from diffusion_e2e_ft_b200.ensemble import normalise_rgb, resize_bicubic_aa
    img = torch.randint(0, 256, (3, 480, 640), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    for size in ((360, 480), (576, 768), (97, 131), (480, 640), (1080, 1440)):
        want = resize(img, list(size), tv_mode("bicubic"), antialias=True)
        got = normalise_rgb(resize_bicubic_aa(img.to(DEV).float(), size), round_u8=True).cpu()
        got_u8 = torch.round((got + 1.0) / 2.0 * 255.0)
        d = (got_u8 - want.float()).abs()
        frac = (d > 0).float().mean().item()
        print("bicubic_input", size, "max_lsb", d.max().item(), "fraction_differing", frac)
        assert d.max().item() <= 1.0 and frac <= 0.005, (size, d.max().item(), frac)


def test_colorize_depth_bit_exact():
    from diffusion_e2e_ft_b200.ensemble import colorize_depth
    lut = mpl_spectral_lut()
    d = special_depths()
    # (the reference's colorize_depth_maps squeezes its input, so a map with a unit dimension is not a case it has)
    for shape in ((27, d.size // 27 + 1), (7, 11), (33, 2), (1080, 1920), (5, 3)):
        n = shape[0] * shape[1]
        x = np.random.default_rng(n).uniform(-0.2, 1.2, n).astype(np.float32)
        x[:min(n, d.size)] = d[:min(n, d.size)]
        x = x.reshape(shape)
        got = colorize_depth(torch.from_numpy(x).to(DEV))
        assert got.dtype == torch.uint8 and got.shape == (*shape, 3)
        np.testing.assert_array_equal(got.cpu().numpy(), mpl_colorize_depth(x, lut))
    got = colorize_depth(torch.from_numpy(x)[None].to(DEV))                                      # [1, H, W]
    np.testing.assert_array_equal(got.cpu().numpy(), mpl_colorize_depth(x, lut))


def test_colorize_normals_bit_exact():
    from diffusion_e2e_ft_b200.ensemble import colorize_normals
    d = special_depths() * 2 - 1
    for hw in ((1, d.size), (7, 11), (1080, 1920), (5, 3)):
        n = 3 * hw[0] * hw[1]
        x = np.random.default_rng(n).uniform(-1.2, 1.2, n).astype(np.float32)
        x[:min(n, d.size)] = d[:min(n, d.size)]
        x[-min(n, d.size):] = d[:min(n, d.size)][::-1]
        x = x.reshape(3, *hw)
        got = colorize_normals(torch.from_numpy(x).to(DEV))
        assert got.dtype == torch.uint8 and got.shape == (*hw, 3)
        np.testing.assert_array_equal(got.cpu().numpy(), np_colorize_normals(x))


# ------------------------------------------------------------------------------------------------ pipelines
@pytest.fixture(scope="module")
def tiny():
    import engine_checks as E
    import make_golden as MG
    unet_ref, vae_ref = MG.build_tiny()
    return E.engine_from_oracle(unet_ref, vae_ref, DEV)


def _spy(pipe):
    """Record what single_infer saw and returned."""
    rec = {}
    orig = pipe.single_infer

    def single_infer(*a, **k):
        out = orig(*a, **k)
        rec["in"], rec["out"] = a[0].detach().clone(), out
        return out
    pipe.single_infer = single_infer
    return rec


# a non-square uint8 image, processed both below (80 < 100) and above (160 > 100) its size
IMG = (torch.rand(3, 60, 100, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)


@pytest.mark.parametrize("method", ["bilinear", "bicubic", "nearest"])
@pytest.mark.parametrize("processing_res", [80, 160])
def test_marigold_call_vs_reference_postprocessing(tiny, method, processing_res):
    from torchvision.transforms.functional import resize
    import make_golden as MG
    from PIL import Image
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    unet, vae = tiny
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=MG.inputs(5, 1, 2, 128, scale=0.5).to(DEV))
    rec = _spy(pipe)
    lut = mpl_spectral_lut()
    H, W = IMG.shape[-2:]
    s = min(processing_res / W, processing_res / H)
    want_in = resize(IMG, [int(H * s), int(W * s)], tv_mode(method), antialias=True) / 255.0 * 2.0 - 1.0
    for normals in (False, True):
        out = pipe(IMG, denoising_steps=1, ensemble_size=1, processing_res=processing_res, resample_method=method,
                   noise="zeros", normals=normals)
        lsb = ((rec["in"][0].cpu() - want_in).abs() * 255 / 2).round()
        # nearest-exact is exact; the antialiased resizes differ from torchvision's by at most one level on x.5 ties
        assert lsb.max().item() <= (0 if method == "nearest" else 1), lsb.max().item()
        pred = rec["out"].squeeze().float()
        want, want_col = ref_marigold_post(pred, (H, W), method, normals, "Spectral", lut)
        got = out.normal_np if normals else out.depth_np
        err = float(np.abs(got - want).max())
        print("marigold", method, processing_res, "normals" if normals else "depth", "max_abs", err,
              "input_lsb_fraction", (lsb > 0).float().mean().item())
        if method == "nearest" and not normals:
            assert err == 0.0
        else:
            # fp32 sums of the antialiased resize / the normal's length in another order than torch's
            assert err <= (1e-6 if method == "nearest" else 3e-5), err
        col = out.normal_colored if normals else out.depth_colored
        assert isinstance(col, Image.Image) and col.size == (W, H)
        want_col = np_colorize_normals(got) if normals else mpl_colorize_depth(got, lut)
        np.testing.assert_array_equal(np.asarray(col), want_col)


def test_marigold_bilinear_outputs_unchanged_by_colouring(tiny):
    """The colour fields are filled without touching depth_np: color_map None and "Spectral" give the same array."""
    import make_golden as MG
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    unet, vae = tiny
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=MG.inputs(5, 1, 2, 128, scale=0.5).to(DEV))
    a = pipe(IMG, denoising_steps=1, ensemble_size=1, processing_res=80, noise="zeros", color_map=None)
    b = pipe(IMG, denoising_steps=1, ensemble_size=1, processing_res=80, noise="zeros")
    assert a.depth_colored is None and b.depth_colored is not None
    np.testing.assert_array_equal(a.depth_np, b.depth_np)


@pytest.fixture(scope="module")
def tiny_geowizard():
    import engine_checks as E
    import make_golden as MG
    gunet_ref, vae_ref = MG.build_tiny("geowizard")
    return E.engine_from_oracle(gunet_ref, vae_ref, DEV)


@pytest.mark.parametrize("processing_res", [80, 160])
def test_geowizard_call_colours_and_ensemble_kwargs(tiny_geowizard, processing_res, monkeypatch):
    import make_golden as MG
    from PIL import Image
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline, pipelines
    unet, vae = tiny_geowizard
    pipe = DepthNormalEstimationPipeline(unet, vae, DDIMScheduler())
    emb = MG.inputs(6, 2, 1, 96, scale=0.5)[:1].to(DEV)
    seen = []
    real = pipelines.ensemble_depths
    monkeypatch.setattr(pipelines, "ensemble_depths", lambda x, **kw: seen.append(kw) or real(x, **kw))
    kw = dict(reduction="mean", max_iter=3)
    out = pipe(IMG, ensemble_size=3, processing_res=processing_res, color_map="Spectral", img_embed=emb,
               noise="gaussian", ensemble_kwargs=kw)
    assert seen == [kw]
    H, W = IMG.shape[-2:]
    assert out.depth_np.shape == (H, W) and out.normal_np.shape == (3, H, W)
    for img, want in ((out.depth_colored, mpl_colorize_depth(out.depth_np, mpl_spectral_lut())),
                      (out.normal_colored, np_colorize_normals(out.normal_np))):
        assert isinstance(img, Image.Image) and img.size == (W, H)
        np.testing.assert_array_equal(np.asarray(img), want)
    # the defaults: no depth colouring, normals always coloured, depth_np as without colouring
    base = pipe(IMG, processing_res=processing_res, img_embed=emb)
    assert base.depth_colored is None and isinstance(base.normal_colored, Image.Image)
    np.testing.assert_array_equal(np.asarray(base.normal_colored), np_colorize_normals(base.normal_np))
