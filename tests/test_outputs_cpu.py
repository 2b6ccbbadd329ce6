"""CPU tests of the pipelines' resampling choice and colour outputs: argument errors raised before any launch, the
built-in Spectral table against a restatement of matplotlib, and both pipelines' `__call__` with the device kernels
emulated in torch, against a restatement of the reference's post-processing on the same predictions (torchvision
`resize` + numpy clip + numpy colouring).  The kernels themselves are checked on the GPU (tests/test_outputs_gpu.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from outputs_reference import (mpl_colorize_depth, mpl_spectral_lut, np_colorize_normals, ref_marigold_post,
                               ref_marigold_pre, special_depths)


# ------------------------------------------------------------------------------------------------ the Spectral table
def test_spectral_table_matches_matplotlib_restated():
    from diffusion_e2e_ft_b200 import ensemble
    want = mpl_spectral_lut()
    got = ensemble.spectral_lut()
    assert got.shape == (256, 3) and got.dtype == np.float64
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal((got * 255).astype(np.uint8), (want * 255).astype(np.uint8))


def test_spectral_end_colours_survive_the_float64_truncation():
    from diffusion_e2e_ft_b200 import ensemble
    table = (ensemble.spectral_lut() * 255).astype(np.uint8)
    assert tuple(table[0]) == (158, 1, 66) and tuple(table[-1]) == (94, 79, 162)


def _emulated_colorize_depth(x, cmap="Spectral"):
    """The b200_colorize_depth contract (include/b200_e2eft.h) on the host's uint8 table."""
    from diffusion_e2e_ft_b200 import ensemble
    ensemble.check_color_map(cmap)
    table = torch.from_numpy((ensemble.spectral_lut() * 255).astype(np.uint8))
    v = x.float().reshape(x.shape[-2:])
    bad = torch.isnan(v)
    k = (v.clamp(0, 1) * torch.tensor(table.shape[0], dtype=torch.float32)).nan_to_num(0).long()
    k = k.clamp(max=table.shape[0] - 1)
    out = table[k]
    out[bad] = 0
    return out


def _emulated_colorize_normals(x):
    """The b200_colorize_normals contract: each fp32 operation rounded on its own, truncated, NaN -> 0."""
    v = x.float().clamp(-1, 1)
    u = (((v + 1) / 2) * 255).nan_to_num(0).to(torch.uint8)
    return u.permute(1, 2, 0).contiguous()


def test_colour_contracts_match_numpy_restatements():
    """The folded uint8 table indexed at (int)(clip(x) * 256) is the reference's float64 colouring, at 0, 1, every
    k/256 boundary, outside the range and at NaN; the normals rule is numpy's float32 expression."""
    lut = mpl_spectral_lut()
    d = special_depths()
    d = np.concatenate([d, np.zeros(-len(d) % 16, np.float32)]).reshape(8, -1)
    got = _emulated_colorize_depth(torch.from_numpy(d)).numpy()
    np.testing.assert_array_equal(got, mpl_colorize_depth(d, lut))
    n = np.random.default_rng(0).uniform(-1.3, 1.3, (3, 8, 40)).astype(np.float32)
    n.reshape(-1)[:len(d.reshape(-1)) // 2] = (d.reshape(-1)[:len(d.reshape(-1)) // 2] * 2 - 1)
    n[0, 0, 0], n[1, 0, 1], n[2, 0, 2] = np.nan, -1.0, 1.0
    np.testing.assert_array_equal(_emulated_colorize_normals(torch.from_numpy(n)).numpy(), np_colorize_normals(n))


# ------------------------------------------------------------------------------------------------ argument errors
class _NoLaunch(torch.nn.Module):
    """A module that fails the test if anything tries to run it."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def forward(self, *a, **k):
        raise AssertionError("launched before the argument check")

    encode_scaled_mean = forward


def test_argument_errors_before_any_launch():
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline, MarigoldPipeline, ensemble
    mari = MarigoldPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler(), empty_text_embed=torch.zeros(1, 2, 128))
    img = torch.zeros(3, 16, 16, dtype=torch.uint8)
    for m in ("lanczos", "nearest-exact", "BILINEAR", None):
        with pytest.raises(ValueError, match="Unknown resampling method"):
            mari(img, resample_method=m)
    for cm in ("viridis", "spectral", "jet"):
        with pytest.raises(ValueError, match="only 'Spectral' is built in"):
            mari(img, color_map=cm)
    geo = DepthNormalEstimationPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler())
    with pytest.raises(ValueError, match="only 'Spectral' is built in"):
        geo(img, color_map="magma", img_embed=torch.zeros(1, 1, 96))
    with pytest.raises(ValueError, match="only 'Spectral' is built in"):
        ensemble.colorize_depth(torch.zeros(4, 4), cmap="jet")         # before the CUDA check, so a ValueError
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.colorize_depth(torch.zeros(4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.colorize_normals(torch.zeros(3, 4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.resize_nearest_exact(torch.zeros(3, 4, 4), (5, 7))


# ------------------------------------------------------------------------------------------------ pipelines, emulated
def _interp(x, size, mode):
    x = x.float()
    lead = x.shape[:-2]
    y = x.reshape(1, -1, *x.shape[-2:])
    kw = dict(align_corners=False, antialias=True) if mode in ("bilinear", "bicubic") else {}
    return F.interpolate(y, size=tuple(int(s) for s in size), mode=mode, **kw).reshape(*lead, int(size[0]), int(size[1]))


def _install(monkeypatch, calls):
    """Emulate every device op the two __call__s use, on the pipelines module (which imported them by name)."""
    import cpu_emulation
    from diffusion_e2e_ft_b200 import ops, pipelines as P

    def minmax_normalise_(x):
        lo, hi = x.min(), x.max()
        return (x - lo) / (hi - lo), torch.stack([lo, hi])

    def ensemble_depths(preds, **kw):
        calls.append(("ensemble_depths", kw))
        return preds.median(0).values, preds.std(0)

    def ensemble_normals(preds):
        calls.append(("ensemble_normals", {}))
        return preds[1], None

    def normalise_rgb(rgb, round_u8=False):
        x = rgb.float()
        if round_u8:
            x = x.round().clamp(0, 255)
        return x / 255.0 * 2.0 - 1.0

    def colorize_depth(x, cmap="Spectral"):
        calls.append(("colorize_depth", x))
        return _emulated_colorize_depth(x, cmap)

    def colorize_normals(x):
        calls.append(("colorize_normals", x))
        return _emulated_colorize_normals(x)

    monkeypatch.setattr(ops, "decode_post", cpu_emulation.decode_post)
    for name, fn in dict(resize_bilinear_aa=lambda x, s: _interp(x, s, "bilinear"),
                         resize_bicubic_aa=lambda x, s: _interp(x, s, "bicubic"),
                         resize_nearest_exact=lambda x, s: _interp(x, s, "nearest-exact"),
                         resize_nearest=lambda x, s: x[:, cpu_emulation._nearest_index(x.shape[1], s[0])][
                             :, :, cpu_emulation._nearest_index(x.shape[2], s[1])],
                         normalise_rgb=normalise_rgb, minmax_normalise_=minmax_normalise_,
                         minmax_rows=lambda x: torch.stack([x.min(1).values, x.max(1).values], 1),
                         ensemble_depths=ensemble_depths, ensemble_normals=ensemble_normals,
                         colorize_depth=colorize_depth, colorize_normals=colorize_normals).items():
        monkeypatch.setattr(P, name, fn)


def _fake_infer(record, channels):
    """single_infer stand-in: a seeded prediction of the batch's shape, the batch recorded."""
    def single_infer(rgb_in, *a, **k):
        record.append(rgb_in.clone())
        B, _, h, w = rgb_in.shape
        g = torch.Generator().manual_seed(h * 1000 + w + len(record))
        return torch.rand(B, channels, h, w, generator=g) * 2 - 1
    return single_infer


@pytest.mark.parametrize("method", ["bilinear", "bicubic", "nearest"])
@pytest.mark.parametrize("processing_res", [24, 80])
@pytest.mark.parametrize("normals", [False, True])
def test_marigold_call_matches_reference_postprocessing(monkeypatch, method, processing_res, normals):
    from PIL import Image
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    calls, seen = [], []
    _install(monkeypatch, calls)
    pipe = MarigoldPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler(), empty_text_embed=torch.zeros(1, 2, 128))
    preds = []
    fake = _fake_infer(seen, 3 if normals else 1)
    pipe.single_infer = lambda *a, **k: preds.append(fake(*a, **k)) or preds[-1]
    img = torch.randint(0, 256, (3, 37, 53), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    ens = 3
    out = pipe(img, denoising_steps=1, ensemble_size=ens, processing_res=processing_res, resample_method=method,
               ensemble_kwargs=dict(reduction="median"), normals=normals)
    # the input side: the batch single_infer saw is the reference's resized, normalised image
    want_in = ref_marigold_pre(img, processing_res, method)
    got_in = seen[0][0]
    assert got_in.shape == want_in.shape and seen[0].shape[0] == ens
    lsb = (got_in - want_in).abs().max().item() * 255 / 2
    # torchvision resizes a uint8 image bilinearly in its own uint8 arithmetic on the CPU (1 LSB from the float
    # resize); the bicubic and nearest-exact resizes go through float and round back, exactly as the engine does
    assert lsb <= (1.0001 if method == "bilinear" else 0.0), lsb
    # the output side, on the same (emulated) ensembled prediction
    stacked = torch.cat(preds).squeeze()
    pred = stacked[1] if normals else stacked.median(0).values
    want, want_col = ref_marigold_post(pred, (37, 53), method, normals, "Spectral", mpl_spectral_lut())
    got = out.normal_np if normals else out.depth_np
    np.testing.assert_array_equal(got, want)
    col = out.normal_colored if normals else out.depth_colored
    assert isinstance(col, Image.Image) and col.size == (53, 37) and col.mode == "RGB"
    np.testing.assert_array_equal(np.asarray(col), want_col)
    assert (out.depth_colored if normals else out.normal_colored) is None
    # colours come from the very device tensor that becomes the numpy output
    src = [c[1] for c in calls if c[0].startswith("colorize")]
    assert len(src) == 1 and np.array_equal(src[0].numpy().clip(*((-1, 1) if normals else (0, 1))), got)
    if not normals:
        assert ("ensemble_depths", dict(reduction="median")) in calls
        assert out.uncertainty is not None


def test_marigold_color_map_none_and_no_resize(monkeypatch):
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    calls, seen = [], []
    _install(monkeypatch, calls)
    pipe = MarigoldPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler(), empty_text_embed=torch.zeros(1, 2, 128))
    pipe.single_infer = _fake_infer(seen, 1)
    img = torch.randint(0, 256, (3, 30, 20), dtype=torch.uint8, generator=torch.Generator().manual_seed(2))
    out = pipe(img, ensemble_size=1, processing_res=16, color_map=None, resample_method="nearest")
    assert out.depth_colored is None and out.normal_colored is None
    assert not [c for c in calls if c[0].startswith("colorize")]
    out = pipe(img, ensemble_size=1, processing_res=16, match_input_res=False, resample_method="bicubic")
    assert out.depth_np.shape == (16, 10) and np.asarray(out.depth_colored).shape == (16, 10, 3)
    np.testing.assert_array_equal(np.asarray(out.depth_colored), mpl_colorize_depth(out.depth_np, mpl_spectral_lut()))


@pytest.mark.parametrize("color_map", [None, "Spectral"])
def test_geowizard_call_colours_and_ensemble_kwargs(monkeypatch, color_map):
    from PIL import Image
    from diffusion_e2e_ft_b200 import DDIMScheduler, DepthNormalEstimationPipeline
    calls, seen = [], []
    _install(monkeypatch, calls)
    pipe = DepthNormalEstimationPipeline(_NoLaunch(), _NoLaunch(), DDIMScheduler())
    fd, fn = _fake_infer(seen, 1), _fake_infer([], 3)
    pipe.single_infer = lambda batch, *a, **k: (fd(batch), fn(batch) * 1.2)        # normals partly outside [-1, 1]
    img = torch.randint(0, 256, (3, 37, 53), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    kw = dict(reduction="mean", regularizer_strength=0.05, max_iter=3)
    out = pipe(img, ensemble_size=3, processing_res=24, color_map=color_map, img_embed=torch.zeros(1, 1, 96),
               ensemble_kwargs=kw)
    assert ("ensemble_depths", kw) in calls
    assert out.depth_np.shape == (37, 53) and out.normal_np.shape == (3, 37, 53)
    assert isinstance(out.normal_colored, Image.Image) and out.normal_colored.size == (53, 37)
    np.testing.assert_array_equal(np.asarray(out.normal_colored), np_colorize_normals(out.normal_np))
    if color_map is None:
        assert out.depth_colored is None
    else:
        assert isinstance(out.depth_colored, Image.Image)
        np.testing.assert_array_equal(np.asarray(out.depth_colored),
                                      mpl_colorize_depth(out.depth_np, mpl_spectral_lut()))
    # without ensemble_kwargs the reference's defaults apply
    calls.clear()
    pipe(img, ensemble_size=2, processing_res=24, img_embed=torch.zeros(1, 1, 96))
    assert ("ensemble_depths", {}) in calls
