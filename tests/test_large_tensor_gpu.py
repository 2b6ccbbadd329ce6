"""-m gpu: the VAE decoder's tensors of more than 2^31 elements, element by element on row bands against fp64.

At the per-image limit (pipelines._check_image_size: 256 H W < 2^32), H x W = 3640 x 4608, the last decoder up block
produces 256-channel full-resolution tensors of 4 293 918 720 elements.  This runs the engine's own modules on them in
the decoder's fp32 stream mode:
  * Upsample2D(256).run from a 1820 x 2304 x 256 input: four out_mul = 2 phase convs sharing one statistics buffer;
  * then the steps of ResnetBlock2D(256 -> 128).run (its fp32-stream branch, restated so the intermediates can be
    checked): GroupNorm + SiLU with the fp16 raw copy, conv1 on the 256-channel input, GroupNorm 2 + SiLU, and conv2
    with the raw copy as the 256-channel 1x1 shortcut operand.
Each output is compared on row bands with an fp64 reference computed from the kernels' own fp16 inputs of that step
(band plus its 1-row halo): the first rows, the rows holding element 2^31 of the 256-channel tensors, the last rows
(offsets just below 2^32) and, for an NB = 2 batch of the same total size, the rows on both sides of the image
boundary.  GroupNorm statistics of the reference come from a chunked fp64 reduction over the whole tensor, which also
checks the fused per-(image, channel) sums of every producer.  The convs are held to the per-element bound of
tests/gemm_geometry.py, the GroupNorm outputs to fp16 rounding plus a small slack for the fp32 normalisation.

Peak device memory measured on an H100 80GB HBM3 (700 W): 32.3 GB for NB = 1, 32.2 GB for NB = 2 (the 17.2 GB fp32 upsample
output, the 8.6 GB fp16 normalised tensor and the 8.6 GB raw copy live together).  Each test skips when the device has
less than 40 GB free."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_geometry as G  # noqa: E402
from diffusion_e2e_ft_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu

GB = 1024 ** 3
NEED = 40 * GB


def _need_free(nbytes, what):
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB free; the device has {free / GB:.1f} of {total / GB:.1f} GB free")


def _chunked_sums(t, rows=32):
    """Per-(image, channel) fp64 [sum, sum of squares, sum of |v|, max |v|] of an NHWC tensor, in row chunks."""
    NB, H, W, C = t.shape
    s = torch.zeros(NB, C, 4, dtype=torch.float64, device=t.device)
    for r in range(0, H, rows):
        c = t[:, r:r + rows].double()
        s[..., 0] += c.sum((1, 2))
        s[..., 1] += (c * c).sum((1, 2))
        s[..., 2] += c.abs().sum((1, 2))
        s[..., 3] = torch.maximum(s[..., 3], c.abs().amax((1, 2)))
        del c
    return s


def _check_cs(cs, want, npix, what):
    """Fused sums against the fp64 reduction, with the tolerances of gemm_geometry.check_stats."""
    tol1 = 1e-5 * (want[..., 2] + npix * want[..., 3]) + 1e-30
    r1 = ((cs[..., 0] - want[..., 0]).abs() / tol1).max().item()
    r2 = ((cs[..., 1] - want[..., 1]).abs() / (1e-5 * want[..., 1] + 1e-30)).max().item()
    assert r1 <= 1.0 and r2 <= 1.0, f"{what}: fused statistics off (sum ratio {r1:.3g}, sum-of-squares ratio {r2:.3g})"


def _band(x, img, lo, hi, halo):
    """Rows [lo - halo, hi + halo) of image img, zero rows outside the image, columns zero padded by halo: fp64."""
    H = x.shape[1]
    a, b = max(lo - halo, 0), min(hi + halo, H)
    xb = x[img, a:b].double()
    return torch.nn.functional.pad(xb, (0, 0, halo, halo, a - (lo - halo), (hi + halo) - b))


def _band_conv(x, w_taps, taps, img, lo, hi, x2=None, w2=None):
    """fp64 stride-1 tap conv (taps in -1..1) of rows [lo, hi) of image img, and the same on |x|, |w|."""
    xb = _band(x, img, lo, hi, 1)              # [hi - lo + 2, W + 2, Cin]
    W = x.shape[2]
    wd = w_taps.double()
    ref = 0.0
    absref = 0.0
    for t, (dy, dx) in enumerate(taps):
        xs = xb[1 + dy:1 + dy + hi - lo, 1 + dx:1 + dx + W]
        ref = ref + xs @ wd[:, t].t()
        absref = absref + xs.abs() @ wd[:, t].abs().t()
    if x2 is not None:
        x2b = x2[img, lo:hi].double()
        ref = ref + x2b @ w2.double().t()
        absref = absref + x2b.abs() @ w2.double().abs().t()
    return ref, absref


def _gn_ref(xb, sums, img, gamma, beta, groups, npix, eps):
    """fp64 GroupNorm + SiLU of a band with statistics from the whole-tensor fp64 sums."""
    C = xb.shape[-1]
    cg = C // groups
    gs = sums[img, :, :2].reshape(groups, cg, 2).sum(1)
    n = npix * cg
    mean = gs[:, 0] / n
    var = gs[:, 1] / n - mean * mean
    rstd = 1.0 / torch.sqrt(var + eps)
    mc = mean.repeat_interleave(cg)
    rc = rstd.repeat_interleave(cg)
    pre = (xb - mc) * rc * gamma.double() + beta.double()
    return torch.nn.functional.silu(pre), pre


def _check_gn(y, x, sums, img, lo, hi, gamma, beta, eps, what):
    ref, pre = _gn_ref(x[img, lo:hi].double(), sums, img, gamma, beta, 32, x.shape[1] * x.shape[2], eps)
    # fp16 rounding of the output, plus fp32 normalisation and __expf in SiLU: 2^-16 (1 + |pre|)
    bound = 2.0 ** -11 * ref.abs() + 2.0 ** -16 * (1.0 + pre.abs()) + 2.0 ** -25
    return G.check_bound(y[img, lo:hi], ref, bound, what)[0]


def _bands(NB, H, W, C):
    """(img, lo, hi) row bands: first rows, the rows holding element 2^31 of a C-channel tensor, the last rows, and
    around each image boundary."""
    per_img = H * W * C
    out = [(0, 0, 3), (NB - 1, H - 3, H)]
    e = 2 ** 31
    img, pix = e // per_img, (e % per_img) // C
    r = pix // W
    out.append((img, max(r - 1, 0), min(r + 2, H)))
    for i in range(1, NB):
        out += [(i - 1, H - 2, H), (i, 0, 2)]
    return sorted(set(out))


def _run(NB, h, w, seed):
    from diffusion_e2e_ft_b200.modules import ResnetBlock2D, Upsample2D
    _need_free(NEED, f"the {NB} x {2 * h} x {2 * w} x 256 decoder tensors")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(seed)
    C, Co = 256, 128
    up_m = Upsample2D(C).to("cuda")
    rb = ResnetBlock2D(C, Co, temb_channels=None).to("cuda")
    with torch.no_grad():
        for gn in (rb.norm1, rb.norm2):
            gn.weight.normal_(1.0, 0.3)
            gn.bias.normal_(0.0, 0.3)
    H, W = 2 * h, 2 * w
    bands = _bands(NB, H, W, C)
    worst = {}
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        x = torch.randn(NB, h, w, C, device="cuda", generator=g, dtype=torch.float16)
        # ---- Upsample2D: four phase convs into one fp32 tensor, statistics summed into one buffer
        up = up_m.run(x, None, torch.float32)
        pk = up_m._packed_phases()
        bias = pk["b"].double()
        for img, lo, hi in bands:
            ref = torch.empty(hi - lo, W, C, dtype=torch.float64, device="cuda")
            bound = torch.empty_like(ref)
            for (py, px), (taps, wp) in pk["ph"].items():
                r0 = lo + ((py - lo) % 2)                     # first output row of this parity in the band
                if r0 >= hi:
                    continue
                i0, i1 = r0 // 2, (hi - 1 - py) // 2 + 1      # low-resolution rows of those outputs
                acc, absacc = _band_conv(x, wp.view(C, len(taps), C), taps, img, i0, i1)
                rr, bd = G.conv_bound(acc + bias, absacc, len(taps) * C, True, extra_abs=bias.abs())
                ref[r0 - lo::2, px::2], bound[r0 - lo::2, px::2] = rr, bd
            worst["upsample"] = max(worst.get("upsample", 0.0),
                                    G.check_bound(up[img, lo:hi], ref, bound, f"upsample rows {lo}:{hi} of image {img}")[0])
        del x
        s_up = _chunked_sums(up)
        _check_cs(up._cs, s_up, H * W, "upsample")
        # ---- ResnetBlock2D(256 -> 128).run on an fp32 stream with a 1x1 shortcut: its GN-with-raw-copy branch
        p = rb._packed()
        a1, raw = ops.group_norm(up, p["g1"], p["b1"], rb.eps, rb.groups, True, want_raw=True)
        for img, lo, hi in bands:
            assert torch.equal(raw[img, lo:hi], up[img, lo:hi].half()), f"raw copy rows {lo}:{hi} of image {img}"
            worst["gn1"] = max(worst.get("gn1", 0.0), _check_gn(a1, up, s_up, img, lo, hi, p["g1"], p["b1"], rb.eps,
                                                                 f"GroupNorm 1 rows {lo}:{hi} of image {img}"))
        del up
        hh = ops.conv2d(a1, p["w1"], Co, bias=p["c1b"], stats=True)
        w1 = p["w1"].view(Co, 9, C)
        for img, lo, hi in bands:
            acc, absacc = _band_conv(a1, w1, ops.TAPS3, img, lo, hi)
            b1 = p["c1b"].double()
            ref, bound = G.conv_bound(acc + b1, absacc, 9 * C, False, extra_abs=b1.abs())
            worst["conv1"] = max(worst.get("conv1", 0.0),
                                 G.check_bound(hh[img, lo:hi], ref, bound, f"conv1 rows {lo}:{hi} of image {img}")[0])
        del a1
        s_h = _chunked_sums(hh)
        _check_cs(hh._cs, s_h, H * W, "conv1")
        a2 = ops.group_norm(hh, p["g2"], p["b2"], rb.eps, rb.groups, True)
        for img, lo, hi in bands:
            worst["gn2"] = max(worst.get("gn2", 0.0), _check_gn(a2, hh, s_h, img, lo, hi, p["g2"], p["b2"], rb.eps,
                                                                f"GroupNorm 2 rows {lo}:{hi} of image {img}"))
        del hh
        out = ops.conv2d(a2, p["w2"], Co, bias=p["c2b"], x2=raw, out_dtype=torch.float32, stats=True)
        w2 = p["w2"][:, :9 * Co].reshape(Co, 9, Co)
        ws = p["w2"][:, 9 * Co:]
        for img, lo, hi in bands:
            acc, absacc = _band_conv(a2, w2, ops.TAPS3, img, lo, hi, raw, ws)
            b2 = p["c2b"].double()
            ref, bound = G.conv_bound(acc + b2, absacc, 9 * Co + C, True, extra_abs=b2.abs())
            worst["conv2"] = max(worst.get("conv2", 0.0),
                                 G.check_bound(out[img, lo:hi], ref, bound, f"conv2 rows {lo}:{hi} of image {img}")[0])
        _check_cs(out._cs, _chunked_sums(out), H * W, "conv2")
        del a2, raw, out
    peak = torch.cuda.max_memory_allocated() / GB
    print(f"\nNB={NB} {H}x{W}: bands {bands}, worst |error| / bound {worst}, peak {peak:.1f} GB")
    torch.cuda.empty_cache()
    return worst


def test_decoder_tensors_at_the_per_image_limit():
    """One 3640 x 4608 image: 256 H W = 4 293 918 720 < 2^32."""
    assert 256 * 3640 * 4608 < 2 ** 32 < 256 * 3640 * 4608 + 256 * 4608
    _run(1, 1820, 2304, seed=71)


def test_decoder_tensors_batch_of_two_just_under_2_32():
    """Two 2560 x 3276 images (256 NB H W = 4 293 918 720): element 2^31 lies at the start of the second image, so the
    image index enters every offset past it."""
    assert 256 * 2 * 2560 * 3276 < 2 ** 32
    _run(2, 1280, 1638, seed=73)
