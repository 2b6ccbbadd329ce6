"""-m gpu: the vectorised swapped epilogue of gemm_conv_kernel, which works straight from the wgmma accumulator registers.

* Per-tap swapped path: its outputs must be bit-identical to the staged epilogue (debug flag 64 selects it) on the same
  tile geometry, because both apply the same per-element arithmetic in the same order to the same accumulators.
* Fused statistics: per-(image, channel) sums carried across a CTA's consecutive tiles, against an fp64 reduction of
  what was stored.
* Halo path: against torch and against the per-tap path (different summation order, so within the conv tolerances)."""
import math

import pytest
import torch
import torch.nn.functional as F

from diffusion_e2e_ft_b200 import ops
from kernel_checks import _conv_ref, _rand, rel_l2

FLAG_STAGED = 64        # swapped orientation without the vectorised epilogue
FLAG_VEC_LINEAR = 128   # vectorised epilogue for a linear layer without fused statistics


def _run(flags, fn):
    L = ops._lib.load()
    L.b200_debug_set_flags(flags)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        L.b200_debug_set_flags(0)
    return out


def _per_tap_swapped(fn):
    """fn() on the per-tap path with 256-pixel swapped tiles, once with the vectorised and once with the staged epilogue."""
    L = ops._lib.load()
    L.b200_debug_set_halo(0)
    L.b200_debug_force_block_n(256)
    try:
        return _run(0, fn), _run(FLAG_STAGED, fn)
    finally:
        L.b200_debug_force_block_n(0)
        L.b200_debug_set_halo(1)


CONV_CASES = {
    # name: (NB, H, W, Cin, Cout, out_f32, residual, act, rowvec, f16_copy, shortcut)
    "ragged_320_f32_res_silu_twin": (2, 15, 21, 64, 320, True, True, ops.ACT_SILU, False, True, 0),
    "ragged_320_f16_gelu_rowvec": (2, 17, 19, 128, 320, False, False, ops.ACT_GELU, True, False, 0),
    "f16_res_rowvec": (2, 24, 40, 128, 256, False, True, ops.ACT_NONE, True, False, 0),
    "f32_shortcut_twin": (1, 20, 36, 128, 128, True, False, ops.ACT_NONE, False, True, 128),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONV_CASES))
def test_vec_epilogue_bit_identical_conv(name):
    NB, H, W, Cin, Cout, out_f32, residual, act, rowvec, f16_copy, shortcut = CONV_CASES[name]
    seed = 300 + sorted(CONV_CASES).index(name) * 10
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, Cin, 3, 3, seed=seed + 1, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    odt = torch.float32 if out_f32 else torch.float16
    res = _rand(NB, H, W, Cout, seed=seed + 3, dtype=odt) if residual else None
    rv = _rand(NB, Cout, seed=seed + 4, dtype=torch.float32) if rowvec else None
    x2 = _rand(NB, H, W, shortcut, seed=seed + 5) if shortcut else None
    ws = _rand(Cout, shortcut, 1, 1, seed=seed + 6, scale=1.0 / math.sqrt(shortcut)) if shortcut else None
    wp = ops.pack_conv(w, ws)
    fn = lambda: ops.conv2d(x, wp, Cout, bias=b, x2=x2, rowvec=rv, residual=res, out_dtype=odt, act=act,
                            stats=True, f16_copy=f16_copy)
    vec, staged = _per_tap_swapped(fn)
    assert torch.equal(vec, staged), f"max |diff| {(vec.float() - staged.float()).abs().max().item():.3e}"
    if f16_copy:
        assert torch.equal(vec._h16, staged._h16)
        assert torch.equal(vec._h16, vec.half())
    # the statistics differ from the staged path's only in summation order
    assert rel_l2(vec._cs, staged._cs) < 1e-6
    ref = _conv_ref(x, w, b, 1, "same")
    if shortcut:
        ref = ref + F.conv2d(x2.float().permute(0, 3, 1, 2), ws.float())
    if rowvec:
        ref = ref + rv[:, :, None, None]
    if residual:
        ref = ref + res.float().permute(0, 3, 1, 2)
    ref = {ops.ACT_SILU: F.silu, ops.ACT_GELU: F.gelu}.get(act, lambda t: t)(ref)
    assert rel_l2(vec.permute(0, 3, 1, 2), ref) < (3e-5 if out_f32 else 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("out_f32", [False, True])
def test_vec_epilogue_bit_identical_linear_res_mul(out_f32):
    """Swapped linear layer with a multiplicative residual operand and a ragged channel tile (N = 960)."""
    M, N, K = 1000, 960, 320
    a = _rand(M, K, seed=401)
    w = _rand(N, K, seed=402, scale=1.0 / math.sqrt(K))
    b = _rand(N, seed=403, dtype=torch.float32)
    odt = torch.float32 if out_f32 else torch.float16
    gate = _rand(M, N, seed=404, dtype=odt)
    fn = lambda: ops.linear(a, w, b, residual=gate, res_mul=True, out_dtype=odt, act=ops.ACT_GELU)
    L = ops._lib.load()
    L.b200_debug_force_block_n(128)
    try:
        vec, staged = _run(FLAG_VEC_LINEAR, fn), _run(FLAG_STAGED, fn)
    finally:
        L.b200_debug_force_block_n(0)
    assert torch.equal(vec, staged), f"max |diff| {(vec.float() - staged.float()).abs().max().item():.3e}"
    ref = F.gelu(a.float() @ w.float().t() + b) * gate.float()
    assert rel_l2(vec, ref) < (3e-5 if out_f32 else 1e-3)


def _stats_ref(out):
    o = out.double()
    return torch.stack([o.sum((1, 2)), (o * o).sum((1, 2))], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("halo", [0, 2])
@pytest.mark.parametrize("out_f32", [False, True])
def test_vec_epilogue_carried_statistics(halo, out_f32):
    """Many small images and three channel tiles (Cout = 320, the last one half full): a CTA walks several tiles per
    (image, channel tile) and several images, so the sums are carried across tiles and flushed on every key change."""
    NB, H, W, Cin, Cout = 12, 20, 44, 64, 320
    x = _rand(NB, H, W, Cin, seed=501)
    w = _rand(Cout, Cin, 3, 3, seed=502, scale=1.0 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=503, dtype=torch.float32)
    odt = torch.float32 if out_f32 else torch.float16
    L = ops._lib.load()
    L.b200_debug_set_halo(halo)
    try:
        out = ops.conv2d(x, ops.pack_conv(w), Cout, bias=b, out_dtype=odt, stats=True)
        torch.cuda.synchronize()
        assert L.b200_debug_last_path() == (1 if halo else 0)
    finally:
        L.b200_debug_set_halo(1)
    want = _stats_ref(out)
    assert rel_l2(out._cs, want) < 1e-6
    # every (image, channel) entry, not just the aggregate: a missed or doubled flush shows up here
    assert ((out._cs[..., 1] - want[..., 1]).abs() / want[..., 1]).max().item() < 1e-5


@pytest.mark.gpu
def test_halo_vec_epilogue_upsample_phases():
    """Halo path with the 4-phase upsample (out_mul = 2, shared statistics across the four launches) against the per-tap
    path and against nearest-2x + conv in torch."""
    from diffusion_e2e_ft_b200.modules import Upsample2D
    NB, H, W, C = 2, 18, 30, 128
    m = Upsample2D(C).to("cuda")
    xs = _rand(NB, H, W, C, seed=601, dtype=torch.float32)
    L = ops._lib.load()
    ys = []
    with torch.no_grad():
        for halo in (2, 0):
            L.b200_debug_set_halo(halo)
            try:
                ys.append(m.run(xs, None, torch.float32))
                torch.cuda.synchronize()
                assert L.b200_debug_last_path() == (1 if halo else 0)
            finally:
                L.b200_debug_set_halo(1)
        up = F.interpolate(xs.half().double().cpu().permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
        ref = F.conv2d(up, m.conv.weight.double().cpu(), m.conv.bias.double().cpu(), padding=1).permute(0, 2, 3, 1)
    assert rel_l2(ys[0], ys[1]) < 3e-5
    assert rel_l2(ys[0].cpu(), ref) < 2e-3          # the kernels use fp16 weights (phase sums rounded once)
    if getattr(ys[0], "_cs", None) is not None:
        assert rel_l2(ys[0]._cs, _stats_ref(ys[0])) < 1e-6
