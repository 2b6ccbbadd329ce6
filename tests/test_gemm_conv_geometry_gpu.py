"""-m gpu: the implicit-GEMM conv / GEMM kernel at every tile geometry class its dispatcher picks, element by element
against an fp64 reference.

Every case asserts, through `b200_debug_last_launch`, that the kernel took the instantiation and tile the Python
restatement of the dispatcher (tests/gemm_geometry.py) predicts, then checks each output element against the bound
written in gemm_geometry.py (`conv_bound`): a missing tap, a wrong border pixel or a dropped epilogue term violates it by
orders of magnitude at any image size, where a whole-tensor rel-L2 (still reported) dilutes it.  Fused statistics are
checked per (image, channel) against an fp64 reduction of what was stored.  The last test fails if any of the 28
instantiations or any of the four halo MMA widths was never launched by the cases before it.

Cases (the CPU test tests/test_gemm_geometry_cpu.py checks that the list covers these classes):
  * halo-resident conv at MMA widths 64 / 128 / 192 / 256, bh = 1 and the largest bh (23), Wo = bw, Wo one past a tile
    multiple, patches within 20 pixels of kHaloMaxPatchPix, a multi-wave launch carrying statistics across tiles, and
    the out_mul = 2 phases of nearest-2x + conv sharing one statistics buffer;
  * per-tap swapped tiles of 64 / 128 / 256 pixels, stride 1 and stride 2 with both pad modes, with the vectorised and
    the staged epilogue;
  * normal-orientation tiles of 32 / 64 / 128 / 160 / 256 channels;
  * linear layers: normal, swapped, every GEGLU width, and the fused-statistics `proj_out` GEMM (rows_per_img % 128 = 64
    forces the 64-pixel swapped tile).
Each runs with fp16 and fp32 output (GEGLU: fp16 only)."""
import math
import os
import sys
import time
from contextlib import contextmanager
from ctypes import c_int

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_geometry as G  # noqa: E402
from diffusion_e2e_ft_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu

FLAG_STAGED = 64            # swapped orientation with the staged (non-vectorised) epilogue
TAPS = {"same": ops.TAPS3, "pad0": ops.TAPS3_PAD0}

LAUNCHES = []               # every record the cases below launched, for the coverage test
REPORT = {}                 # geometry class -> worst error / bound ratio
T0 = time.time()


def _rand(*shape, seed=0, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to("cuda")


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def last_launch():
    buf = (c_int * len(G.FIELDS))()
    n = ops._lib.load().b200_debug_last_launch(buf, len(G.FIELDS))
    assert n == len(G.FIELDS)
    return dict(zip(G.FIELDS, list(buf)))


@contextmanager
def dispatch(halo=1, force_bn=0, flags=0):
    L = ops._lib.load()
    L.b200_debug_set_halo(halo)
    L.b200_debug_force_block_n(force_bn)
    L.b200_debug_set_flags(flags)
    try:
        yield
    finally:
        L.b200_debug_set_flags(0)
        L.b200_debug_force_block_n(0)
        L.b200_debug_set_halo(1)


def expect_launch(pred, what):
    rec = last_launch()
    LAUNCHES.append(rec)
    assert rec == pred, f"{what}: kernel launched {rec}, the dispatcher restatement predicts {pred}"
    return rec


def _report(cls, ratio):
    REPORT[cls] = max(REPORT.get(cls, 0.0), ratio)


# ------------------------------------------------------------------------------------------------ conv cases
# name: (NB, H, W, Cin, Cout, stride, pad, features).  Features: res, rowvec, act, twin (fp16 copy of an fp32
# output), c2 (1x1 shortcut channels), stats, halo (0 = per-tap, 1 = automatic), bn (forced tile width)
CONV_CASES = {
    # halo-resident: MMA width 64
    "halo64_bh1_wo_eq_bw": (3, 13, 60, 64, 128, 1, "same", dict(act=ops.ACT_SILU, twin=1, stats=1)),
    "halo64_bh2_res": (2, 10, 28, 192, 256, 1, "same", dict(res=1, rowvec=1, stats=1)),
    # width 128 (125 x 1 patch: 384 of the 400 patch pixels)
    "halo128_tight_bh1_shortcut": (4, 2, 125, 64, 128, 1, "same", dict(c2=64, twin=1, stats=1)),
    "halo128_bh3_ragged_cout": (2, 9, 40, 64, 320, 1, "same", dict(act=ops.ACT_GELU, rowvec=1, stats=1)),
    # width 192
    "halo192_tight_res": (2, 4, 93, 192, 128, 1, "same", dict(res=1, stats=1)),
    "halo192_bh4_shortcut_silu": (2, 20, 44, 64, 256, 1, "same", dict(c2=128, act=ops.ACT_SILU, stats=1)),
    # width 256: the 400-pixel patch, Wo = 61 with bh = 4, Wo one past a tile multiple, the largest bh
    "halo256_patch400": (2, 3, 69, 64, 128, 1, "same", dict(rowvec=1, twin=1, stats=1)),
    "halo256_tight_wo61_gelu_res": (2, 4, 61, 192, 128, 1, "same", dict(res=1, act=ops.ACT_GELU, stats=1)),
    "halo256_one_past_tile": (1, 11, 169, 64, 128, 1, "same", dict(act=ops.ACT_SILU, stats=1)),
    "halo256_bh23": (1, 69, 9, 64, 128, 1, "same", dict(twin=1, stats=1)),
    # more tiles than SMs: a CTA carries the statistics across tiles of one (image, channel tile)
    "halo_multiwave_stats": (8, 24, 56, 64, 320, 1, "same", dict(rowvec=1, stats=1)),
    # per-tap swapped tiles (the staged epilogue runs them too, see test_conv_swapped_staged)
    "swap64_s1": (2, 17, 23, 64, 256, 1, "same", dict(halo=0, bn=64, res=1, act=ops.ACT_SILU, stats=1)),
    "swap128_s1": (2, 17, 23, 64, 256, 1, "same", dict(halo=0, bn=128, rowvec=1, c2=64, twin=1, stats=1)),
    "swap256_s1": (2, 17, 23, 64, 320, 1, "same", dict(halo=0, bn=256, act=ops.ACT_GELU, stats=1)),
    "swap64_s2_same": (2, 33, 45, 64, 256, 2, "same", dict(bn=64, rowvec=1, twin=1, stats=1)),
    "swap128_s2_same": (2, 33, 45, 64, 256, 2, "same", dict(bn=128, res=1, stats=1)),
    "swap256_s2_same": (2, 33, 45, 64, 128, 2, "same", dict(bn=256, c2=64, act=ops.ACT_SILU, stats=1)),
    "swap64_s2_pad0": (2, 34, 46, 64, 128, 2, "pad0", dict(bn=64, act=ops.ACT_GELU, stats=1)),
    "swap128_s2_pad0": (2, 34, 46, 64, 256, 2, "pad0", dict(bn=128, rowvec=1, res=1, stats=1)),
    "swap256_s2_pad0": (2, 34, 46, 64, 256, 2, "pad0", dict(bn=256, twin=1, stats=1)),
    # normal orientation (Cout < 128 never swaps)
    "normal32": (2, 15, 21, 64, 96, 1, "same", dict(bn=32, res=1, rowvec=1, stats=1)),
    "normal64_auto": (2, 15, 21, 64, 64, 1, "same", dict(act=ops.ACT_SILU, twin=1, stats=1)),
    "normal128_s2": (2, 29, 41, 64, 96, 2, "same", dict(bn=128, c2=64, stats=1)),
    "normal160": (2, 15, 21, 128, 96, 1, "same", dict(bn=160, act=ops.ACT_GELU, res=1)),
    "normal256_pad0": (2, 30, 42, 64, 96, 2, "pad0", dict(bn=256, rowvec=1, twin=1, stats=1)),
}


def conv_case_plan(name, out_f32, staged=False, sms=132):
    NB, H, W, Cin, Cout, stride, pad, f = CONV_CASES[name]
    taps = TAPS[pad]
    Ho, Wo = (H, W) if stride == 1 else (((H - 1) // 2 + 1, (W - 1) // 2 + 1) if pad == "same"
                                         else ((H - 2) // 2 + 1, (W - 2) // 2 + 1))
    return G.conv_plan(NB, H, W, Cin, Cout, taps, stride, (Ho, Wo), C2=f.get("c2", 0), out_f32=out_f32,
                       residual=bool(f.get("res")), stats=bool(f.get("stats")), sms=sms, halo_mode=f.get("halo", 1),
                       force_bn=f.get("bn", 0), staged=staged), (Ho, Wo)


def run_conv_case(name, out_f32, staged=False, seed=0):
    NB, H, W, Cin, Cout, stride, pad, f = CONV_CASES[name]
    taps = TAPS[pad]
    pred, (Ho, Wo) = conv_case_plan(name, out_f32, staged, _sms())
    odt = torch.float32 if out_f32 else torch.float16
    T, C2 = len(taps), f.get("c2", 0)
    x = _rand(NB, H, W, Cin, seed=seed)
    w = _rand(Cout, T, Cin, seed=seed + 1, scale=1.0 / math.sqrt(T * Cin))
    b = _rand(Cout, seed=seed + 2, dtype=torch.float32)
    rv = _rand(NB, Cout, seed=seed + 3, dtype=torch.float32) if f.get("rowvec") else None
    res = _rand(NB, Ho, Wo, Cout, seed=seed + 4, dtype=odt) if f.get("res") else None
    x2 = _rand(NB, Ho, Wo, C2, seed=seed + 5) if C2 else None
    w2 = _rand(Cout, C2, seed=seed + 6, scale=1.0 / math.sqrt(C2)) if C2 else None
    wp = w.reshape(Cout, T * Cin)
    if C2:
        wp = torch.cat([wp, w2], 1)
    wp = wp.contiguous()
    twin = bool(f.get("twin")) and out_f32
    act = f.get("act", ops.ACT_NONE)
    with dispatch(halo=f.get("halo", 1), force_bn=f.get("bn", 0), flags=FLAG_STAGED if staged else 0):
        out = ops.conv2d(x, wp, Cout, bias=b, taps=taps, stride=stride, out_hw=(Ho, Wo), x2=x2, rowvec=rv,
                         residual=res, out_dtype=odt, act=act, stats=True if f.get("stats") else None, f16_copy=twin)
        torch.cuda.synchronize()
        rec = expect_launch(pred, name)
    acc, absacc = G.tap_conv_ref(x, w, taps, stride, (Ho, Wo), x2, w2)
    pre, extra = acc + b.double(), b.double().abs().expand_as(acc)
    if rv is not None:
        pre, extra = pre + rv.double()[:, None, None, :], extra + rv.double().abs()[:, None, None, :]
    if res is not None:
        pre, extra = pre + res.double(), extra + res.double().abs()
    ref, bound = G.conv_bound(pre, absacc, T * Cin + C2, out_f32, act, extra)
    worst, _ = G.check_bound(out, ref, bound, f"{name} ({'fp32' if out_f32 else 'fp16'} out)")
    if twin:
        assert torch.equal(out._h16, out.half()), f"{name}: fp16 twin differs from the fp32 output rounded to fp16"
    if f.get("stats"):
        G.check_stats(out._cs, out, name)
    cls = ("halo%d" % rec["halo_n"]) if rec["halo"] else G.instantiation(rec)[0] + str(rec["bn"]) + (
        "_s2" if stride == 2 else "")
    _report(cls, worst)
    return out, rec


@pytest.mark.parametrize("out_f32", [False, True], ids=["f16", "f32"])
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv_geometry(name, out_f32):
    run_conv_case(name, out_f32, seed=1000 + 17 * list(CONV_CASES).index(name))


@pytest.mark.parametrize("out_f32", [False, True], ids=["f16", "f32"])
@pytest.mark.parametrize("name", [n for n in CONV_CASES if n.startswith("swap")])
def test_conv_swapped_staged(name, out_f32):
    """The same per-tap swapped tiles through the staged (non-vectorised) epilogue instantiations."""
    run_conv_case(name, out_f32, staged=True, seed=2000 + 17 * list(CONV_CASES).index(name))


@pytest.mark.parametrize("out_f32", [False, True], ids=["f16", "f32"])
@pytest.mark.parametrize("shape", [(2, 10, 28, 128), (2, 9, 40, 128), (1, 12, 61, 128)], ids=["w64", "w128", "w256"])
def test_halo_upsample_phases(shape, out_f32):
    """nearest-2x + conv as four out_mul = 2 phase convs on the low-resolution input, written into one tensor and summed
    into one statistics buffer (Upsample2D.run), at halo widths 64 / 128 / 256."""
    from diffusion_e2e_ft_b200.modules import Upsample2D
    NB, H, W, C = shape
    odt = torch.float32 if out_f32 else torch.float16
    seed = 3000 + H * W
    x = _rand(NB, H, W, C, seed=seed)
    b = _rand(C, seed=seed + 1, dtype=torch.float32)
    out = torch.empty(NB, 2 * H, 2 * W, C, dtype=odt, device="cuda")
    cs = ops._new_stats(NB, C, x.device)
    ref = torch.empty(NB, 2 * H, 2 * W, C, dtype=torch.float64, device="cuda")
    bound = torch.empty_like(ref)
    for i, (py, px) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        taps = [(dy, dx) for dy, _ in Upsample2D._PHASE[py] for dx, _ in Upsample2D._PHASE[px]]
        w = _rand(C, 4, C, seed=seed + 10 + i, scale=1.0 / math.sqrt(4 * C))
        pred = G.conv_plan(NB, H, W, C, C, taps, out_mul=2, out_f32=out_f32, stats=True, sms=_sms())
        with dispatch():
            ops.conv2d(x, w.reshape(C, 4 * C).contiguous(), C, bias=b, taps=taps, out_hw=(H, W), out=out, out_mul=2,
                       out_off=(py, px), stats=cs)
            torch.cuda.synchronize()
            rec = expect_launch(pred, f"phase {py}{px}")
        assert rec["halo"] == 1
        acc, absacc = G.tap_conv_ref(x, w, taps)
        r, bd = G.conv_bound(acc + b.double(), absacc, 4 * C, out_f32, extra_abs=b.double().abs())
        ref[:, py::2, px::2], bound[:, py::2, px::2] = r, bd
    worst, _ = G.check_bound(out, ref, bound, f"upsample phases {shape}")
    G.check_stats(cs, out, f"upsample phases {shape}")
    _report("halo_out_mul2", worst)


# ------------------------------------------------------------------------------------------------ linear cases
def _linear_ref(a, w, b, res, act):
    acc = a.double() @ w.double().t()
    absacc = a.double().abs() @ w.double().abs().t()
    pre, extra = acc + b.double(), b.double().abs().expand_as(acc)
    if res is not None:
        pre, extra = pre + res.double(), extra + res.double().abs()
    return pre, absacc, extra


# name: (M, N, K, act, residual, forced bn, staged)
LINEAR_CASES = {
    "auto_gelu_res": (1000, 320, 320, ops.ACT_GELU, True, 0, False),
    "auto_small_n": (300, 96, 192, ops.ACT_NONE, True, 0, False),
    "swap256_silu": (700, 256, 128, ops.ACT_SILU, False, 256, False),
    "swap64_staged": (333, 384, 192, ops.ACT_NONE, True, 64, True),
}


@pytest.mark.parametrize("out_f32", [False, True], ids=["f16", "f32"])
@pytest.mark.parametrize("name", list(LINEAR_CASES))
def test_linear_geometry(name, out_f32):
    M, N, K, act, residual, bn, staged = LINEAR_CASES[name]
    seed = 4000 + 13 * list(LINEAR_CASES).index(name)
    odt = torch.float32 if out_f32 else torch.float16
    a = _rand(M, K, seed=seed)
    w = _rand(N, K, seed=seed + 1, scale=1.0 / math.sqrt(K))
    b = _rand(N, seed=seed + 2, dtype=torch.float32)
    res = _rand(M, N, seed=seed + 3, dtype=odt) if residual else None
    pred = G.linear_plan(M, N, K, act, out_f32, sms=_sms(), force_bn=bn, staged=staged)
    with dispatch(force_bn=bn, flags=FLAG_STAGED if staged else 0):
        out = ops.linear(a, w, b, residual=res, out_dtype=odt, act=act)
        torch.cuda.synchronize()
        rec = expect_launch(pred, name)
    pre, absacc, extra = _linear_ref(a, w, b, res, act)
    ref, bound = G.conv_bound(pre, absacc, K, out_f32, act, extra)
    worst, _ = G.check_bound(out, ref, bound, name)
    _report("linear_" + G.instantiation(rec)[0] + str(rec["bn"]), worst)


@pytest.mark.parametrize("N", [192, 384, 320, 512], ids=["bn64", "bn128", "bn160", "bn256"])
def test_linear_geglu_widths(N):
    """GEGLU epilogue (out = (x Wv + bv) gelu(x Wg + bg), value / gate halves interleaved per tile) at every tile width."""
    M, K = 300, 320
    seed = 5000 + N
    a = _rand(M, K, seed=seed)
    w = _rand(N, K, seed=seed + 1, scale=1.0 / math.sqrt(K))
    b = _rand(N, seed=seed + 2, dtype=torch.float32)
    wp, bp = ops.pack_geglu(w, b)
    pred = G.linear_plan(M, N, K, G.ACT_GEGLU, False, sms=_sms())
    with dispatch():
        out = ops.linear(a, wp, bp, act=ops.ACT_GEGLU)
        torch.cuda.synchronize()
        expect_launch(pred, f"geglu N={N}")
    pre, absacc, extra = _linear_ref(a, w, b, None, ops.ACT_NONE)
    h = N // 2
    e = (K + 4) * G.U_ACC * (absacc + extra)
    val, gate, ev, eg = pre[:, :h], pre[:, h:], e[:, :h], e[:, h:]
    g = torch.nn.functional.gelu(gate)
    ref = val * g
    e_gate = G.ACT_LIP * eg + 2.0 ** -18 * (1.0 + gate.abs()) ** 2
    bound = G.U_OUT[False] * ref.abs() + (g.abs() + e_gate) * ev + val.abs() * e_gate + 2.0 ** -25
    worst, _ = G.check_bound(out, ref, bound, f"geglu N={N}")
    _report("geglu%d" % G.geglu_block_n(N), worst)


@pytest.mark.parametrize("N", [320, 640, 1280])
@pytest.mark.parametrize("L", [576, 448, 9216])
def test_linear_fused_statistics(L, N):
    """Transformer2DModel's proj_out (modules.py): fp32 output with the residual stream and per-image GroupNorm
    statistics (stats_rows_per_img = L).  L % 128 = 64 (576 is the 24 x 24 latent of a 768^2 input, 448 = 64 x 7)
    leaves only the 64-pixel swapped tile; L = 9216 (96 x 96) lets the cost model choose."""
    NB, K = 2, 320
    M = NB * L
    seed = 6000 + L + N
    a = _rand(M, K, seed=seed)
    w = _rand(N, K, seed=seed + 1, scale=1.0 / math.sqrt(K))
    b = _rand(N, seed=seed + 2, dtype=torch.float32)
    res = _rand(M, N, seed=seed + 3, dtype=torch.float32)
    pred = G.linear_plan(M, N, K, out_f32=True, stats_rows=L, sms=_sms())
    with dispatch():
        out = ops.linear(a, w, b, residual=res, out_dtype=torch.float32, stats_rows_per_img=L)
        torch.cuda.synchronize()
        rec = expect_launch(pred, f"proj_out L={L} N={N}")
    if L % 128 == 64:
        assert rec["swap"] == 1 and rec["bn"] == 64
    pre, absacc, extra = _linear_ref(a, w, b, res, ops.ACT_NONE)
    ref, bound = G.conv_bound(pre, absacc, K, True, extra_abs=extra)
    worst, _ = G.check_bound(out, ref, bound, f"proj_out L={L} N={N}")
    G.check_stats(out._cs, out, f"proj_out L={L} N={N}", per_img_rows=L)
    _report("linear_stats_" + G.instantiation(rec)[0] + str(rec["bn"]), worst)


# ------------------------------------------------------------------------------------------------ coverage
def test_every_instantiation_and_halo_width_launched():
    """Runs after the cases above (file order): each of the 28 instantiations and each halo MMA width must have been
    launched by them, so a change of the cost model cannot leave a path untested."""
    seen = {G.instantiation(r) for r in LAUNCHES}
    widths = {r["halo_n"] for r in LAUNCHES if r["halo"]}
    print(f"\n{len(LAUNCHES)} launches, {len(seen & G.ALL_INSTANTIATIONS)} of 28 instantiations, halo widths "
          f"{sorted(widths)}, {time.time() - T0:.1f} s since import")
    for cls in sorted(REPORT):
        print(f"  worst |error| / bound  {cls:28s} {REPORT[cls]:.3g}")
    missing = sorted(G.ALL_INSTANTIATIONS - seen)
    assert not missing, f"instantiations never launched: {missing}"
    assert widths == {64, 128, 192, 256}, f"halo MMA widths launched: {sorted(widths)}"
