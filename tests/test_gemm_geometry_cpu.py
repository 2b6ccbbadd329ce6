"""CPU: the case list of tests/test_gemm_conv_geometry_gpu.py covers every geometry class of the conv / GEMM dispatcher,
as predicted by its Python restatement (tests/gemm_geometry.py) on a 132-SM H100.  The GPU tests then assert each
prediction against the kernel's own launch record."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_geometry as G  # noqa: E402
import test_gemm_conv_geometry_gpu as T  # noqa: E402

SMS = 132


def _conv_records():
    out = []
    for name in T.CONV_CASES:
        for f32 in (False, True):
            out.append((name, f32, False, T.conv_case_plan(name, f32, False, SMS)[0]))
            if name.startswith("swap"):
                out.append((name, f32, True, T.conv_case_plan(name, f32, True, SMS)[0]))
    return out


def _linear_records():
    recs = []
    for M, N, K, act, res, bn, staged in T.LINEAR_CASES.values():
        recs += [G.linear_plan(M, N, K, act, f32, sms=SMS, force_bn=bn, staged=staged) for f32 in (False, True)]
    recs += [G.linear_plan(300, N, 320, G.ACT_GEGLU, False, sms=SMS) for N in (192, 384, 320, 512)]
    recs += [G.linear_plan(2 * L, N, 320, out_f32=True, stats_rows=L, sms=SMS) for L in (576, 448, 9216)
             for N in (320, 640, 1280)]
    return recs


def test_picker_restatement_matches_documented_geometries():
    # feature maps the halo picker sends to each MMA width (native-resolution inputs reach all of them)
    assert G.pick_halo_tile(10, 28) == (28, 2, True) and G.halo_n(28, 2) == 64
    assert G.pick_halo_tile(13, 60) == (60, 1, True) and G.halo_n(60, 1) == 64
    assert G.pick_halo_tile(9, 40) == (40, 3, True) and G.halo_n(40, 3) == 128
    assert G.pick_halo_tile(10, 56) == (56, 2, True) and G.halo_n(56, 2) == 128
    for Ho, Wo in ((24, 24), (48, 48), (96, 96), (20, 44)):
        bw, bh, ok = G.pick_halo_tile(Ho, Wo)
        if ok:
            assert G.patch_pix(bw, bh) <= G.HALO_MAX_PATCH_PIX and G.halo_n(bw, bh) <= 256


def test_case_list_covers_every_halo_geometry_class():
    halo = [(n, f32, r) for n, f32, _, r in _conv_records() if r["halo"]]
    for f32 in (False, True):
        assert {r["halo_n"] for _, o, r in halo if o == f32} == {64, 128, 192, 256}
    recs = [r for _, _, r in halo]
    wo = [(T.CONV_CASES[name][2], r) for name, _, r in halo]
    assert any(r["bh"] == 1 for _, r in wo)
    assert any(W == r["bw"] for W, r in wo)
    assert any(W > r["bw"] and W % r["bw"] == 1 for W, r in wo)
    tight = {(r["bw"], r["bh"]) for r in recs if G.HALO_MAX_PATCH_PIX - G.patch_pix(r["bw"], r["bh"]) <= 20}
    assert len(tight) >= 3, tight
    # 23 rows is the tallest patch the picker accepts over Ho <= 129, Wo <= 40
    assert max(r["bh"] for r in recs) == 23
    assert any(r["stats"] and r["m_tiles"] * r["n_tiles"] > SMS for r in recs), "no multi-wave statistics case"
    assert any(r["n_tiles"] > 1 and r["stats"] for r in recs)


def test_case_list_covers_per_tap_and_normal_tiles():
    seen = set()
    for name, f32, staged, r in _conv_records():
        if r["halo"]:
            continue
        stride, pad = T.CONV_CASES[name][5], T.CONV_CASES[name][6]
        seen.add(("swap" if r["swap"] else "normal", r["bn"], stride, pad, bool(r["vec"])))
    for bn in (64, 128, 256):
        for stride, pad in ((1, "same"), (2, "same"), (2, "pad0")):
            for vec in (True, False):
                assert ("swap", bn, stride, pad, vec) in seen, (bn, stride, pad, vec)
    assert {k[1] for k in seen if k[0] == "normal"} == {32, 64, 128, 160, 256}


def test_case_list_launches_all_28_instantiations():
    recs = [r for *_, r in _conv_records()] + _linear_records()
    seen = {G.instantiation(r) for r in recs}
    assert seen == G.ALL_INSTANTIATIONS, sorted(G.ALL_INSTANTIATIONS ^ seen)
    assert {r["bn"] for r in recs if r["geglu"]} == {64, 128, 160, 256}


@pytest.mark.parametrize("L", [576, 448])
def test_proj_out_statistics_force_the_64_pixel_swapped_tile(L):
    for N in (320, 640, 1280):
        r = G.linear_plan(2 * L, N, N, out_f32=True, stats_rows=L, sms=SMS)
        assert r["swap"] == 1 and r["bn"] == 64 and r["vec"] == 1


def test_tap_conv_reference_matches_torch_conv():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 9, 11, 8, generator=g).half()
    w = torch.randn(5, 8, 3, 3, generator=g).half()
    wt = w.permute(0, 2, 3, 1).reshape(5, 9, 8)
    for stride, taps, pad in ((1, T.TAPS["same"], (1, 1, 1, 1)), (2, T.TAPS["same"], (1, 1, 1, 1)),
                              (2, T.TAPS["pad0"], (0, 1, 0, 1))):
        want = torch.nn.functional.conv2d(torch.nn.functional.pad(x.double().permute(0, 3, 1, 2), pad), w.double(),
                                          stride=stride).permute(0, 2, 3, 1)
        got, absref = G.tap_conv_ref(x, wt, taps, stride, tuple(want.shape[1:3]))
        assert torch.allclose(got, want, rtol=0, atol=1e-12)
        assert (absref >= got.abs() - 1e-12).all()
