"""Tile geometry of the implicit-GEMM conv / GEMM kernel (diffusion_e2e_ft_b200/csrc/gemm_conv.cu), restated in Python,
and an fp64 reference with a per-element error bound for it.

* `conv_plan` / `linear_plan` predict, for a call of `b200_conv2d_nhwc` / `b200_linear`, the record that
  `b200_debug_last_launch` reports (include/b200_e2eft.h): which of the kernel's 28 instantiations runs and on which
  tile.  They restate `pick_halo_tile`, `pick_patch` and the cost model (`tiles_cost`, the 0.85 swap factor,
  `epi_bound`, `vec_ok`).  The GPU tests assert the prediction against the record, so a drift of the C++ picker fails
  them instead of silently moving a check onto another path.
* `tap_conv_ref` is the conv the kernel computes (any tap set, stride 1 or 2, zero padding) in fp64, together with the
  same conv on |x| and |w|, which the error bound needs.
* `conv_bound` is the per-element bound  |out - ref| <= u_out |ref| + (K + 4) u_acc (sum|x||w| + |bias| + |rowvec| +
  |residual|)  (+ the activation terms), with u_acc = 2^-22.  ASSUMPTION: the tensor cores' fp32 accumulation on
  Hopper is not IEEE round-to-nearest and how far it departs has not been measured here, so the unit is taken four
  times the fp32 unit roundoff.  fp16 x fp16 products are exact in fp32, so the accumulation is the only rounding before
  the epilogue.
"""
import math

import torch

# record fields of b200_debug_last_launch
FIELDS = ("conv", "halo", "swap", "bn", "vec", "geglu", "f32", "bw", "bh", "halo_n", "tiles_w", "tiles_h", "m_tiles",
          "n_tiles", "grid", "stats")

HALO_MAX_PATCH_PIX = 400                           # kHaloMaxPatchPix (gemm_conv.cuh)
ACT_NONE, ACT_SILU, ACT_GEGLU, ACT_GELU = 0, 1, 2, 3
U_ACC = 2.0 ** -22
U_OUT = {True: 2.0 ** -24, False: 2.0 ** -11}      # fp32 / fp16 output rounding (unit roundoff)
ACT_LIP = 1.13                                     # max |d act / dx| of SiLU (1.0998) and erf-GELU (1.1289)


# ------------------------------------------------------------------------------------------------ the picker
def kblock_cycles(n):
    return n * 4.0 if n * 4.0 > 365.0 else 365.0


def tiles_cost(tiles, n, sms):
    return ((tiles + sms - 1) // sms) * (kblock_cycles(n) + 40.0)


def pick_halo_tile(Ho, Wo):
    """(bw, bh, accepted) of the halo-resident conv's output patch."""
    best, bbw, bbh = 0.0, 0, 0
    for bw in range(8, min(254, Wo) + 1):
        for bh in range(1, min(32, Ho) + 1):
            pitch = bw + 2
            n = (pitch * bh + 63) // 64 * 64
            if n > 256:
                break
            if (bh + 2) * pitch + (n - pitch * bh) + 2 > HALO_MAX_PATCH_PIX:
                continue
            ew = Wo / (((Wo + bw - 1) // bw) * bw)
            eh = Ho / (((Ho + bh - 1) // bh) * bh)
            score = ew * eh * (bw * bh) / n
            score *= 0.9 + 0.1 * n / 256.0
            score *= 1.0 - 0.03 * ((bw + 2) * (bh + 2) / (bw * bh) - 1.0)
            if score > best + 1e-9:
                best, bbw, bbh = score, bw, bh
    return bbw, bbh, bbw != 0 and best >= 0.78


def halo_n(bw, bh):
    return ((bw + 2) * bh + 63) // 64 * 64


def patch_pix(bw, bh):
    """Patch rows the halo tile reads: (bh + 2) rows of bw + 2 pixels plus the tail the last taps read past them."""
    pitch = bw + 2
    n = halo_n(bw, bh)
    return (bh + 2) * pitch + (n - pitch * bh) + 2


def pick_patch(Ho, Wo, stride, target):
    best, bbw, bbh = -1.0, 1, 1
    for bw in range(1, min(target, Wo) + 1):
        if bw * stride > 256:
            break
        bh = target // bw
        bh = min(bh, Ho)
        if bh * stride > 256:
            bh = 256 // stride
        if bh < 1:
            continue
        tw, th = (Wo + bw - 1) // bw, (Ho + bh - 1) // bh
        eff = Ho * Wo / (tw * th * target)
        if eff > best + 1e-9 or (eff > best - 1e-9 and bw > bbw):
            best, bbw, bbh = eff, bw, bh
    return bbw, bbh


def _grid(tiles, swap, stats, n_tiles, sms):
    g = min(tiles, sms)
    if swap and stats and n_tiles > 1 and g > n_tiles:
        g -= g % n_tiles
    return g


def conv_plan(NB, H, W, Cin, Cout, taps, stride=1, out_hw=None, C2=0, out_mul=1, out_f32=False, residual=False,
              stats=False, out_nchw=False, sms=132, halo_mode=1, force_bn=0, staged=False):
    """The record b200_conv2d_nhwc reports (all pointers 16-byte aligned, as torch allocates them)."""
    Ho, Wo = out_hw or (H, W)
    can_swap = Cout >= 128 and not out_nchw
    taps_ok = stride == 1 and (Ho, Wo) == (H, W) and not (C2 and out_mul != 1) and \
        all(-1 <= dy <= 1 and -1 <= dx <= 1 for dy, dx in taps)
    epi_bound = out_f32 and residual and len(taps) * Cin <= 1152 and not C2
    halo_vec = not staged and Cout % 4 == 0
    if can_swap and halo_mode and taps_ok and not force_bn and halo_vec and (not epi_bound or halo_mode == 2):
        bw, bh, ok = pick_halo_tile(Ho, Wo)
        if ok:
            tw, th = (Wo + bw - 1) // bw, (Ho + bh - 1) // bh
            m_tiles, n_tiles = NB * tw * th, (Cout + 127) // 128
            return dict(conv=1, halo=1, swap=1, bn=256, vec=1, geglu=0, f32=int(out_f32), bw=bw, bh=bh,
                        halo_n=halo_n(bw, bh), tiles_w=tw, tiles_h=th, m_tiles=m_tiles, n_tiles=n_tiles,
                        grid=_grid(m_tiles * n_tiles, True, stats, n_tiles, sms), stats=int(stats))
    best, swap, pix, bn_norm = 1e30, False, 128, 0
    bw, bh = pick_patch(Ho, Wo, stride, 128)
    mt = NB * ((Wo + bw - 1) // bw) * ((Ho + bh - 1) // bh)
    for n in (256, 160, 128, 64, 32):
        if force_bn and n != force_bn:
            continue
        c = tiles_cost(mt * ((Cout + n - 1) // n), n, sms)
        if c < best - 1e-9:
            best, bn_norm, swap = c, n, False
    if can_swap:
        for pc in (256, 128, 64):
            if force_bn and pc != force_bn:
                continue
            bw, bh = pick_patch(Ho, Wo, stride, pc)
            tiles = NB * ((Wo + bw - 1) // bw) * ((Ho + bh - 1) // bh) * ((Cout + 127) // 128)
            c = tiles_cost(tiles, pc, sms) * 0.85
            if c < best - 1e-9:
                best, pix, swap = c, pc, True
    if not swap:
        pix = 128
    bw, bh = pick_patch(Ho, Wo, stride, pix)
    tw, th = (Wo + bw - 1) // bw, (Ho + bh - 1) // bh
    m_tiles = NB * tw * th
    bn = pix if swap else bn_norm
    n_tiles = (Cout + 127) // 128 if swap else (Cout + bn - 1) // bn
    stats = stats and not out_nchw
    return dict(conv=1, halo=0, swap=int(swap), bn=bn, vec=int(swap and halo_vec), geglu=0, f32=int(out_f32),
                bw=bw, bh=bh, halo_n=0, tiles_w=tw, tiles_h=th, m_tiles=m_tiles, n_tiles=n_tiles,
                grid=_grid(m_tiles * n_tiles, swap, stats, n_tiles, sms), stats=int(stats))


def geglu_block_n(N):
    return 160 if N % 160 == 0 else 256 if N % 256 == 0 else 128 if N % 128 == 0 else 64 if N % 64 == 0 else 0


def linear_plan(M, N, K, act=ACT_NONE, out_f32=False, stats_rows=0, sms=132, force_bn=0, vec_flag=False,
                staged=False):
    """The record b200_linear reports (batch 1, K-major operands, contiguous 16-byte aligned tensors)."""
    m_tiles = (M + 127) // 128
    swap, bn, best = False, 0, 1e30
    if act == ACT_GEGLU:
        bn = geglu_block_n(N)
    else:
        can_swap = N >= 128
        normal_ok = not stats_rows or stats_rows % 128 == 0
        if normal_ok:
            for n in (256, 160, 128, 64, 32):
                if force_bn and n != force_bn:
                    continue
                c = tiles_cost(m_tiles * ((N + n - 1) // n), n, sms)
                if c < best - 1e-9:
                    best, bn, swap = c, n, False
        if can_swap or (stats_rows and not normal_ok and N >= 128):
            for pc in (256, 128, 64):
                if force_bn and pc != force_bn:
                    continue
                if stats_rows and stats_rows % pc:
                    continue
                c = tiles_cost(((M + pc - 1) // pc) * ((N + 127) // 128), pc, sms) * 0.85
                if c < best - 1e-9:
                    best, bn, swap = c, pc, True
    if swap:
        m_tiles, n_tiles = (M + bn - 1) // bn, (N + 127) // 128
    else:
        n_tiles = (N + bn - 1) // bn
    vec = swap and (bool(stats_rows) or vec_flag) and not staged and N % 4 == 0
    return dict(conv=0, halo=0, swap=int(swap), bn=bn, vec=int(vec), geglu=int(act == ACT_GEGLU), f32=int(out_f32),
                bw=0, bh=0, halo_n=0, tiles_w=0, tiles_h=0, m_tiles=m_tiles, n_tiles=n_tiles,
                grid=_grid(m_tiles * n_tiles, swap, bool(stats_rows), n_tiles, sms), stats=int(bool(stats_rows)))


def instantiation(rec):
    """Key of the kernel template instantiation a record names."""
    if rec["halo"]:
        kind = "halo"
    elif rec["geglu"]:
        kind = "geglu"
    elif rec["swap"]:
        kind = "swap_vec" if rec["vec"] else "swap"
    else:
        kind = "normal"
    return (kind, 256 if kind == "halo" else rec["bn"], "f32" if rec["f32"] else "f16")


ALL_INSTANTIATIONS = frozenset(
    [("normal", n, o) for n in (32, 64, 128, 160, 256) for o in ("f16", "f32")]
    + [(k, n, o) for k in ("swap", "swap_vec") for n in (64, 128, 256) for o in ("f16", "f32")]
    + [("geglu", n, "f16") for n in (64, 128, 160, 256)]
    + [("halo", 256, o) for o in ("f16", "f32")])
assert len(ALL_INSTANTIATIONS) == 28


# ------------------------------------------------------------------------------------------------ reference
def tap_conv_ref(x, w_taps, taps, stride=1, out_hw=None, x2=None, w2=None):
    """fp64 sum_t x[ho*s + dy_t, wo*s + dx_t] W_t^T (zero outside the image) and the same on |x|, |W|.
    x: [NB, H, W, Cin] (any float dtype), w_taps: [Cout, T, Cin], x2: [NB, Ho, Wo, C2] with w2: [Cout, C2] (1x1).
    Returns (ref, absref), each [NB, Ho, Wo, Cout] fp64."""
    NB, H, W, Cin = x.shape
    Ho, Wo = out_hw or (H, W)
    lo = max(0, -min(min(t) for t in taps))
    xd = x.double()
    pad_hi_h = max(0, (Ho - 1) * stride + max(dy for dy, _ in taps) - (H - 1))
    pad_hi_w = max(0, (Wo - 1) * stride + max(dx for _, dx in taps) - (W - 1))
    xp = torch.nn.functional.pad(xd, (0, 0, lo, pad_hi_w, lo, pad_hi_h))
    wd = w_taps.double()
    ref = torch.zeros(NB, Ho, Wo, wd.shape[0], dtype=torch.float64, device=x.device)
    absref = torch.zeros_like(ref)
    for t, (dy, dx) in enumerate(taps):
        xs = xp[:, lo + dy: lo + dy + (Ho - 1) * stride + 1: stride, lo + dx: lo + dx + (Wo - 1) * stride + 1: stride]
        wt = wd[:, t]
        ref += xs @ wt.t()
        absref += xs.abs() @ wt.abs().t()
    if x2 is not None:
        ref += x2.double() @ w2.double().t()
        absref += x2.double().abs() @ w2.double().abs().t()
    return ref, absref


def conv_bound(pre, absacc, K, out_f32, act=ACT_NONE, extra_abs=None):
    """Per-element bound of |out - ref| where ref = act(pre) and pre = acc + bias + rowvec + residual in fp64.
    absacc: sum|x||w| of the accumulation; extra_abs: |bias| + |rowvec| + |residual| (broadcast)."""
    a = absacc if extra_abs is None else absacc + extra_abs
    e_pre = (K + 4) * U_ACC * a
    if act in (ACT_SILU, ACT_GELU):
        ref = torch.nn.functional.silu(pre) if act == ACT_SILU else torch.nn.functional.gelu(pre)
        # __expf / __fdividef (SiLU) and the Abramowitz-Stegun erf (|err| <= 1.5e-7, GELU): 2^-18 (1 + |x|)^2 covers both
        e_act = ACT_LIP * e_pre + 2.0 ** -18 * (1.0 + pre.abs()) ** 2
    else:
        ref, e_act = pre, e_pre
    return ref, U_OUT[out_f32] * ref.abs() + e_act * (1.0 + U_OUT[out_f32]) + 2.0 ** -25


def check_bound(out, ref, bound, what):
    """Element-wise |out - ref| <= bound.  Returns (worst error / bound ratio, rel-L2) for the report."""
    err = (out.double() - ref).abs()
    ratio = err / bound
    worst = ratio.max().item()
    rl2 = ((out.double() - ref).norm() / (ref.norm() + 1e-30)).item()
    if not worst <= 1.0:
        idx = [int(i) for i in torch.nonzero(ratio == ratio.max())[0]]
        bad = int((ratio > 1.0).sum().item())
        raise AssertionError(f"{what}: {bad} elements exceed the bound; worst at {idx}: out {out[tuple(idx)].item():.7g} "
                             f"ref {ref[tuple(idx)].item():.7g} bound {bound[tuple(idx)].item():.3g} "
                             f"(ratio {worst:.3g}, rel-L2 {rl2:.3g})")
    return worst, rl2


def check_stats(cs, stored, what, per_img_rows=None):
    """Fused per-(image, channel) [sum, sum of squares] against an fp64 reduction of the stored values.
    stored: [NB, pixels..., C] (or [M, C] with per_img_rows)."""
    o = stored.double()
    if per_img_rows:
        o = o.reshape(-1, per_img_rows, o.shape[-1])
    else:
        o = o.reshape(o.shape[0], -1, o.shape[-1])
    s1, s2 = o.sum(1), (o * o).sum(1)
    n = o.shape[1]
    # fp32 shifted partial sums: n u (sum|v| + n |shift|) bounds the sum; the squares are non-negative
    tol1 = 1e-5 * (o.abs().sum(1) + n * o.abs().amax(1)) + 1e-30
    tol2 = 1e-5 * s2 + 1e-30
    r1 = ((cs[..., 0] - s1).abs() / tol1).max().item()
    r2 = ((cs[..., 1] - s2).abs() / tol2).max().item()
    assert r1 <= 1.0 and r2 <= 1.0, f"{what}: fused statistics off (sum ratio {r1:.3g}, sum-of-squares ratio {r2:.3g})"
    return max(r1, r2)
