"""The footprint case table (tests/footprint_cases.py) covers the whole C ABI, and its masks count what the header
documents.  CPU only: the masks are index arithmetic."""
import os
import re

import torch

import footprint_cases as FC

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200_e2eft.h")
CASES = FC.all_cases()


def _header_entry_points():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    return set(re.findall(r"\b(b200_\w+)\s*\(", src))


def test_every_entry_point_is_covered_or_exempt():
    entries = _header_entry_points()
    assert len(entries) > 70
    covered = {c.entry for c in CASES}
    assert not covered - entries, f"cases name unknown entry points: {sorted(covered - entries)}"
    assert not set(FC.EXEMPT) - entries, sorted(set(FC.EXEMPT) - entries)
    assert not covered & set(FC.EXEMPT), sorted(covered & set(FC.EXEMPT))
    missing = entries - covered - set(FC.EXEMPT)
    assert not missing, f"entry points with neither a footprint case nor an exemption: {sorted(missing)}"
    assert all(r.strip() for r in FC.EXEMPT.values())


def test_case_names_are_unique_and_operands_well_formed():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))
    for c in CASES:
        for n, o in c.ops.items():
            assert (o.start * o.dtype.itemsize) % 8 == 0, (c.name, n)
            assert not o.mask[:FC.GUARD].any() and not o.mask[-FC.GUARD:].any(), (c.name, n)
            assert not (o.check & ~o.mask).any(), (c.name, n)
            if o.zero is not None:
                assert not (o.zero & ~o.mask).any(), (c.name, n)
            if o.role in ("in", "inout"):
                assert o.values is not None, (c.name, n)
                # every element a kernel may read holds a defined value: the footprint lies inside the view
                in_view = torch.zeros_like(o.mask)
                in_view[o.index.reshape(-1)] = True
                assert not (o.mask & ~in_view).any(), (c.name, n)


def _case(name):
    return next(c for c in CASES if c.name == name)


def test_conv_out_mul2_phases_partition_the_output():
    for prefix in ("conv_dgrad_s2", "conv_upsample"):
        phases = [_case(f"{prefix}_phase{oy}{ox}") for oy in (0, 1) for ox in (0, 1)]
        masks = [c.ops["out"].mask for c in phases]
        total = torch.stack(masks).sum(0)
        view = torch.zeros_like(total, dtype=torch.bool)
        view[phases[0].ops["out"].index.reshape(-1)] = True
        assert bool((total[view] == 1).all()) and not total[~view].any()
        NB, OH, OW, C = phases[0].ops["out"].shape
        assert all(int(m.sum()) == NB * (OH // 2) * (OW // 2) * C for m in masks)


def test_gather_planar_zero_tail_is_ldo_minus_pixels():
    c = _case("gather_planar_slice")
    o = c.ops["out"]
    C, ldo = o.shape
    P = 2 * 5 * 7
    assert ldo == FC.ru8(P) + 64
    assert int(o.zero.sum()) == C * (ldo - P)
    assert int(o.mask.sum()) == C * ldo
    s2 = _case("gather_planar_s2").ops["out"]
    assert int(s2.zero.sum()) == s2.shape[0] * (FC.ru8(2 * 5 * 5) - 2 * 5 * 5)


def test_linear_pitch_gaps_sit_outside_the_read_footprint():
    c = _case("linear_pitched")
    a = c.ops["A"]
    M, K, lda = 200, 72, 88
    assert a.shape == (1, M, K) and a.strides[1] == lda
    assert int(a.mask.sum()) == M * K
    row0 = a.mask[a.start:a.start + lda]
    assert bool(row0[:K].all()) and not row0[K:].any()
    out = c.ops["out"]
    assert int(out.mask.sum()) == M * 136 and out.strides[1] == 144


def test_self_test_cases_declare_smaller_footprints():
    short = FC.linear_case("x", 200, 136, 72, lda=88, ldw=96, ldo=144, short_out=True)
    full = FC.linear_case("x", 200, 136, 72, lda=88, ldw=96, ldo=144)
    assert int(full.ops["out"].mask.sum()) - int(short.ops["out"].mask.sum()) == 136
    short = FC.linear_case("x", 200, 136, 72, lda=88, ldw=96, ldo=144, short_a=True)
    assert int(full.ops["A"].mask.sum()) - int(short.ops["A"].mask.sum()) == 200


def test_group_norm_bwd_footprint_is_the_channel_slice():
    S = _case("group_norm_bwd_0_sums").ops["S"]
    NB, Ctot, _ = S.shape
    assert int(S.mask.sum()) == NB * 32 * 2
    assert bool(S.mask[S.index[:, 64:96].reshape(-1)].all()) and not S.mask[S.index[:, :64].reshape(-1)].any()


def test_eval_normal_error_short_buffer_footprint():
    c = _case("eval_normal_error_short")
    buf, mask = c.ops["buf"], c.ops["mask"].values
    assert buf.shape[0] < int(mask.sum())
    assert int(buf.mask.sum()) == buf.shape[0] and int(buf.check.sum()) == 0


def test_compact_twins_hold_the_same_values_contiguously():
    twins = [c for c in CASES if c.compact is not None]
    assert len(twins) > 50
    for c in twins:
        t = c.compact
        assert t.name == c.name and t.entry == c.entry and t.ops.keys() == c.ops.keys(), c.name
        for n, o in c.ops.items():
            ot = t.ops[n]
            if o.role in ("in", "inout"):
                assert torch.equal(o.values, ot.values), (c.name, n)
                if n != "S":
                    # a compact input is one dense block (MN-major pitches are rounded up to 16 bytes)
                    assert int(ot.mask.sum()) == ot.index.numel(), (c.name, n)
    layouts = {c.name: (c.ops["A"].strides, c.compact.ops["A"].strides) for c in twins if c.entry == "b200_linear"}
    assert layouts["linear_pitched"] == ((200 * 88, 88, 1), (200 * 72, 72, 1))
