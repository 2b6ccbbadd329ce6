"""Every C-ABI entry point reads and writes only its documented footprint (tests/footprint_cases.py).

Each case runs three times on the same strided layout, with every output / workspace backing buffer filled with a
byte pattern and every input's out-of-footprint elements (pitch gaps, rows past M / Lk, batch gaps, guard bands)
set to zero or poisoned (NaN, 0xFF, integer max):
  1. pattern 0xA5, clean inputs;   2. pattern 0x5A, clean inputs;   3. pattern 0xA5, poisoned inputs.
Outside the footprint every output byte must keep its pattern and every input byte its value; inside it runs 1
and 2 must agree (an element left unwritten would differ), documented zero fills must be zero, and run 3 must
equal run 1 (a read of poisoned memory would differ).  A case with strides or pitches also runs its compact twin
(the same values in contiguous buffers), whose outputs run 1 must equal: byte for byte when both launches leave the
same b200_debug_last_launch record (and for kernels without one), within LAYOUT_TOL when the layout changed the
tile choice.  Operands accumulated with floating-point atomics use their declared tolerance throughout.  Finally
the outputs of the compact call are held to an fp64 reference of the operation (REFERENCES) for the GEMM, conv,
attention, softmax, row-dot, gather and column-sum entry points, with the tolerances of tests/kernel_checks.py.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import footprint_cases as FC

pytestmark = pytest.mark.gpu

PATTERNS = (0xA5, 0x5A)
LAYOUT_TOL = {torch.float16: (2e-3, 2e-3), torch.float32: (1e-4, 1e-4)}    # other tile geometry: other fp32 sum order


def _poison(dtype):
    if dtype.is_floating_point:
        return float("nan")
    if dtype == torch.uint8:
        return 255
    if dtype == torch.int16:
        return -1                     # 0xFFFF: the largest uint16
    return torch.iinfo(dtype).max


def _lib():
    from diffusion_e2e_ft_b200 import lib
    return lib.load()


def _reset(L):
    L.b200_debug_set_swap(1)
    L.b200_debug_set_halo(1)
    L.b200_debug_set_flags(0)
    L.b200_debug_force_block_n(0)


def _launch(case, pattern, poison):
    L = _lib()
    dev = torch.device("cuda")
    bufs, ptrs = {}, {}
    for name, o in case.ops.items():
        b = torch.empty(o.size, dtype=o.dtype, device=dev)
        if o.role == "in":
            b.fill_(_poison(o.dtype) if poison else 0)
        else:
            b.view(torch.uint8).fill_(pattern)
        if o.role in ("in", "inout"):
            idx = o.index.reshape(-1)
            sel = o.mask[idx]                                # view elements inside the footprint
            b[idx[sel].to(dev)] = o.values.reshape(-1)[sel].to(dev)
        bufs[name] = b
        ptrs[name] = b.data_ptr() + o.start * b.element_size()
    before = {n: b.clone() for n, b in bufs.items() if case.ops[n].role == "in"}
    if case.setup is not None:
        case.setup(L)
    try:
        rc = case.call(L, ptrs, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        rec = None
        if case.record:
            arr = (ctypes.c_int * 16)()
            L.b200_debug_last_launch(arr, 16)
            rec = list(arr)
    finally:
        _reset(L)
    if rc != 0:
        msg = L.b200_last_error_string()
        raise RuntimeError(f"{case.entry} ({case.name}) failed rc={rc}: {msg.decode() if msg else '?'}")
    torch.cuda.synchronize()
    return {n: b.cpu() for n, b in bufs.items()}, {n: b.cpu() for n, b in before.items()}, rec


def _same_values(o, x, y, tol=None):
    tol = o.tol or tol
    if o.sort:
        x, y = torch.sort(x.double())[0], torch.sort(y.double())[0]
    if tol is not None:
        return torch.allclose(x.double(), y.double(), rtol=tol[0], atol=tol[1], equal_nan=True)
    return torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8))


def _same(o, a, b, where):
    """a, b: backing buffers; compare them on the bool mask `where`."""
    return _same_values(o, a[where], b[where])


def _common(o, oc):
    """Backing indices of the checked elements of the leading block two layouts of one operand share."""
    sl = tuple(slice(0, min(x, y)) for x, y in zip(o.shape, oc.shape))
    ia, ib = o.index[sl].reshape(-1), oc.index[sl].reshape(-1)
    sel = o.check[ia] & oc.check[ib]
    return ia[sel], ib[sel]


def _views(case, run):
    return {n: run[n][o.index] for n, o in case.ops.items() if o.role != "scratch"}


def footprint_violations(case, reference=True):
    """Runs the case and returns the list of violations (empty when the kernel keeps its footprint and computes the
    reference's values).  `reference=False`: footprint checks only (the self-tests declare shortened views)."""
    r1, in1, rec1 = _launch(case, PATTERNS[0], poison=False)
    r2, _, _ = _launch(case, PATTERNS[1], poison=False)
    r3, in3, rec3 = _launch(case, PATTERNS[0], poison=True)
    bad = []
    for name, o in case.ops.items():
        if o.role == "in":
            for tag, run, ref in (("clean", r1, in1), ("poisoned", r3, in3)):
                if not torch.equal(run[name].view(torch.uint8), ref[name].view(torch.uint8)):
                    bad.append(f"{name}: input modified ({tag} run)")
            continue
        outside = ~o.mask
        for run, pat in ((r1, PATTERNS[0]), (r2, PATTERNS[1]), (r3, PATTERNS[0])):
            bytes_out = run[name].view(torch.uint8).reshape(o.size, -1)[outside]
            if not bool((bytes_out == pat).all()):
                n = int(((bytes_out != pat).any(1)).sum())
                first = int(torch.nonzero(outside)[(bytes_out != pat).any(1)][0])
                bad.append(f"{name}: {n} element(s) written outside the footprint (pattern {pat:#x}; first at backing "
                           f"index {first}, view starts at {o.start})")
                break
        if o.role == "scratch":
            continue
        if not _same(o, r1[name], r2[name], o.check):
            bad.append(f"{name}: footprint differs between fill patterns (an element left unwritten, or a read of "
                       "the output buffer)")
        if o.zero is not None:
            for run in (r1, r2):
                if not bool((run[name].view(torch.uint8).reshape(o.size, -1)[o.zero] == 0).all()):
                    bad.append(f"{name}: documented zero fill not zero")
                    break
        if not _same(o, r1[name], r3[name], o.check):
            bad.append(f"{name}: result depends on poisoned memory outside the input footprints")
    ref_case, ref_run = case, r1
    if case.compact is not None:
        rc, _, recc = _launch(case.compact, PATTERNS[0], poison=False)
        same_launch = not case.record or rec1 == recc
        for name, o in case.ops.items():
            if o.role in ("in", "scratch"):
                continue
            ia, ib = _common(o, case.compact.ops[name])
            if not _same_values(o, r1[name][ia], rc[name][ib], None if same_launch else LAYOUT_TOL[o.dtype]):
                bad.append(f"{name}: strided result differs from the compact call "
                           f"({'same launch' if same_launch else f'launch records {rec1} / {recc}'})")
        ref_case, ref_run = case.compact, rc
    ref = REFERENCES.get(case.entry) if reference else None
    if ref is not None:
        bad += ref(ref_case, _views(ref_case, ref_run))
    return bad


# ---------------------------------------------------------------------------------------------- fp64 references
def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _within(name, got, want, tol):
    err = rel_l2(got, want)
    return [] if err <= tol else [f"{name}: rel-L2 {err:.3g} from the fp64 reference > {tol:g}"]


def _val(case, name):
    return case.ops[name].values.double()


def _act(y, act):
    return {0: y, 1: F.silu(y), 3: F.gelu(y), 4: torch.exp2(y)}[act]


def _stats_and_twin(case, out, rows_of_img):
    """chan_stats = per-(image, channel) sum / sum of squares of the stored output; out2 = the stored output in fp16."""
    bad = []
    if "stats" in out:
        y = out["out"].double().reshape(-1, rows_of_img, out["out"].shape[-1])
        want = torch.stack([y.sum(1), (y * y).sum(1)], -1)
        bad += _within("stats", out["stats"], want, 1e-6)
    if "out2" in out and not torch.equal(out["out2"], out["out"].half()):
        bad.append("out2: not the fp16 rounding of out")
    return bad


def ref_linear(case, out):
    m = case.meta
    A, W = _val(case, "A"), _val(case, "W")
    A = A.transpose(-1, -2) if m["a_mn"] else A                    # [b, M, K]
    W = W.transpose(-1, -2) if m["w_mn"] else W                    # [b, N, K]
    y = m["alpha"] * (A @ W.transpose(-1, -2))
    if "bias" in case.ops:
        b = _val(case, "bias")
        y = y + (b[:, :, None] if m["bias_row"] else b)
    if m["act"] == 2:                                               # GEGLU: [value | gate] rows interleaved per tile
        from diffusion_e2e_ft_b200 import lib
        bn = lib.load().b200_geglu_block_n(m["N"])
        t = y.reshape(*y.shape[:-1], m["N"] // bn, bn)
        y = (t[..., :bn // 2] * F.gelu(t[..., bn // 2:])).reshape(*y.shape[:-1], m["N"] // 2)
    elif m["res_mul"]:
        y = _act(y, m["act"]) * _val(case, "res")
    else:
        y = _act(y + (_val(case, "res") if "res" in case.ops else 0), m["act"])
    tol = 3e-5 if out["out"].dtype == torch.float32 else 1e-3
    return _within("out", out["out"], y, tol) + _stats_and_twin(case, out, m["stats_rows"] or 1)


def ref_conv(case, out):
    m = case.meta
    NB, Cin, Cout, Ho, Wo, s = m["NB"], m["Cin"], m["Cout"], m["Ho"], m["Wo"], m["stride"]
    X = F.pad(_val(case, "X"), (0, 0, 2, 2, 2, 2))                  # every tap offset lies in [-2, 2]
    Wp = _val(case, "Wp")
    oy_, ox_ = torch.arange(Ho) * s + 2, torch.arange(Wo) * s + 2
    y = torch.zeros(NB, Ho, Wo, Cout, dtype=torch.float64)
    for t, (dy, dx) in enumerate(m["taps"]):
        xs = X[:, oy_ + dy][:, :, ox_ + dx]
        y += xs @ Wp[:, t * Cin:(t + 1) * Cin].T
    if m["C2"]:
        y += _val(case, "X2") @ Wp[:, len(m["taps"]) * Cin:].T
    if "bias" in case.ops:
        y += _val(case, "bias")
    if "rowvec" in case.ops:
        y += _val(case, "rowvec")[:, None, None, :]
    mul, (py, px) = m["out_mul"], m["phase"]
    got = out["out"]
    if m["out_nchw"]:
        got = got.permute(0, 2, 3, 1)
    got = got[:, py::mul, px::mul]
    if "res" in case.ops:
        y += _val(case, "res")[:, py::mul, px::mul]
    y = _act(y, m["act"])
    tol = 3e-5 if got.dtype == torch.float32 else 1e-3
    bad = _within("out", got, y, tol)
    if mul == 1 and not m["out_nchw"]:
        bad += _stats_and_twin(case, out, Ho * Wo)
    return bad


def ref_attention(case, out):
    m = case.meta
    h, D = m["heads"], m["D"]
    q, k, v = (_val(case, n) for n in "qkv")
    B, Lq, Lk = q.shape[0], q.shape[1], k.shape[1]
    qf = q.reshape(B, Lq, h, D).transpose(1, 2)
    kf, vf = (t.reshape(B, Lk, h, D).transpose(1, 2) for t in (k, v))
    if m["kv_segments"] == 2:                                       # b attends to b % (B/2) and b % (B/2) + B/2
        k0, k1 = kf.chunk(2, 0)
        v0, v1 = vf.chunk(2, 0)
        kf, vf = torch.cat([torch.cat([k0, k1], 2)] * 2, 0), torch.cat([torch.cat([v0, v1], 2)] * 2, 0)
    s = qf @ kf.transpose(-1, -2) * m["scale"]
    want = (torch.softmax(s, -1) @ vf).transpose(1, 2).reshape(B, Lq, h * D)
    bad = _within("o", out["o"], want, 2e-3)
    if "lse" in out:
        lse = torch.logsumexp(s, -1) / math.log(2.0)
        err = (out["lse"].double() - lse).abs().max().item()
        if err > 1e-3:
            bad.append(f"lse: max error {err:.3g} from the fp64 log2-sum-exp > 1e-3")
    return bad


def ref_rowdot(case, out):
    m = case.meta
    a, c = _val(case, "a"), _val(case, "c")
    B, L_ = a.shape[:2]
    want = (a * c).reshape(B, L_, m["heads"], m["D"]).sum(-1).transpose(1, 2)
    return _within("out", out["out"], want, 1e-5)


def ref_softmax_rows(case, out):
    return _within("P", out["P"], torch.softmax(case.meta["scale"] * _val(case, "S"), -1), 6e-4)


def ref_softmax_groups(case, out):
    m = case.meta
    x = _val(case, "logits")
    want = torch.softmax(x.reshape(x.shape[0], m["heads"], m["S"]), -1).reshape(x.shape)
    return _within("P", out["P"][:, :x.shape[1]], want, 6e-4)


def ref_softmax_bwd(case, out):
    P, dP = _val(case, "P"), _val(case, "dP")
    want = case.meta["scale"] * P * (dP - (dP * P).sum(-1, keepdim=True))
    return _within("dS", out["dS"], want, 1e-3)


def ref_gather_planar(case, out):
    m = case.meta
    x = case.ops["x"].values
    NB, H, W, C = x.shape
    Ho, Wo, st, up = m["Ho"], m["Wo"], m["stride"], m["up"]
    ys, xs = torch.arange(Ho) * st + m["oy"], torch.arange(Wo) * st + m["ox"]
    vy, vx = (ys >= 0) & (ys < H * up), (xs >= 0) & (xs < W * up)
    g = x.half()[:, (ys.clamp(0, H * up - 1) // up)][:, :, (xs.clamp(0, W * up - 1) // up)]
    g = g * (vy[None, :, None, None] & vx[None, None, :, None])
    want = g.permute(3, 0, 1, 2).reshape(C, NB * Ho * Wo)
    got = out["out"][:, :want.shape[1]]
    return [] if torch.equal(got, want) else ["out: not the exact gather of x"]


def ref_col_sum(case, out):
    want = _val(case, "out") + _val(case, "x").sum(0)
    return _within("out", out["out"], want, 1e-5)


def ref_normal_error(case, out):
    n = case.meta["count"]
    bad = []
    if int(out["buf_len"][0]) != n:
        bad.append(f"buf_len: {int(out['buf_len'][0])}, not the {n} masked angles")
    if int(out["counts"][0]) != n:                                  # counts start at (0, 1, ..., 5)
        bad.append(f"counts[0]: {int(out['counts'][0])}, not {n}")
    return bad


REFERENCES = {
    "b200_linear": ref_linear, "b200_conv2d_nhwc": ref_conv, "b200_attention": ref_attention,
    "b200_attention_d64": ref_attention, "b200_attention_d512": ref_attention, "b200_rowdot_heads_d": ref_rowdot,
    "b200_rowdot_heads": ref_rowdot, "b200_softmax_rows": ref_softmax_rows, "b200_softmax_groups": ref_softmax_groups,
    "b200_softmax_bwd_rows": ref_softmax_bwd, "b200_gather_planar": ref_gather_planar, "b200_col_sum": ref_col_sum,
    "b200_eval_normal_error": ref_normal_error,
}


CASES = FC.all_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_kernel_footprint(case):
    bad = footprint_violations(case)
    assert not bad, f"{case.name} ({case.entry}): " + "; ".join(bad)


# ---------------------------------------------------------------------------------------------- harness self-tests
def test_harness_reports_a_write_outside_the_declared_footprint():
    """The output is declared one row short of what the kernel writes: the last row is a footprint violation."""
    case = FC.linear_case("linear_pitched", 200, 136, 72, lda=88, ldw=96, ldo=144, residual=True, ld_res=152,
                          short_out=True)
    bad = footprint_violations(case, reference=False)
    assert any(b.startswith("out:") and "outside the footprint" in b for b in bad), bad


def test_harness_reports_a_read_outside_the_declared_footprint():
    """A's read footprint leaves out the last K column: poisoning it must change the result."""
    case = FC.linear_case("linear_pitched", 200, 136, 72, lda=88, ldw=96, ldo=144, residual=True, ld_res=152,
                          short_a=True)
    bad = footprint_violations(case, reference=False)
    assert any("poisoned memory" in b for b in bad), bad


def test_harness_reports_a_wrong_value():
    """A reference that disagrees with the kernel is reported: the pitched linear case with its bias dropped from the
    reference (the kernel still adds it)."""
    case = FC.linear_cases()[0]
    r1, _, _ = _launch(case, PATTERNS[0], poison=False)
    view = _views(case, r1)
    assert not ref_linear(case, view)
    del case.ops["bias"]
    assert ref_linear(case, view)


def test_geglu_rejects_an_alpha_it_cannot_apply():
    """The GEGLU epilogue adds the bias to the raw accumulators; any alpha but 1 is refused before launch."""
    L = _lib()
    dummy = ctypes.c_void_p(1 << 20)           # 16-byte aligned; never dereferenced, the call fails its argument check
    # act 2 = B200_ACT_GEGLU
    rc = L.b200_linear(dummy, 72, 0, dummy, 64, 0, 150, 320, 64, 1, dummy, 0, None, 0, 0, dummy, 168, 0, 0,
                       2, 0.75, None, 0, None, 0, 0, 0, 0, None)
    assert rc < 0 and b"alpha" in L.b200_last_error_string(), rc

