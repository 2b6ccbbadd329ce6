"""Memory footprints of the C-ABI entry points (include/b200_e2eft.h): which elements of each operand a kernel may
read (inputs) or write (outputs), as the header documents them.  Pure index arithmetic on CPU tensors, so the
table imports and its masks can be checked without a GPU; tests/test_kernel_footprint_gpu.py runs the cases.

Every operand lives in a flat backing buffer: GUARD elements before the view, the view itself (row pitches wider
than the row, gaps between batch strides, rows past M / Lk), then `pad` + GUARD elements after it.  `mask` marks
the footprint in the backing buffer; everything else is poisoned (inputs) or must keep its fill pattern (outputs).
"""
import ctypes
import zlib

import numpy as np
import torch

GUARD = 64                      # elements; a multiple of 16 bytes for every dtype, so views stay 16-byte aligned
F16, F32, F64 = torch.float16, torch.float32, torch.float64
U8, I16, I32, I64 = torch.uint8, torch.int16, torch.int32, torch.int64     # I16 holds uint16, I32 / I64 uint32 / uint64
ROLES = ("in", "out", "inout", "scratch")
TAPS3 = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]
TAPS3_PAD0 = [(ky, kx) for ky in range(3) for kx in range(3)]
TAPS2 = [(dy, dx) for dy in (-1, 0) for dx in (-1, 0)]


def ru8(n):
    return (n + 7) // 8 * 8


def contiguous_strides(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return tuple(reversed(st))


class Op:
    """One operand.  role: in (read only), out (written), inout (initialised, then accumulated into / updated),
    scratch (written and read back by the kernel; only its footprint is checked).
    `index`: flat backing index of every view element.  `mask`: the footprint (bool over the backing buffer),
    by default the view.  `check`: the part of an output compared between runs (default: the mask).  `zero`: the
    documented zero-filled part of an output.  `tol`: (rtol, atol) for outputs accumulated with floating-point
    atomics, else outputs compare byte for byte.  `sort`: compare the sorted values (outputs appended in no
    particular order)."""

    def __init__(self, role, dtype, shape, strides=None, *, offset=0, pad=0, values=None, mask=None, check=None,
                 zero=None, tol=None, sort=False):
        assert role in ROLES
        self.role, self.dtype, self.shape = role, dtype, tuple(shape)
        self.strides = tuple(strides) if strides is not None else contiguous_strides(self.shape)
        start = GUARD + offset
        span = 1 + sum((s - 1) * st for s, st in zip(self.shape, self.strides))
        self.start = start
        self.size = start + span + pad + GUARD
        self.index = torch.arange(self.size).as_strided(self.shape, self.strides, start)
        self.mask = self._flat(self.index if mask is None else mask(self.index))
        self.check = self.mask.clone() if check is None else self._flat(check(self.index))
        self.zero = None if zero is None else self._flat(zero(self.index))
        self.tol, self.sort = tol, sort
        self.values = values
        if role in ("in", "inout") and values is not None:
            assert tuple(values.shape) == self.shape and values.dtype == dtype, (values.shape, self.shape, values.dtype)

    def _flat(self, idx):
        m = torch.zeros(self.size, dtype=torch.bool)
        m[idx.reshape(-1)] = True
        return m


class Case:
    """`call(L, p, s)` launches the entry point: p[name] is the device address of operand `name`'s view (None for
    absent operands), s the stream.  `setup(L)` sets the debug switches of the launch; `record`: the entry point
    leaves a b200_debug_last_launch record.  `compact`: the same call on contiguous copies of the inputs (None when
    the layout already is compact apart from the guard bands); `meta`: the arguments a reference needs."""

    def __init__(self, name, entry, ops, call, setup=None, record=False, meta=None):
        self.name, self.entry, self.ops, self.call, self.setup, self.record = name, entry, ops, call, setup, record
        self.compact, self.meta = None, meta or {}


def paired(builder, *args, **kw):
    """The strided case with its compact twin: the same builder with `compact=True` (same values, same name)."""
    case = builder(*args, **kw)
    case.compact = builder(*args, compact=True, **kw)
    return case


def _gen(name):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(name.encode()))
    return g


class _Vals:
    def __init__(self, name):
        self.g = _gen(name)

    def randn(self, shape, dtype=F32, scale=1.0, shift=0.0):
        return (torch.randn(shape, generator=self.g, dtype=F64) * scale + shift).to(dtype)

    def uniform(self, shape, lo, hi, dtype=F32):
        return (torch.rand(shape, generator=self.g, dtype=F64) * (hi - lo) + lo).to(dtype)

    def ints(self, shape, lo, hi, dtype=I32):
        return torch.randint(lo, hi, shape, generator=self.g, dtype=I64).to(dtype)

    def mask(self, shape, p=0.7):
        return (torch.rand(shape, generator=self.g) < p).to(U8)


def _v(x):
    return ctypes.c_void_p(x)


# ------------------------------------------------------------------------------------------------ b200_linear
def linear_case(name, M, N, K, *, batch=1, lda=None, ldw=None, ldo=None, a_bs=None, w_bs=None, o_bs=None,
                shared_w=False, out_f32=False, bias=True, bias_row=False, bias_bs=0, residual=False, ld_res=None,
                res_bs=None, res_mul=False, act=0, geglu=False, a_mn=False, w_mn=False, stats_rows=0, out2=False,
                swap=1, flags=0, short_out=False, short_a=False, compact=False):
    """`short_out` / `short_a`: declare a footprint one output row short / without A's last K column (harness
    self-tests: the check must report them)."""
    v = _Vals(name)
    if compact:
        lda = ldw = ldo = a_bs = w_bs = o_bs = ld_res = res_bs = None
        bias_bs = M if bias_row else 0
    act = 2 if geglu else act
    alpha = 1.0 if geglu else 0.75          # the GEGLU epilogue takes no alpha
    n_out = N // 2 if geglu else N
    a_rows, a_cols = (K, M) if a_mn else (M, K)
    w_rows, w_cols = (K, N) if w_mn else (N, K)
    lda, ldw, ldo = lda or ru8(a_cols), ldw or ru8(w_cols), ldo or n_out      # TMA pitches: 16-byte multiples
    a_bs = a_bs or a_rows * lda
    w_bs = 0 if shared_w else (w_bs or w_rows * ldw)
    o_bs = o_bs or M * ldo
    ld_res = ld_res or n_out
    res_bs = res_bs or M * ld_res
    odt = F32 if out_f32 else F16

    ops = {}
    shp = (batch, a_rows, a_cols - 1 if short_a else a_cols)
    ops["A"] = Op("in", F16, shp, (a_bs, lda, 1), pad=lda, values=v.randn(shp, F16, 0.5))
    shp = (1 if shared_w else batch, w_rows, w_cols)
    ops["W"] = Op("in", F16, shp, (w_bs or w_rows * ldw, ldw, 1), pad=ldw, values=v.randn(shp, F16, 0.5))
    if bias:
        if bias_row:
            bs = bias_bs or M
            ops["bias"] = Op("in", F32, (batch, M), (bs, 1), values=v.randn((batch, M)))
        else:
            ops["bias"] = Op("in", F32, (N,), values=v.randn((N,)))
    if residual:
        shp = (batch, M, n_out)
        ops["res"] = Op("in", odt, shp, (res_bs, ld_res, 1), pad=ld_res, values=v.randn(shp, odt))
    o_rows = M - 1 if short_out else M
    shp = (batch, o_rows, n_out)
    ops["out"] = Op("out", odt, shp, (o_bs, ldo, 1), pad=2 * ldo)
    if out2:
        ops["out2"] = Op("out", F16, shp, (o_bs, ldo, 1), pad=2 * ldo)
    if stats_rows:
        shp = (M // stats_rows, n_out, 2)
        ops["stats"] = Op("inout", F64, shp, values=torch.zeros(shp, dtype=F64), tol=(1e-9, 1e-9))

    def call(L, p, s):
        return L.b200_linear(_v(p["A"]), lda, a_bs if batch > 1 else 0, _v(p["W"]), ldw, w_bs if batch > 1 else 0,
                             M, N, K, batch, _v(p.get("bias")), int(bias_row), _v(p.get("res")), ld_res,
                             res_bs if batch > 1 else 0, _v(p["out"]), ldo, o_bs if batch > 1 else 0, int(out_f32),
                             act, alpha, _v(p.get("stats")), stats_rows, _v(p.get("out2")), int(res_mul), int(a_mn),
                             int(w_mn), bias_bs if batch > 1 else 0, s)

    def setup(L):
        L.b200_debug_set_swap(swap)
        L.b200_debug_set_flags(flags)
    meta = dict(M=M, N=N, K=K, batch=batch, act=act, alpha=alpha, bias_row=bias_row, res_mul=res_mul, a_mn=a_mn,
                w_mn=w_mn, stats_rows=stats_rows)
    return Case(name, "b200_linear", ops, call, setup, record=True, meta=meta)


def linear_cases():
    return [
        # pitch gaps on every operand, ragged M and N against the 64 / 128 / 256 tiles
        paired(linear_case, "linear_pitched", 200, 136, 72, lda=88, ldw=96, ldo=144, bias=True, residual=True, ld_res=152),
        paired(linear_case, "linear_pitched_noswap", 200, 136, 72, lda=88, ldw=96, ldo=144, residual=True, ld_res=152, swap=0),
        paired(linear_case, "linear_swap_f32_staged", 300, 256, 136, lda=144, ldw=144, ldo=264, out_f32=True, residual=True,
                    ld_res=264, flags=64),
        paired(linear_case, "linear_ragged_gelu", 77, 40, 40, lda=48, ldw=48, ldo=48, act=3),
        paired(linear_case, "linear_batched_gaps", 70, 90, 64, batch=3, lda=72, ldw=80, ldo=96, a_bs=70 * 72 + 40,
                    w_bs=90 * 80 + 24, o_bs=70 * 96 + 56, residual=True, ld_res=104, res_bs=70 * 104 + 8),
        paired(linear_case, "linear_batched_shared_w", 65, 129, 48, batch=2, lda=56, ldo=136, shared_w=True, a_bs=65 * 56 + 8,
                    o_bs=65 * 136 + 16),
        paired(linear_case, "linear_a_mn", 136, 200, 96, a_mn=True, lda=152, ldw=104, ldo=208, out_f32=True),
        paired(linear_case, "linear_w_mn", 130, 192, 80, w_mn=True, lda=88, ldw=200, ldo=200),
        paired(linear_case, "linear_a_mn_w_mn_batched", 100, 128, 70, batch=2, a_mn=True, w_mn=True, lda=112, ldw=136,
                    ldo=136, a_bs=70 * 112 + 32, w_bs=70 * 136 + 16, o_bs=100 * 136 + 24, bias=False),
        paired(linear_case, "linear_bias_row_batched", 90, 77, 64, batch=2, lda=64, ldw=72, ldo=88, bias_row=True, bias_bs=96,
                    a_bs=90 * 64 + 16, w_bs=77 * 72 + 8, o_bs=90 * 88 + 8, act=4),
        paired(linear_case, "linear_res_mul", 96, 136, 64, ldo=144, residual=True, ld_res=152, res_mul=True),
        paired(linear_case, "linear_geglu", 150, 320, 64, geglu=True, lda=72, ldo=168),
        paired(linear_case, "linear_stats_out2", 256, 192, 64, lda=72, ldo=200, out_f32=True, out2=True, stats_rows=128),
        paired(linear_case, "linear_stats_swap_vec", 256, 256, 64, ldo=264, out_f32=True, out2=True, stats_rows=64),
        paired(linear_case, "linear_stats_staged", 256, 256, 64, ldo=264, out_f32=True, out2=True, stats_rows=64, flags=64),
    ]


# ------------------------------------------------------------------------------------------------ b200_conv2d_nhwc
def conv_case(name, NB, H, W, Cin, Cout, *, taps=TAPS3, stride=1, Ho=None, Wo=None, C2=0, out_mul=1, phase=(0, 0),
              bias=True, rowvec=False, ld_rowvec=0, residual=False, out_f32=False, out_nchw=False, act=0,
              stats=False, out2=False, halo=1, swap=1, compact=False):
    v = _Vals(name)
    ld_rowvec = Cout if compact else ld_rowvec
    Ho, Wo = Ho or H, Wo or W
    odt = F32 if out_f32 else F16
    ops = {"X": Op("in", F16, (NB, H, W, Cin), values=v.randn((NB, H, W, Cin), F16, 0.5))}
    if C2:
        ops["X2"] = Op("in", F16, (NB, Ho, Wo, C2), values=v.randn((NB, Ho, Wo, C2), F16, 0.5))
    kw = len(taps) * Cin + C2
    ops["Wp"] = Op("in", F16, (Cout, kw), values=v.randn((Cout, kw), F16, 0.05))
    if bias:
        ops["bias"] = Op("in", F32, (Cout,), values=v.randn((Cout,)))
    if rowvec:
        ops["rowvec"] = Op("in", F32, (NB, Cout), (ld_rowvec, 1), pad=ld_rowvec, values=v.randn((NB, Cout)))
    OHm, OWm = Ho * out_mul, Wo * out_mul
    oshape = (NB, Cout, OHm, OWm) if out_nchw else (NB, OHm, OWm, Cout)
    oy, ox = phase

    def phase_mask(idx):
        return idx[:, :, oy::out_mul, ox::out_mul] if out_nchw else idx[:, oy::out_mul, ox::out_mul, :]
    if residual:
        ops["res"] = Op("in", odt, oshape, values=v.randn(oshape, odt), mask=phase_mask)
    ops["out"] = Op("out", odt, oshape, mask=phase_mask)
    if out2:
        ops["out2"] = Op("out", F16, oshape, mask=phase_mask)
    if stats:
        ops["stats"] = Op("inout", F64, (NB, Cout, 2), values=torch.zeros((NB, Cout, 2), dtype=F64), tol=(1e-9, 1e-9))
    dy = (ctypes.c_int * len(taps))(*[t[0] for t in taps])
    dx = (ctypes.c_int * len(taps))(*[t[1] for t in taps])

    def call(L, p, s):
        return L.b200_conv2d_nhwc(_v(p["X"]), NB, H, W, Cin, _v(p.get("X2")), C2, _v(p["Wp"]), Cout, len(taps), dy, dx,
                                  stride, Ho, Wo, out_mul, oy, ox, _v(p.get("bias")), _v(p.get("rowvec")), ld_rowvec,
                                  _v(p.get("res")), _v(p["out"]), int(out_f32), int(out_nchw), act,
                                  _v(p.get("stats")), _v(p.get("out2")), s)

    def setup(L):
        L.b200_debug_set_halo(halo)
        L.b200_debug_set_swap(swap)
    meta = dict(NB=NB, H=H, W=W, Cin=Cin, Cout=Cout, C2=C2, taps=taps, stride=stride, Ho=Ho, Wo=Wo, act=act,
                out_mul=out_mul, phase=phase, out_nchw=out_nchw)
    return Case(name, "b200_conv2d_nhwc", ops, call, setup, record=True, meta=meta)


def conv_phase_cases(name, Cout, **kw):
    """The four parity phases of a stride-2 data gradient / nearest-2x upsample conv, each into the same layout."""
    return [conv_case(f"{name}_phase{oy}{ox}", 2, 7, 9, 64, Cout, taps=TAPS2, out_mul=2, phase=(oy, ox), **kw)
            for oy in (0, 1) for ox in (0, 1)]


def conv_cases():
    return [
        conv_case("conv_halo_nb1", 1, 13, 11, 64, 128, residual=True, halo=1),
        conv_case("conv_halo_nb2_f32_stats", 2, 9, 10, 64, 128, out_f32=True, residual=True, stats=True, out2=True),
        paired(conv_case, "conv_pertap_nb2", 2, 13, 11, 64, 128, residual=True, rowvec=True, ld_rowvec=136, halo=0, act=1),
        paired(conv_case, "conv_normal_x2", 2, 9, 7, 64, 96, C2=64, rowvec=True, ld_rowvec=104, act=1),
        conv_case("conv_normal_stats_out2", 2, 8, 8, 64, 64, out_f32=True, stats=True, out2=True, swap=0),
        conv_case("conv_stride2", 2, 14, 13, 64, 128, taps=TAPS3_PAD0, stride=2, Ho=6, Wo=6),
        conv_case("conv_nchw", 2, 9, 11, 64, 4, out_f32=True, out_nchw=True),
        *conv_phase_cases("conv_dgrad_s2", 128, out_f32=True),
        *conv_phase_cases("conv_upsample", 64, residual=True),
    ]


# ------------------------------------------------------------------------------------------------ attention
def attention_case(name, D, *, B=2, heads=2, Lq=70, Lk=77, kv_segments=1, lse=True, entry="b200_attention",
                   compact=False):
    v = _Vals(name)
    C = heads * D
    q_ls, k_ls, v_ls, o_ls = (C, C, C, C) if compact else (C + 24, C + 8, C + 16, C + 40)
    q_bs, k_bs, v_bs, o_bs = ((Lq * C, Lk * C, Lk * C, Lq * C) if compact else
                              (Lq * q_ls + 8, (Lk + 5) * k_ls, (Lk + 3) * v_ls + 16, Lq * o_ls + 24))
    ops = {
        "q": Op("in", F16, (B, Lq, C), (q_bs, q_ls, 1), pad=q_ls, values=v.randn((B, Lq, C), F16)),
        "k": Op("in", F16, (B, Lk, C), (k_bs, k_ls, 1), pad=5 * k_ls, values=v.randn((B, Lk, C), F16)),
        "v": Op("in", F16, (B, Lk, C), (v_bs, v_ls, 1), pad=3 * v_ls, values=v.randn((B, Lk, C), F16)),
        "o": Op("out", F16, (B, Lq, C), (o_bs, o_ls, 1), pad=o_ls),
    }
    if lse:
        ops["lse"] = Op("out", F32, (B, heads, Lq))
    scale = D ** -0.5

    def call(L, p, s):
        args = (_v(p["q"]), q_bs, q_ls, _v(p["k"]), k_bs, k_ls, _v(p["v"]), v_bs, v_ls, _v(p["o"]), o_bs, o_ls, B, heads)
        if entry == "b200_attention_d64":
            return L.b200_attention_d64(*args, Lq, Lk, kv_segments, scale, _v(p.get("lse")), s)
        return L.b200_attention(*args, D, Lq, Lk, kv_segments, scale, _v(p.get("lse")), s)
    return Case(name, entry, ops, call, meta=dict(heads=heads, D=D, kv_segments=kv_segments, scale=scale))


def attention_d512_case(name, B=2, Lq=70, Lk=77, compact=False):
    v = _Vals(name)
    q_ls, k_ls, v_ls, o_ls = (512,) * 4 if compact else (536, 520, 528, 520)
    q_bs, k_bs, v_bs, o_bs = ((Lq * 512, Lk * 512, Lk * 512, Lq * 512) if compact else
                              (Lq * q_ls + 8, (Lk + 4) * k_ls, Lk * v_ls + 16, Lq * o_ls + 8))
    ops = {
        "q": Op("in", F16, (B, Lq, 512), (q_bs, q_ls, 1), pad=q_ls, values=v.randn((B, Lq, 512), F16, 0.3)),
        "k": Op("in", F16, (B, Lk, 512), (k_bs, k_ls, 1), pad=4 * k_ls, values=v.randn((B, Lk, 512), F16, 0.3)),
        "v": Op("in", F16, (B, Lk, 512), (v_bs, v_ls, 1), pad=v_ls, values=v.randn((B, Lk, 512), F16)),
        "o": Op("out", F16, (B, Lq, 512), (o_bs, o_ls, 1), pad=o_ls),
    }

    def call(L, p, s):
        return L.b200_attention_d512(_v(p["q"]), q_bs, q_ls, _v(p["k"]), k_bs, k_ls, _v(p["v"]), v_bs, v_ls,
                                     _v(p["o"]), o_bs, o_ls, B, Lq, Lk, 512 ** -0.5, s)
    return Case(name, "b200_attention_d512", ops, call, meta=dict(heads=1, D=512, kv_segments=1, scale=512 ** -0.5))


def attention_cases():
    c = [paired(attention_case, f"attention_d{D}_lk{Lk}", D, Lk=Lk) for D in (40, 80, 160) for Lk in (1, 77, 129)]
    c += [paired(attention_case, f"attention_d64_lk{Lk}", 64, Lk=Lk, entry="b200_attention_d64") for Lk in (1, 77, 129)]
    return c + [paired(attention_case, "attention_d80_joint", 80, B=4, kv_segments=2),
                paired(attention_case, "attention_d64_joint_nolse", 64, B=4, kv_segments=2, lse=False),
                paired(attention_case, "attention_d64_generic_entry", 64, Lk=33),
                paired(attention_d512_case, "attention_d512"),
                paired(attention_d512_case, "attention_d512_lk1", B=1, Lk=1)]


# ------------------------------------------------------------------------------------------------ row kernels
def rowdot_case(D, entry="b200_rowdot_heads_d", compact=False):
    name = f"rowdot_d{D}" + ("_generic" if entry == "b200_rowdot_heads" else "")
    v = _Vals(name)
    B, L_, heads = 2, 37, 3
    C = heads * D
    a_ls, c_ls = (C, C) if compact else (3 * C, C + 8)    # a: a head slice of a fused buffer, c: padded rows
    a_bs, c_bs = (L_ * C, L_ * C) if compact else (L_ * a_ls + 16, L_ * c_ls + 8)
    ops = {"a": Op("in", F16, (B, L_, C), (a_bs, a_ls, 1), offset=0 if compact else C, pad=a_ls, values=v.randn((B, L_, C), F16)),
           "c": Op("in", F16, (B, L_, C), (c_bs, c_ls, 1), pad=c_ls, values=v.randn((B, L_, C), F16)),
           "out": Op("out", F32, (B, heads, L_))}

    def call(L, p, s):
        if entry == "b200_rowdot_heads":
            return L.b200_rowdot_heads(_v(p["a"]), a_bs, a_ls, _v(p["c"]), c_bs, c_ls, B, L_, heads, _v(p["out"]), s)
        return L.b200_rowdot_heads_d(_v(p["a"]), a_bs, a_ls, _v(p["c"]), c_bs, c_ls, B, L_, heads, D, _v(p["out"]), s)
    return Case(name, entry, ops, call, meta=dict(heads=heads, D=D))


def softmax_rows_case(name, rows, cols, lds, ldp, compact=False):
    v = _Vals(name)
    lds, ldp = (cols, cols) if compact else (lds, ldp)
    ops = {"S": Op("in", F32, (rows, cols), (lds, 1), pad=lds, values=v.randn((rows, cols), F32, 3.0)),
           "P": Op("out", F16, (rows, cols), (ldp, 1), pad=ldp)}
    return Case(name, "b200_softmax_rows", ops,
                lambda L, p, s: L.b200_softmax_rows(_v(p["S"]), lds, _v(p["P"]), ldp, rows, cols, 0.7, s),
                meta=dict(scale=0.7))


def softmax_groups_case(compact=False):
    name = "softmax_groups"
    v = _Vals(name)
    rows, heads, S, ld_in, ld_out = 75, 5, 3, 15 if compact else 24, 24
    ops = {"logits": Op("in", F32, (rows, heads * S), (ld_in, 1), pad=ld_in, values=v.randn((rows, heads * S))),
           "P": Op("out", F16, (rows, ld_out), zero=lambda i: i[:, heads * S:])}
    return Case(name, "b200_softmax_groups", ops,
                lambda L, p, s: L.b200_softmax_groups(_v(p["logits"]), ld_in, rows, heads, S, _v(p["P"]), ld_out, s),
                meta=dict(heads=heads, S=S))


def softmax_bwd_case(compact=False):
    name = "softmax_bwd_rows"
    v = _Vals(name)
    rows, cols, ldp, ldd = (37, 77, 77, 77) if compact else (37, 77, 88, 84)
    ops = {"P": Op("in", F16, (rows, cols), (ldp, 1), pad=ldp, values=v.uniform((rows, cols), 0, 0.1, F16)),
           "dP": Op("in", F32, (rows, cols), (ldd, 1), pad=ldd, values=v.randn((rows, cols))),
           "dS": Op("out", F16, (rows, cols), (ldp, 1), pad=ldp)}
    return Case(name, "b200_softmax_bwd_rows", ops,
                lambda L, p, s: L.b200_softmax_bwd_rows(_v(p["P"]), ldp, _v(p["dP"]), ldd, _v(p["dS"]), rows, cols,
                                                        0.3, s), meta=dict(scale=0.3))


def gather_planar_case(name, NB, H, W, C, ldx, *, in_f32=False, Ho=None, Wo=None, stride=1, up=1, oy=0, ox=0,
                       ldo=None, compact=False):
    v = _Vals(name)
    Ho, Wo = Ho or H, Wo or W
    P = NB * Ho * Wo
    ldx, ldo = (C, None) if compact else (ldx, ldo)
    ldo = ldo or ru8(P)
    dt = F32 if in_f32 else F16
    shp = (NB, H, W, C)
    ops = {"x": Op("in", dt, shp, (H * W * ldx, W * ldx, ldx, 1), offset=8, pad=ldx, values=v.randn(shp, dt)),
           "out": Op("out", F16, (C, ldo), zero=lambda i: i[:, P:])}
    return Case(name, "b200_gather_planar", ops,
                lambda L, p, s: L.b200_gather_planar(_v(p["x"]), int(in_f32), ldx, NB, H, W, C, Ho, Wo, stride, up,
                                                     oy, ox, _v(p["out"]), ldo, s),
                meta=dict(Ho=Ho, Wo=Wo, stride=stride, up=up, oy=oy, ox=ox))


def col_sum_case(in_f32, compact=False):
    name = f"col_sum_{'f32' if in_f32 else 'f16'}"
    v = _Vals(name)
    rows, C, ld = 301, 72, 72 if compact else 88
    dt = F32 if in_f32 else F16
    ops = {"x": Op("in", dt, (rows, C), (ld, 1), pad=ld, values=v.randn((rows, C), dt)),
           "out": Op("inout", F32, (C,), values=v.randn((C,)), tol=(1e-5, 1e-5))}
    return Case(name, "b200_col_sum", ops,
                lambda L, p, s: L.b200_col_sum(_v(p["x"]), int(in_f32), rows, C, ld, _v(p["out"]), s))


def geglu_bwd_case(compact=False):
    name = "geglu_bwd"
    v = _Vals(name)
    rows, inner, ld_hg, ld_d = (45, 40, 40, 40) if compact else (45, 40, 96, 104)
    ops = {"h": Op("in", F16, (rows, inner), (ld_hg, 1), pad=ld_hg, values=v.randn((rows, inner), F16)),
           "g": Op("in", F16, (rows, inner), (ld_hg, 1), pad=ld_hg, values=v.randn((rows, inner), F16)),
           "dy": Op("in", F16, (rows, inner), values=v.randn((rows, inner), F16)),
           "dh": Op("out", F16, (rows, inner), (ld_d, 1), pad=ld_d),
           "dg": Op("out", F16, (rows, inner), (ld_d, 1), pad=ld_d)}
    return Case(name, "b200_geglu_bwd", ops,
                lambda L, p, s: L.b200_geglu_bwd(_v(p["h"]), _v(p["g"]), ld_hg, _v(p["dy"]), rows, inner, _v(p["dh"]),
                                                 _v(p["dg"]), ld_d, s))


def row_cases():
    c = [paired(rowdot_case, D) for D in (40, 64, 80, 160)] + [paired(rowdot_case, 64, "b200_rowdot_heads")]
    return c + [
        paired(softmax_rows_case, "softmax_rows_smem", 33, 77 * 4, 320, 312),
        paired(softmax_rows_case, "softmax_rows_vec4", 3, 16392, 16400, 16396),
        paired(softmax_rows_case, "softmax_rows_scalar", 35, 77, 81, 83),
        paired(softmax_groups_case), paired(softmax_bwd_case),
        paired(gather_planar_case, "gather_planar_slice", 2, 5, 7, 40, 136, ldo=ru8(70) + 64),
        paired(gather_planar_case, "gather_planar_s2", 2, 9, 9, 24, 32, in_f32=True, Ho=5, Wo=5, stride=2, oy=1, ox=1),
        paired(gather_planar_case, "gather_planar_up2", 1, 5, 6, 16, 24, Ho=10, Wo=12, up=2, ox=1),
        paired(col_sum_case, False), paired(col_sum_case, True), paired(geglu_bwd_case)]


# ------------------------------------------------------------------------------------------------ small-channel convs
def small_cout_case(Cout):
    name = f"conv3x3_small_cout_{Cout}"
    v = _Vals(name)
    NB, H, W, C = 2, 9, 13, 128
    ops = {"x": Op("in", F16, (NB, H, W, C), values=v.randn((NB, H, W, C), F16)),
           "wq": Op("in", F16, (C // 64, 9, 4, 8, 16), values=v.randn((C // 64, 9, 4, 8, 16), F16, 0.05)),
           "bias": Op("in", F32, (Cout,), values=v.randn((Cout,))),
           "out": Op("out", F32, (NB, Cout, H, W))}
    return Case(name, "b200_conv3x3_small_cout", ops,
                lambda L, p, s: L.b200_conv3x3_small_cout(_v(p["x"]), NB, H, W, C, _v(p["wq"]), _v(p["bias"]), Cout,
                                                          _v(p["out"]), s))


def im2col_case(C, x_f32):
    name = f"im2col3x3_c{C}_{'f32' if x_f32 else 'f16'}"
    v = _Vals(name)
    NB, H, W = 2, 7, 9
    kpad = ru8(9 * C)
    dt = F32 if x_f32 else F16
    ops = {"x": Op("in", dt, (NB, C, H, W), values=v.randn((NB, C, H, W), dt)),
           "out": Op("out", F16, (NB * H * W, kpad), zero=lambda i: i[:, 9 * C:])}
    return Case(name, "b200_im2col3x3_nchw", ops,
                lambda L, p, s: L.b200_im2col3x3_nchw(_v(p["x"]), int(x_f32), NB, C, H, W, _v(p["out"]), kpad, s))


# ------------------------------------------------------------------------------------------------ norms
def _gn_sums(v, NB, groups, n):
    s = v.randn((NB, groups, 1), F64, 0.1 * n)
    return torch.cat([s, s * s / n + n * v.uniform((NB, groups, 1), 0.5, 2.0, F64)], 2)


def _cs(v, NB, C, HW):
    s = v.randn((NB, C, 1), F64, 0.1 * HW)
    return torch.cat([s, s * s / HW + HW * v.uniform((NB, C, 1), 0.5, 2.0, F64)], 2)


def norm_cases():
    out = []
    NB, HW, C1, C2, G = 2, 45, 64, 32, 32
    for in_f32 in (0, 1):
        name = f"group_norm_stats_{in_f32}"
        v = _Vals(name)
        dt = F32 if in_f32 else F16
        ops = {"x1": Op("in", dt, (NB, HW, C1), values=v.randn((NB, HW, C1), dt)),
               "x2": Op("in", dt, (NB, HW, C2), values=v.randn((NB, HW, C2), dt)),
               "sums": Op("inout", F64, (NB, G, 2), values=torch.zeros((NB, G, 2), dtype=F64), tol=(1e-9, 1e-9))}
        out.append(Case(name, "b200_group_norm_stats", ops,
                        lambda L, p, s, f=in_f32: L.b200_group_norm_stats(_v(p["x1"]), C1, _v(p["x2"]), C2, f, NB, HW,
                                                                          G, _v(p["sums"]), s)))
    C = C1 + C2
    name = "group_norm_apply"
    v = _Vals(name)
    ops = {"x1": Op("in", F16, (NB, HW, C1), values=v.randn((NB, HW, C1), F16)),
           "x2": Op("in", F16, (NB, HW, C2), values=v.randn((NB, HW, C2), F16)),
           "sums": Op("in", F64, (NB, G, 2), values=_gn_sums(v, NB, G, HW * C // G)),
           "gamma": Op("in", F32, (C,), values=v.randn((C,))), "beta": Op("in", F32, (C,), values=v.randn((C,))),
           "y": Op("out", F16, (NB, HW, C)), "raw": Op("out", F16, (NB, HW, C))}
    out.append(Case(name, "b200_group_norm_apply", ops,
                    lambda L, p, s: L.b200_group_norm_apply(_v(p["x1"]), C1, _v(p["x2"]), C2, 0, NB, HW, G,
                                                            _v(p["sums"]), _v(p["gamma"]), _v(p["beta"]), 1e-6, 1,
                                                            _v(p["y"]), _v(p["raw"]), s)))
    name = "group_norm_apply_cs"
    v = _Vals(name)
    ops = {"x1": Op("in", F32, (NB, HW, C1), values=v.randn((NB, HW, C1))),
           "cs1": Op("in", F64, (NB, C1, 2), values=_cs(v, NB, C1, HW)),
           "x2": Op("in", F32, (NB, HW, C2), values=v.randn((NB, HW, C2))),
           "cs2": Op("in", F64, (NB, C2, 2), values=_cs(v, NB, C2, HW)),
           "gamma": Op("in", F32, (C,), values=v.randn((C,))), "beta": Op("in", F32, (C,), values=v.randn((C,))),
           "y": Op("out", F16, (NB, HW, C)), "raw": Op("out", F16, (NB, HW, C))}
    out.append(Case(name, "b200_group_norm_apply_cs", ops,
                    lambda L, p, s: L.b200_group_norm_apply_cs(_v(p["x1"]), C1, _v(p["cs1"]), _v(p["x2"]), C2,
                                                               _v(p["cs2"]), 1, NB, HW, G, _v(p["gamma"]),
                                                               _v(p["beta"]), 1e-6, 0, _v(p["y"]), _v(p["raw"]), s)))
    for use_cs in (0, 1):
        name = f"group_norm_mean_rstd_{'cs' if use_cs else 'sums'}"
        v = _Vals(name)
        ops = {"mr": Op("out", F32, (NB, G, 2))}
        if use_cs:
            ops["cs1"] = Op("in", F64, (NB, C1, 2), values=_cs(v, NB, C1, HW))
            ops["cs2"] = Op("in", F64, (NB, C2, 2), values=_cs(v, NB, C2, HW))
        else:
            ops["sums"] = Op("in", F64, (NB, G, 2), values=_gn_sums(v, NB, G, HW * C // G))
        out.append(Case(name, "b200_group_norm_mean_rstd", ops,
                        lambda L, p, s: L.b200_group_norm_mean_rstd(_v(p.get("sums")), _v(p.get("cs1")), C1,
                                                                    _v(p.get("cs2")), C2, NB, HW, G, 1e-6,
                                                                    _v(p["mr"]), s)))
    # GroupNorm backward of the second input of a concat: channels [c_off, c_off + Cx) of S and only those
    Ctot, c_off, Cx = 96, 64, 32
    mr = torch.stack([torch.linspace(-0.2, 0.2, NB * G).reshape(NB, G),
                      torch.linspace(0.5, 1.5, NB * G).reshape(NB, G)], 2).float()
    for in_f32 in (0, 1):
        name = f"group_norm_bwd_{in_f32}"
        v = _Vals(name)
        dt = F32 if in_f32 else F16
        S_vals = v.randn((NB, Ctot, 2), F32, 10.0)
        S_mask = lambda i: i[:, c_off:c_off + Cx]   # noqa: E731
        ops_s = {"x": Op("in", dt, (NB, HW, Cx), values=v.randn((NB, HW, Cx), dt)),
                 "dy": Op("in", F16, (NB, HW, Ctot), values=v.randn((NB, HW, Ctot), F16)),
                 "mr": Op("in", F32, (NB, G, 2), values=mr),
                 "gamma": Op("in", F32, (Ctot,), values=v.randn((Ctot,))),
                 "beta": Op("in", F32, (Ctot,), values=v.randn((Ctot,))),
                 "S": Op("inout", F32, (NB, Ctot, 2), values=torch.zeros((NB, Ctot, 2)), mask=S_mask,
                         tol=(1e-4, 1e-4))}
        out.append(Case(name + "_sums", "b200_group_norm_bwd_sums", ops_s,
                        lambda L, p, s, f=in_f32: L.b200_group_norm_bwd_sums(
                            _v(p["x"]), f, Cx, c_off, Ctot, _v(p["dy"]), NB, HW, G, _v(p["mr"]), _v(p["gamma"]),
                            _v(p["beta"]), 1, _v(p["S"]), s)))
        ops_a = {k: o for k, o in ops_s.items() if k != "S"}
        # pass 2 reads S over every group the slice touches: group 21 (channels 63..65) straddles c_off
        cpg = Ctot // G
        lo, hi = c_off // cpg * cpg, ((c_off + Cx - 1) // cpg + 1) * cpg
        ops_a["S"] = Op("in", F32, (NB, Ctot, 2), values=S_vals, mask=lambda i, lo=lo, hi=hi: i[:, lo:hi])
        ops_a["add"] = Op("in", dt, (NB, HW, Cx), values=v.randn((NB, HW, Cx), dt))
        ops_a["dx"] = Op("out", dt, (NB, HW, Cx))
        out.append(Case(name + "_apply", "b200_group_norm_bwd_apply", ops_a,
                        lambda L, p, s, f=in_f32: L.b200_group_norm_bwd_apply(
                            _v(p["x"]), f, Cx, c_off, Ctot, _v(p["dy"]), NB, HW, G, _v(p["mr"]), _v(p["gamma"]),
                            _v(p["beta"]), 1, _v(p["S"]), _v(p["add"]), _v(p["dx"]), f, s)))
    rows, C = 37, 72
    for in_f32 in (0, 1):
        name = f"layer_norm_{in_f32}"
        v = _Vals(name)
        dt = F32 if in_f32 else F16
        ops = {"x": Op("in", dt, (rows, C), values=v.randn((rows, C), dt)),
               "gamma": Op("in", F32, (C,), values=v.randn((C,))), "beta": Op("in", F32, (C,), values=v.randn((C,))),
               "y": Op("out", F16, (rows, C))}
        out.append(Case(name, "b200_layer_norm", ops,
                        lambda L, p, s, f=in_f32: L.b200_layer_norm(_v(p["x"]), f, rows, C, _v(p["gamma"]),
                                                                    _v(p["beta"]), 1e-5, _v(p["y"]), s)))
        name = f"layer_norm_bwd_{in_f32}"
        v = _Vals(name)
        ops = {"x": Op("in", dt, (rows, C), values=v.randn((rows, C), dt)),
               "gamma": Op("in", F32, (C,), values=v.randn((C,))),
               "dy": Op("in", F16, (rows, C), values=v.randn((rows, C), F16)),
               "add": Op("in", dt, (rows, C), values=v.randn((rows, C), dt)),
               "dx": Op("out", dt, (rows, C)),
               "dgamma": Op("inout", F32, (C,), values=torch.zeros(C), tol=(1e-4, 1e-4)),
               "dbeta": Op("inout", F32, (C,), values=torch.zeros(C), tol=(1e-4, 1e-4))}
        out.append(Case(name, "b200_layer_norm_bwd", ops,
                        lambda L, p, s, f=in_f32: L.b200_layer_norm_bwd(
                            _v(p["x"]), f, rows, C, _v(p["gamma"]), _v(p["dy"]), 1e-5, _v(p["add"]), _v(p["dx"]), f,
                            _v(p["dgamma"]), _v(p["dbeta"]), s)))
    return out


# ------------------------------------------------------------------------------------------------ elementwise et al.
def pointwise_case(compact=False):
    name = "pointwise_nchw"
    v = _Vals(name)
    NB, Cin, Cout, HW = 2, 4, 3, 77
    Cs = Cin if compact else 8          # in1 / in2: the first Cin channels of a Cs-channel tensor
    strided = (Cs * HW, HW, 1)
    ops = {"in1": Op("in", F32, (NB, Cin, HW), strided, pad=Cs * HW, values=v.randn((NB, Cin, HW))),
           "in2": Op("in", F32, (NB, Cin, HW), strided, pad=Cs * HW, values=v.randn((NB, Cin, HW))),
           "Wm": Op("in", F32, (Cout, Cin), values=v.randn((Cout, Cin))),
           "bias": Op("in", F32, (Cout,), values=v.randn((Cout,))),
           "out": Op("out", F32, (NB, Cout, HW))}
    return Case(name, "b200_pointwise_nchw", ops,
                lambda L, p, s: L.b200_pointwise_nchw(_v(p["in1"]), 0.5, _v(p["in2"]), -1.5, Cs, _v(p["Wm"]),
                                                      _v(p["bias"]), NB, Cin, Cout, HW, _v(p["out"]), s))


def ddim_case(mo_f16, compact=False):
    name = f"ddim_step_{mo_f16}"
    v = _Vals(name)
    B, C, HW = 2, 4, 75
    mdt = F16 if mo_f16 else F32
    # unet_in: the noisy-latent channel slice (channels C..2C) of the next step's [B][2C][HW] UNet input
    mo_bs, s_bs, ui_bs = (C * HW,) * 3 if compact else (C * HW + 20, C * HW + 4, 2 * C * HW)
    ops = {"mo": Op("in", mdt, (B, C, HW), (mo_bs, HW, 1), pad=20, values=v.randn((B, C, HW), mdt)),
           "x": Op("in", F32, (B, C, HW), (s_bs, HW, 1), pad=4, values=v.randn((B, C, HW))),
           "prev": Op("out", F32, (B, C, HW)), "x0": Op("out", F32, (B, C, HW)),
           "ui": Op("out", mdt, (B, C, HW), (ui_bs, HW, 1), offset=0 if compact else C * HW)}
    return Case(name, "b200_ddim_step", ops,
                lambda L, p, s: L.b200_ddim_step(_v(p["mo"]), mo_f16, mo_bs, _v(p["x"]), s_bs, B, C, HW, 1, 0.3, 0.6,
                                                 _v(p["prev"]), _v(p["x0"]), _v(p["ui"]), mo_f16, ui_bs, s))


def misc_cases():
    c = []
    NB, H, W, C = 2, 5, 7, 24
    for in_f32 in (0, 1):
        name = f"upsample_nearest_{in_f32}"
        v = _Vals(name)
        dt = F32 if in_f32 else F16
        ops = {"x": Op("in", dt, (NB, H, W, C), values=v.randn((NB, H, W, C), dt)),
               "y": Op("out", F16, (NB, 11, 13, C))}
        c.append(Case(name, "b200_upsample_nearest_nhwc", ops,
                         lambda L, p, s, f=in_f32: L.b200_upsample_nearest_nhwc(_v(p["x"]), f, NB, H, W, C, 11, 13,
                                                                                _v(p["y"]), s)))
    v = _Vals("upsample_nearest_bwd")
    ops = {"dy": Op("in", F32, (NB, 11, 13, C), values=v.randn((NB, 11, 13, C))),
           "add": Op("in", F32, (NB, H, W, C), values=v.randn((NB, H, W, C))),
           "dx": Op("out", F32, (NB, H, W, C))}
    c.append(Case("upsample_nearest_bwd", "b200_upsample_nearest_bwd", ops,
                     lambda L, p, s: L.b200_upsample_nearest_bwd(_v(p["dy"]), NB, H, W, C, 11, 13, _v(p["add"]),
                                                                 _v(p["dx"]), s)))
    v = _Vals("timestep_embedding")
    ops = {"t": Op("in", F32, (3,), values=torch.tensor([999.0, 0.0, 421.0])), "out": Op("out", F16, (3, 320))}
    c.append(Case("timestep_embedding", "b200_timestep_embedding", ops,
                     lambda L, p, s: L.b200_timestep_embedding(_v(p["t"]), 3, 320, _v(p["out"]), s)))
    for w_f32 in (0, 1):
        name = f"embed_tokens_{w_f32}"
        v = _Vals(name)
        rows, Lt, Ct, vocab = 2 * 7, 7, 40, 50
        dt = F32 if w_f32 else F16
        ops = {"ids": Op("in", I64, (rows,), values=v.ints((rows,), 0, vocab, I64)),
               "tok": Op("in", dt, (vocab, Ct), values=v.randn((vocab, Ct), dt)),
               "pos": Op("in", dt, (Lt, Ct), values=v.randn((Lt, Ct), dt)),
               "out": Op("out", F32, (rows, Ct))}
        c.append(Case(name, "b200_embed_tokens", ops,
                         lambda L, p, s, f=w_f32: L.b200_embed_tokens(_v(p["ids"]), _v(p["tok"]), _v(p["pos"]), f,
                                                                      rows, Lt, Ct, vocab, _v(p["out"]), s)))
    c.append(paired(pointwise_case))
    c += [paired(ddim_case, mo_f16) for mo_f16 in (0, 1)]
    NBd, HWp = 2, 77
    for mode in range(4):
        name = f"decode_post_{mode}"
        v = _Vals(name)
        oc = 3 if mode in (1, 3) else 1
        ops = {"x": Op("in", F32, (NBd, 3, HWp), values=v.randn((NBd, 3, HWp))), "out": Op("out", F32, (NBd, oc, HWp))}
        c.append(Case(name, "b200_decode_post", ops,
                         lambda L, p, s, m=mode: L.b200_decode_post(_v(p["x"]), NBd, HWp, m, -1.0, _v(p["out"]), s)))
        if mode >= 2:
            name = f"decode_post_bwd_{mode}"
            v = _Vals(name)
            ops = {"x": Op("in", F32, (NBd, 3, HWp), values=v.randn((NBd, 3, HWp))),
                   "dout": Op("in", F32, (NBd, oc, HWp), values=v.randn((NBd, oc, HWp))),
                   "dx": Op("out", F32, (NBd, 3, HWp))}
            c.append(Case(name, "b200_decode_post_bwd", ops,
                             lambda L, p, s, m=mode: L.b200_decode_post_bwd(_v(p["x"]), _v(p["dout"]), NBd, HWp, m,
                                                                            _v(p["dx"]), s)))
    n = 1037
    v = _Vals("cast_f32_to_f16")
    c.append(Case("cast_f32_to_f16", "b200_cast_f32_to_f16",
                     {"x": Op("in", F32, (n,), values=v.randn((n,))), "y": Op("out", F16, (n,))},
                     lambda L, p, s: L.b200_cast_f32_to_f16(_v(p["x"]), _v(p["y"]), n, s)))
    for in_f32 in (0, 1):
        name = f"nhwc_to_nchw_{in_f32}"
        v = _Vals(name)
        dt = F32 if in_f32 else F16
        ops = {"x": Op("in", dt, (2, 35, 12), values=v.randn((2, 35, 12), dt)), "y": Op("out", F32, (2, 12, 35))}
        c.append(Case(name, "b200_nhwc_to_nchw_f32", ops,
                         lambda L, p, s, f=in_f32: L.b200_nhwc_to_nchw_f32(_v(p["x"]), f, 2, 12, 35, _v(p["y"]), s)))
    for act in (1, 3):
        name = f"act_bwd_{act}"
        v = _Vals(name)
        ops = {"x": Op("in", F16, (n,), values=v.randn((n,), F16)), "dy": Op("in", F16, (n,), values=v.randn((n,), F16)),
               "dx": Op("out", F16, (n,))}
        c.append(Case(name, "b200_act_bwd", ops,
                         lambda L, p, s, a=act: L.b200_act_bwd(_v(p["x"]), _v(p["dy"]), n, a, _v(p["dx"]), s)))
    return c


def loss_optim_cases():
    c = []
    B, HW = 2, 301
    for kind, ch, ws_fwd, ws_bwd in (("ssi", 1, 5 * B + 2, 7 * B), ("angular", 3, 2, 1)):
        v = _Vals(kind + "_loss")
        base = {"pred": Op("in", F32, (B, ch, HW), values=v.randn((B, ch, HW))),
                "target": Op("in", F32, (B, ch, HW), values=v.randn((B, ch, HW))),
                "mask": Op("in", U8, (B, HW), values=v.mask((B, HW)))}
        fwd = dict(base, ws=Op("inout", F64, (ws_fwd,), values=torch.zeros(ws_fwd, dtype=F64), tol=(1e-9, 1e-9)),
                   out=Op("out", F32, (1,), tol=(1e-5, 1e-6)))
        c.append(Case(f"{kind}_loss", f"b200_{kind}_loss", fwd,
                         lambda L, p, s, k=kind: getattr(L, f"b200_{k}_loss")(_v(p["pred"]), _v(p["target"]), _v(p["mask"]),
                                                                         B, HW, _v(p["ws"]), _v(p["out"]), s)))
        bwd = dict(base, ws=Op("inout", F64, (ws_bwd,), values=torch.zeros(ws_bwd, dtype=F64), tol=(1e-9, 1e-9)),
                   go=Op("in", F32, (1,), values=torch.tensor([8.0])),
                   dpred=Op("out", F32, (B, ch, HW), tol=(1e-5, 1e-7)))
        c.append(Case(f"{kind}_loss_bwd", f"b200_{kind}_loss_bwd", bwd,
                         lambda L, p, s, k=kind: getattr(L, f"b200_{k}_loss_bwd")(
                             _v(p["pred"]), _v(p["target"]), _v(p["mask"]), B, HW, _v(p["ws"]), _v(p["go"]),
                             _v(p["dpred"]), s)))
    n = 1037
    v = _Vals("sumsq")
    c.append(Case("sumsq", "b200_sumsq", {"x": Op("in", F32, (n,), values=v.randn((n,))),
                                             "out": Op("inout", F64, (1,), values=torch.tensor([2.0], dtype=F64),
                                                       tol=(1e-12, 0.0))},
                     lambda L, p, s: L.b200_sumsq(_v(p["x"]), n, _v(p["out"]), s)))

    def adam_ops(name, n):
        v = _Vals(name)
        return {"param": Op("inout", F32, (n,), values=v.randn((n,))),
                "grad": Op("in", F32, (n,), values=v.randn((n,), F32, 0.1)),
                "m": Op("inout", F32, (n,), values=v.randn((n,), F32, 0.01)),
                "v2": Op("inout", F32, (n,), values=v.uniform((n,), 0.0, 1e-3)),
                "gn": Op("in", F64, (1,), values=torch.tensor([40.0], dtype=F64))}
    ops = adam_ops("adamw_step", n)
    c.append(Case("adamw_step", "b200_adamw_step", ops,
                     lambda L, p, s: L.b200_adamw_step(_v(p["param"]), _v(p["grad"]), _v(p["m"]), _v(p["v2"]), n, 1e-3,
                                                       0.9, 0.999, 1e-8, 1e-2, 3, _v(p["gn"]), 1.0, s)))
    ops = adam_ops("adamw_step_scaled", n)
    c.append(Case("adamw_step_scaled", "b200_adamw_step_scaled", ops,
                     lambda L, p, s: L.b200_adamw_step_scaled(_v(p["param"]), _v(p["grad"]), _v(p["m"]), _v(p["v2"]),
                                                              n, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 3, _v(p["gn"]), 1.0,
                                                              0.5, s)))
    state = torch.tensor([1024.0, 0, 2, 0, 0, 0, 0, 0])
    ops = adam_ops("adamw_step_state", n)
    ops["state"] = Op("inout", F32, (8,), values=state)
    c.append(Case("adamw_step_state", "b200_adamw_step_state", ops,
                     lambda L, p, s: L.b200_adamw_step_state(_v(p["param"]), _v(p["grad"]), _v(p["m"]), _v(p["v2"]), n,
                                                             1e-3, 0.9, 0.999, 1e-8, 1e-2, _v(p["gn"]), 1.0, 1.0,
                                                             _v(p["state"]), 1, 2000.0, 1.0, 65536.0, s)))
    ops = adam_ops("adamw_step_state_groups", n)
    ops["state"] = Op("inout", F32, (8,), values=state)
    ops["run_start"] = Op("in", I64, (3,), values=torch.tensor([0, 400, 800]))
    ops["run_group"] = Op("in", I32, (3,), values=torch.tensor([1, 0, 1], dtype=I32))
    lr, wd = (ctypes.c_float * 2)(1e-3, 1e-2), (ctypes.c_float * 2)(0.0, 0.1)
    c.append(Case("adamw_step_state_groups", "b200_adamw_step_state_groups", ops,
                     lambda L, p, s: L.b200_adamw_step_state_groups(
                         _v(p["param"]), _v(p["grad"]), _v(p["m"]), _v(p["v2"]), n, _v(p["run_start"]),
                         _v(p["run_group"]), 3, lr, wd, 2, 0.9, 0.999, 1e-8, _v(p["gn"]), 1.0, 1.0, _v(p["state"]), 1,
                         2000.0, 1.0, 65536.0, s)))
    v = _Vals("ema_update")
    c.append(Case("ema_update", "b200_ema_update", {"ema": Op("inout", F32, (n,), values=v.randn((n,))),
                                                       "param": Op("in", F32, (n,), values=v.randn((n,)))},
                     lambda L, p, s: L.b200_ema_update(_v(p["ema"]), _v(p["param"]), n, 1e-3, s)))
    # diffusion objective
    B, Cd, HWd, T = 2, 4, 63, 1000
    v = _Vals("diffusion_inputs")
    ops = {"rgb": Op("in", F32, (B, Cd, HWd), values=v.randn((B, Cd, HWd))),
           "x0": Op("in", F32, (2 * B, Cd, HWd), values=v.randn((2 * B, Cd, HWd))),
           "noise": Op("in", F32, (2 * B, Cd, HWd), values=v.randn((2 * B, Cd, HWd))),
           "t": Op("in", I64, (2 * B,), values=torch.tensor([0, 999, 311, 42])),
           "ac": Op("in", F32, (T,), values=torch.linspace(0.9991, 0.0047, T)),
           "unet_in": Op("out", F32, (2 * B, 2 * Cd, HWd)), "target": Op("out", F32, (2 * B, Cd, HWd))}
    c.append(Case("diffusion_inputs", "b200_diffusion_inputs", ops,
                     lambda L, p, s: L.b200_diffusion_inputs(_v(p["rgb"]), _v(p["x0"]), _v(p["noise"]), _v(p["t"]),
                                                             _v(p["ac"]), B, Cd, HWd, 1, _v(p["unet_in"]),
                                                             _v(p["target"]), s)))
    H, W, h, w = 40, 56, 5, 7
    for f16 in (0, 1):
        name = f"masked_latent_mse_{f16}"
        v = _Vals(name)
        dt = F16 if f16 else F32
        ops = {"pred": Op("in", dt, (2 * B, Cd, h, w), values=v.randn((2 * B, Cd, h, w), dt)),
               "target": Op("in", F32, (2 * B, Cd, h, w), values=v.randn((2 * B, Cd, h, w))),
               "vm": Op("in", U8, (B, H, W), values=v.mask((B, H, W), 0.995)),
               "lm": Op("out", U8, (B, h, w)),
               "ws": Op("inout", F64, (2,), values=torch.zeros(2, dtype=F64), tol=(1e-12, 0.0)),
               "out": Op("out", F32, (1,), tol=(1e-6, 0.0))}
        c.append(Case(name, "b200_masked_latent_mse", ops,
                         lambda L, p, s, f=f16: L.b200_masked_latent_mse(_v(p["pred"]), f, _v(p["target"]),
                                                                         _v(p["vm"]), B, Cd, H, W, h, w, _v(p["lm"]),
                                                                         _v(p["ws"]), _v(p["out"]), s)))
        name = f"masked_latent_mse_bwd_{f16}"
        v = _Vals(name)
        ops = {"pred": Op("in", dt, (2 * B, Cd, h, w), values=v.randn((2 * B, Cd, h, w), dt)),
               "target": Op("in", F32, (2 * B, Cd, h, w), values=v.randn((2 * B, Cd, h, w))),
               "lm": Op("in", U8, (B, h, w), values=v.mask((B, h, w))),
               "ws": Op("in", F64, (2,), values=torch.tensor([12.5, 40.0], dtype=F64)),
               "go": Op("in", F32, (1,), values=torch.tensor([4.0])),
               "grad": Op("out", dt, (2 * B, Cd, h, w))}
        c.append(Case(name, "b200_masked_latent_mse_bwd", ops,
                         lambda L, p, s, f=f16: L.b200_masked_latent_mse_bwd(_v(p["pred"]), f, _v(p["target"]),
                                                                             _v(p["lm"]), _v(p["ws"]), _v(p["go"]), B,
                                                                             Cd, h * w, _v(p["grad"]), s)))
    return c


def postproc_cases():
    c = []
    E, HW = 5, 301
    v = _Vals("ensemble_normals")
    ops = {"preds": Op("in", F32, (E, 3, HW), values=v.randn((E, 3, HW))), "err": Op("scratch", F64, (E,)),
           "out": Op("out", F32, (3, HW)), "index": Op("out", I32, (1,))}
    c.append(Case("ensemble_normals", "b200_ensemble_normals", ops,
                     lambda L, p, s: L.b200_ensemble_normals(_v(p["preds"]), E, HW, _v(p["err"]), _v(p["out"]),
                                                             _v(p["index"]), s)))
    for red in (0, 1):
        name = f"ensemble_depths_{red}"
        v = _Vals(name)
        base = {"imgs": Op("in", F32, (E, HW), values=v.uniform((E, HW), 0, 1)),
                "s": Op("in", F32, (E,), values=v.uniform((E,), 0.5, 1.5)),
                "t": Op("in", F32, (E,), values=v.uniform((E,), -0.2, 0.2))}
        obj = dict(base, ws=Op("out", F64, (2,), check=lambda i: i[:1], tol=(1e-12, 0.0)),
                   out3=Op("out", F32, (3,), mask=lambda i: i[1:]))
        c.append(Case(name + "_objective", "b200_ensemble_depths_objective", obj,
                         lambda L, p, s, r=red: L.b200_ensemble_depths_objective(
                             _v(p["imgs"]), _v(p["s"]), _v(p["t"]), E, HW, r, _v(p["ws"]), _v(p["out3"]), s)))
        rd = dict(base, ws=Op("scratch", F64, (2,)), aligned=Op("out", F32, (HW,)), unc=Op("out", F32, (HW,)))
        c.append(Case(name + "_reduce", "b200_ensemble_depths_reduce", rd,
                         lambda L, p, s, r=red: L.b200_ensemble_depths_reduce(
                             _v(p["imgs"]), _v(p["s"]), _v(p["t"]), E, HW, r, _v(p["ws"]), _v(p["aligned"]),
                             _v(p["unc"]), s)))
    v = _Vals("minmax_rows")
    ops = {"x": Op("in", F32, (E, HW), values=v.randn((E, HW))), "ws": Op("scratch", I32, (2 * E,)),
           "out": Op("out", F32, (E, 2))}
    c.append(Case("minmax_rows", "b200_minmax_rows", ops,
                     lambda L, p, s: L.b200_minmax_rows(_v(p["x"]), E, HW, _v(p["ws"]), _v(p["out"]), s)))
    v = _Vals("minmax_normalise")
    ops = {"x": Op("inout", F32, (HW,), values=v.randn((HW,))), "ws": Op("scratch", I32, (2,)),
           "mm": Op("out", F32, (2,))}
    c.append(Case("minmax_normalise", "b200_minmax_normalise", ops,
                     lambda L, p, s: L.b200_minmax_normalise(_v(p["x"]), HW, _v(p["ws"]), _v(p["mm"]), s)))
    for u8 in (0, 1):
        name = f"rgb_normalise_{u8}"
        v = _Vals(name)
        x = v.ints((HW,), 0, 256, U8) if u8 else v.uniform((HW,), 0, 255)
        ops = {"x": Op("in", U8 if u8 else F32, (HW,), values=x), "out": Op("out", F32, (HW,))}
        c.append(Case(name, "b200_rgb_normalise", ops,
                         lambda L, p, s, f=u8: L.b200_rgb_normalise(_v(p["x"]), f, HW, 1 - f, _v(p["out"]), s)))
    planes, H, W, OH, OW = 3, 13, 17, 7, 23
    for kind in ("bicubic_aa", "bilinear_aa"):
        name = f"resize_{kind}"
        v = _Vals(name)
        ops = {"x": Op("in", F32, (planes, H, W), values=v.randn((planes, H, W))),
               "tmp": Op("scratch", F32, (planes, H, OW)), "out": Op("out", F32, (planes, OH, OW))}
        c.append(Case(name, f"b200_resize_{kind}", ops,
                         lambda L, p, s, k=kind: getattr(L, f"b200_resize_{k}")(_v(p["x"]), planes, H, W, OH, OW,
                                                                                 _v(p["tmp"]), _v(p["out"]), s)))
    for kind in ("nearest", "nearest_exact"):
        name = f"resize_{kind}"
        v = _Vals(name)
        ops = {"x": Op("in", F32, (planes, H, W), values=v.randn((planes, H, W))), "out": Op("out", F32, (planes, OH, OW))}
        c.append(Case(name, f"b200_resize_{kind}", ops,
                         lambda L, p, s, k=kind: getattr(L, f"b200_resize_{k}")(_v(p["x"]), planes, H, W, OH, OW,
                                                                                 _v(p["out"]), s)))
    # colour outputs: 4-pixel vector stores and the scalar tail
    for n in (1025, 1026, 1027):
        name = f"colorize_depth_{n}"
        v = _Vals(name)
        x = v.uniform((n,), -0.1, 1.1)
        x[::97] = float("nan")
        ops = {"x": Op("in", F32, (n,), values=x), "table": Op("in", U8, (256, 3), values=v.ints((256, 3), 0, 256, U8)),
               "out": Op("out", U8, (n, 3))}
        c.append(Case(name, "b200_colorize_depth", ops,
                         lambda L, p, s, n=n: L.b200_colorize_depth(_v(p["x"]), n, _v(p["table"]), 256, _v(p["out"]), s)))
        name = f"colorize_normals_{n}"
        v = _Vals(name)
        ops = {"x": Op("in", F32, (3, n), values=v.uniform((3, n), -1.2, 1.2)), "out": Op("out", U8, (n, 3))}
        c.append(Case(name, "b200_colorize_normals", ops,
                         lambda L, p, s, n=n: L.b200_colorize_normals(_v(p["x"]), n, _v(p["out"]), s)))
    return c


def normal_error_case(cap_name, compact=False):
    """pred stored HWC ([B][H][W][3] read in place as [B][3][H][W]; CHW in the compact twin), gt CHW.  The short
    buffer holds a third of the masked angles: nothing may land past it, and *buf_len still counts them all."""
    B, H, W = 2, 13, 21
    name = f"eval_normal_error_{cap_name}"
    v = _Vals(name)
    m = v.mask((B, H, W))
    count = int(m.sum())
    cap = count + 40 if cap_name == "full" else count // 3
    pred_st = (3 * H * W, H * W, W, 1) if compact else (H * W * 3, 1, W * 3, 3)
    ops = {"pred": Op("in", F32, (B, 3, H, W), pred_st, values=v.randn((B, 3, H, W))),
           "gt": Op("in", F32, (B, 3, H, W), values=v.randn((B, 3, H, W))),
           "mask": Op("in", U8, (B, H, W), values=m),
           "err": Op("out", F32, (B, H, W)),
           "buf": Op("out", F32, (cap,), mask=lambda i: i[:min(count, cap)],
                     check=None if cap_name == "full" else (lambda i: i[:0]), sort=True),
           "buf_len": Op("inout", I64, (1,), values=torch.tensor([0])),
           "ws": Op("scratch", F64, (B * 512 * 8,)),
           "sums": Op("inout", F64, (2,), values=torch.tensor([1.0, 2.0], dtype=F64)),
           "counts": Op("inout", I64, (6,), values=torch.arange(6))}
    ps = (ctypes.c_longlong * 4)(*pred_st)
    gs = (ctypes.c_longlong * 4)(3 * H * W, H * W, W, 1)
    return Case(name, "b200_eval_normal_error", ops,
                lambda L, p, s: L.b200_eval_normal_error(
                    _v(p["pred"]), ps, _v(p["gt"]), gs, _v(p["mask"]), B, H, W, _v(p["err"]), _v(p["buf"]), cap,
                    _v(p["buf_len"]), _v(p["ws"]), _v(p["sums"]), _v(p["counts"]), s),
                meta=dict(count=count))


def eval_cases():
    c = []
    B, H, W = 2, 13, 21
    MAXB = 512
    v = _Vals("eval_align_depth")
    ops = {"gt": Op("in", F32, (B, H, W), values=v.uniform((B, H, W), 0.5, 10)),
           "pred": Op("in", F32, (B, H, W), values=v.uniform((B, H, W), 0.0, 1.0)),
           "mask": Op("in", U8, (B, H, W), values=v.mask((B, H, W))),
           "ws": Op("scratch", F64, (B * MAXB * 7,)), "ss": Op("out", F32, (B, 2))}
    c.append(Case("eval_align_depth", "b200_eval_align_depth", ops,
                     lambda L, p, s: L.b200_eval_align_depth(_v(p["gt"]), _v(p["pred"]), _v(p["mask"]), B, H, W, 10,
                                                             0.5, 0, _v(p["ws"]), _v(p["ss"]), s)))
    v = _Vals("eval_depth_metrics")
    ops = {"pred": Op("in", F32, (B, H * W), values=v.uniform((B, H * W), 0.0, 1.0)),
           "gt": Op("in", F32, (B, H * W), values=v.uniform((B, H * W), 0.5, 10)),
           "mask": Op("in", U8, (B, H * W), values=v.mask((B, H * W))),
           "ss": Op("in", F32, (B, 2), values=torch.tensor([[8.0, 0.5], [6.0, 1.0]])),
           "aligned": Op("out", F32, (B, H * W)), "ws": Op("scratch", F64, (B * MAXB * 11,)),
           "out": Op("out", F32, (10,))}
    c.append(Case("eval_depth_metrics", "b200_eval_depth_metrics", ops,
                     lambda L, p, s: L.b200_eval_depth_metrics(_v(p["pred"]), _v(p["gt"]), _v(p["mask"]), B, H * W,
                                                               _v(p["ss"]), 0, 1, 1e-3, 8.0, _v(p["aligned"]),
                                                               _v(p["ws"]), _v(p["out"]), s)))
    c += [paired(normal_error_case, cap_name) for cap_name in ("full", "short")]
    v = _Vals("eval_kth_smallest")
    n, n_max = 301, 400
    ops = {"x": Op("in", F32, (n,), values=v.uniform((n,), 0, 50), pad=n_max - n),
           "n": Op("in", I64, (1,), values=torch.tensor([n])),
           "ws": Op("scratch", I64, (261,)), "out": Op("out", F32, (3,))}
    c.append(Case("eval_kth_smallest", "b200_eval_kth_smallest", ops,
                     lambda L, p, s: L.b200_eval_kth_smallest(_v(p["x"]), _v(p["n"]), n_max, -1, _v(p["ws"]),
                                                              _v(p["out"]), s)))
    return c


def data_cases():
    from diffusion_e2e_ft_b200 import data as D
    c = []
    B, H, W = 2, 13, 19
    v = _Vals("data_hypersim_source")
    ik = (ctypes.c_double * 9)(*D.hypersim_inv_k(H, W).reshape(-1).tolist())
    flip = torch.tensor([1, 0], dtype=U8)
    ops = {"depth": Op("in", I16, (B, H, W), values=v.ints((B, H, W), 0, 60000, I16)),
           "normal": Op("in", U8, (B, H, W, 3), values=v.ints((B, H, W, 3), 0, 256, U8)),
           "flip": Op("in", U8, (B,), values=flip),
           "depth_m": Op("out", F32, (B, H, W)), "normal_out": Op("out", U8, (B, H, W, 3))}
    c.append(Case("data_hypersim_source", "b200_data_hypersim_source", ops,
                     lambda L, p, s: L.b200_data_hypersim_source(_v(p["depth"]), _v(p["normal"]), _v(p["flip"]), B, H,
                                                                 W, ik, _v(p["depth_m"]), _v(p["normal_out"]), s)))
    OH, OW = 9, 11
    xmin, xk = D.pillow_bilinear_coeffs(W, OW)
    ymin, yk = D.pillow_bilinear_coeffs(H, OH)
    v = _Vals("data_resize_u8")
    ops = {"src": Op("in", U8, (B, H, W, 3), values=v.ints((B, H, W, 3), 0, 256, U8)),
           "xmin": Op("in", I32, xmin.shape, values=torch.from_numpy(xmin)),
           "xk": Op("in", I32, xk.shape, values=torch.from_numpy(xk)),
           "ymin": Op("in", I32, ymin.shape, values=torch.from_numpy(ymin)),
           "yk": Op("in", I32, yk.shape, values=torch.from_numpy(yk)),
           "flip": Op("in", U8, (B,), values=flip),
           "tmp": Op("scratch", U8, (B, H, OW, 3)), "dst": Op("out", U8, (B, OH, OW, 3))}
    c.append(Case("data_resize_u8", "b200_data_resize_u8", ops,
                     lambda L, p, s: L.b200_data_resize_u8(_v(p["src"]), B, H, W, 3, OH, OW, _v(p["xmin"]), _v(p["xk"]),
                                                           xk.shape[1], _v(p["ymin"]), _v(p["yk"]), yk.shape[1],
                                                           _v(p["flip"]), _v(p["tmp"]), _v(p["dst"]), s)))
    rows = torch.from_numpy(D.pillow_nearest_index(H, OH))
    cols = torch.from_numpy(D.pillow_nearest_index(W, OW))
    for src in ("m", "cm"):
        name = f"data_depth_gather_{src}"
        v = _Vals(name)
        sv = v.uniform((B, H, W), 0.1, 60.0) if src == "m" else v.ints((B, H, W), 0, 30000, I16)
        ops = {"src": Op("in", F32 if src == "m" else I16, (B, H, W), values=sv),
               "rows": Op("in", I32, (OH,), values=rows), "cols": Op("in", I32, (OW,), values=cols),
               "flip": Op("in", U8, (B,), values=flip), "dst": Op("out", F32, (B, OH, OW))}
        c.append(Case(name, "b200_data_depth_gather", ops,
                         lambda L, p, s, m=(src == "m"): L.b200_data_depth_gather(
                             _v(p["src"] if m else None), _v(None if m else p["src"]), B, H, W, OH, OW, _v(p["rows"]),
                             _v(p["cols"]), _v(p["flip"]), _v(p["dst"]), s)))
    v = _Vals("data_depth_range")
    d = v.uniform((B, OH * OW), 0.0, 70.0)
    ops = {"depth": Op("in", F32, (B, OH * OW), values=d), "range": Op("out", F32, (B, 2)), "flag": Op("out", I32, (B,))}
    c.append(Case("data_depth_range", "b200_data_depth_range", ops,
                     lambda L, p, s: L.b200_data_depth_range(_v(p["depth"]), B, OH * OW, 1e-5, 65.0, _v(p["range"]),
                                                             _v(p["flag"]), s)))
    v = _Vals("data_finalise")
    top, left = 2, 3
    ops = {"rgb": Op("in", U8, (B, H, W, 3), values=v.ints((B, H, W, 3), 0, 256, U8)),
           "normal": Op("in", U8, (B, H, W, 3), values=v.ints((B, H, W, 3), 0, 256, U8)),
           "flip": Op("in", U8, (B,), values=flip),
           "depth": Op("in", F32, (B, OH, OW), values=v.uniform((B, OH, OW), 0.0, 70.0)),
           "range": Op("in", F32, (B, 2), values=torch.tensor([[1.0, 50.0], [2.0, 30.0]])),
           "flag": Op("in", I32, (B,), values=torch.tensor([2, 2], dtype=I32)),
           "rgb_out": Op("out", F32, (B, 3, OH, OW)), "depth_out": Op("out", F32, (B, 3, OH, OW)),
           "metric": Op("out", F32, (B, OH, OW)), "normal_out": Op("out", F32, (B, 3, OH, OW)),
           "mask": Op("out", U8, (B, OH, OW))}
    c.append(Case("data_finalise", "b200_data_finalise", ops,
                     lambda L, p, s: L.b200_data_finalise(_v(p["rgb"]), _v(p["normal"]), B, H, W, top, left,
                                                          _v(p["flip"]), _v(p["depth"]), OH, OW, 1e-5, 65.0,
                                                          _v(p["range"]), _v(p["flag"]), _v(p["rgb_out"]),
                                                          _v(p["depth_out"]), _v(p["metric"]), _v(p["normal_out"]),
                                                          _v(p["mask"]), s)))
    v = _Vals("data_vkitti_normals")
    ops = {"depth": Op("in", I16, (B, H, W), values=v.ints((B, H, W), 100, 20000, I16)),
           "out": Op("out", I16, (B, H, W, 3))}
    c.append(Case("data_vkitti_normals", "b200_data_vkitti_normals", ops,
                     lambda L, p, s: L.b200_data_vkitti_normals(_v(p["depth"]), B, H, W, D.VKITTI_FX, D.VKITTI_FY,
                                                                D.VKITTI_U0, D.VKITTI_V0, _v(p["out"]), s)))
    n = 1037
    v = _Vals("debug_pow_e32_neg")
    ops = {"x": Op("in", F32, (n,), values=v.uniform((n,), 0.0, 20.0)), "out": Op("out", F32, (n,)),
           "slow": Op("inout", I32, (1,), values=torch.tensor([3], dtype=I32))}
    c.append(Case("debug_pow_e32_neg", "b200_debug_pow_e32_neg", ops,
                     lambda L, p, s: L.b200_debug_pow_e32_neg(_v(p["x"]), n, 0, _v(p["out"]), _v(p["slow"]), s)))
    v = _Vals("debug_hypersim_pow")
    ops = {"x": Op("in", F64, (n,), values=v.uniform((n,), 0.0, 1.0, F64)), "p": Op("out", F64, (n,)),
           "level": Op("out", U8, (n,)), "slow": Op("inout", I32, (1,), values=torch.tensor([0], dtype=I32))}
    c.append(Case("debug_hypersim_pow", "b200_debug_hypersim_pow", ops,
                     lambda L, p, s: L.b200_debug_hypersim_pow(_v(p["x"]), n, 0, _v(p["p"]), _v(p["level"]),
                                                               _v(p["slow"]), s)))
    for half in (0, 1):
        name = f"data_hypersim_frames_{half}"
        v = _Vals(name)
        dt = F16 if half else F32
        eid = v.ints((B, H, W), 1, 9, I32)
        eid[:, :2] = -1
        ws_elems = 1 << 17
        ops = {"rgb": Op("in", dt, (B, H, W, 3), values=v.uniform((B, H, W, 3), 0.0, 3.0, dt)),
               "dist": Op("in", dt, (B, H, W), values=v.uniform((B, H, W), 0.5, 20.0, dt)),
               "eid": Op("in", I32, (B, H, W), values=eid),
               "bgr": Op("out", U8, (B, H, W, 3)), "depth": Op("out", I16, (B, H, W)), "err": Op("out", I32, (B,)),
               "stats": Op("out", F64, (B, 2)), "ws": Op("scratch", F64, (ws_elems,))}

        def call(L, p, s, half=half, ws_elems=ws_elems):
            assert L.b200_data_hypersim_workspace_bytes(B, H, W) <= ws_elems * 8
            return L.b200_data_hypersim_frames(_v(p["rgb"]), half, _v(p["dist"]), half, _v(p["eid"]), B, H, W,
                                               D.HYPERSIM_FOCAL, D._tone_map_numerator(), _v(p["bgr"]),
                                               _v(p["depth"]), _v(p["err"]), _v(p["stats"]), _v(p["ws"]),
                                               ws_elems * 8, s)
        c.append(Case(name, "b200_data_hypersim_frames", ops, call))
    return c


def all_cases():
    return (linear_cases() + conv_cases() + attention_cases() + row_cases()
            + [small_cout_case(3), small_cout_case(4)] + [im2col_case(C, f) for C in (3, 4, 8) for f in (0, 1)]
            + norm_cases() + misc_cases() + loss_optim_cases() + postproc_cases() + eval_cases() + data_cases())


# Entry points without a memory footprint of their own, or whose footprint another entry point exercises.
EXEMPT = {
    "b200_last_error_string": "host-side string of the calling thread's last failure; touches no device memory",
    "b200_abi_version": "host-side constant",
    "b200_debug_force_block_n": "debug setter of a host-side tile-width switch; no device memory",
    "b200_debug_set_flags": "debug setter of host-side epilogue flags; the linear cases run with flag 64",
    "b200_debug_set_swap": "debug setter of the tile orientation; the linear / conv cases run both orientations",
    "b200_debug_set_halo": "debug setter of the conv path; the conv cases run the halo and per-tap paths",
    "b200_debug_last_path": "host-side record of the last conv path; no device memory",
    "b200_debug_last_launch": "host-side record of the last GEMM launch; the footprint check compares it",
    "b200_geglu_block_n": "host-side tile-width query; no device memory",
    "b200_data_hypersim_workspace_bytes": "host-side size query; the hypersim_frames cases check their workspace",
}
