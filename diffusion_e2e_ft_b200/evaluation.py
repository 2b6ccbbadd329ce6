"""Evaluation of depth and normal predictions on the device (DESIGN.md §3 "Evaluation").

    align_depth_least_square            <- Marigold/src/util/alignment.py:8-55
    metric.<name> (the ten depth metrics) <- Marigold/src/util/metric.py
    DepthEvaluator                      <- the per-sample loop of Marigold/eval.py:147-220 + MetricTracker
    compute_normal_error                <- DSINE/utils/utils.py:150-159
    NormalEvaluator                     <- DSINE/projects/dsine/test.py:100-130 + compute_normal_metrics (utils.py:162-180)

Signatures and return conventions are the reference's.  The arithmetic runs in libb200_e2eft.so
(csrc/evaluation.cu); torch only allocates.  Inputs are CUDA tensors (align_depth_least_square also takes numpy arrays
and then returns numpy arrays); maps are evaluated in fp32.  Shape, dtype and device errors raise ValueError before
anything is launched, and `update()` never synchronises with the host: rows, sums and pooled errors stay on the
device until `result()` / `per_sample()` copy them back once.
"""
import ctypes
import math
import types

import numpy as np
import torch

from . import lib as _lib
from .ops import _ck, _p, _stream

F32 = torch.float32
METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10",
           "delta1_acc", "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")       # Marigold/eval.py:46-57
NORMAL_METRICS = ("mean", "median", "rmse", "a1", "a2", "a3", "a4", "a5")
ALIGNMENTS = (None, "least_square", "least_square_disparity")
MAX_BLOCKS = 512                 # B200_EVAL_MAX_BLOCKS
KTH_WS_WORDS = 261               # B200_EVAL_KTH_WS_WORDS
_FIELDS = dict(align=7, depth=11, normal=8)


def _need_cuda(*ts):
    dev = None
    for t in ts:
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("diffusion_e2e_ft_b200.evaluation needs CUDA tensors (no CPU fallback), got "
                             f"{type(t).__name__ if not isinstance(t, torch.Tensor) else t.device}")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError(f"tensors on different devices: {dev} and {t.device}")


def _float_map(t, what):
    if not t.is_floating_point():
        raise ValueError(f"{what} must be a floating-point tensor, got {t.dtype}")
    return t.to(F32)


def _bool_mask(t, what):
    if t.dtype != torch.bool:
        raise ValueError(f"{what} must be a bool tensor, got {t.dtype}")
    return t.contiguous().view(torch.uint8)


def sampling_columns(H, W, max_resolution):
    """Columns of the grid alignment.py:21-32 takes its moments on: (OW, col_scale) with source column
    min(floor(float32(j) * col_scale), W - 1) for j < OW.  The reference hands torch.nn.Upsample(scale_factor=s,
    mode="nearest") a [1, H, W] tensor, which it interpolates along W only; s = min(max_res / H, max_res / W) applies
    when it is < 1, the output width is floor(W * s) and the fp32 source step is float(1 / s)."""
    if max_resolution is None:
        return W, 1.0
    s = float(np.min(max_resolution / np.array((H, W))))
    if not s < 1:
        return W, 1.0
    ow = math.floor(float(W) * s)
    if ow < 1:
        raise ValueError(f"max_resolution={max_resolution} leaves no column of a {H}x{W} map")
    return ow, float(np.float32(1.0 / s))


# ------------------------------------------------------------------------------------ one launch each
def align_scale_shift(gt, pred, mask, max_resolution=None, disparity=False):
    """[B,H,W] fp32 gt / pred and uint8 mask (CUDA) -> fp32 [B,2] (scale, shift) on the device: np.linalg.lstsq of
    [p 1] x = g over the mask on the sampling grid (disparity: target 1/gt, mask & gt > 0 & pred > 0)."""
    B, H, W = pred.shape
    ow, col_scale = sampling_columns(H, W, max_resolution)
    ws = torch.empty(B * MAX_BLOCKS * _FIELDS["align"], dtype=torch.float64, device=pred.device)
    out = torch.empty((B, 2), dtype=F32, device=pred.device)
    _ck(_lib.load().b200_eval_align_depth(_p(gt), _p(pred), _p(mask), B, H, W, ow, col_scale, int(disparity), _p(ws),
                                          _p(out), _stream()), "b200_eval_align_depth")
    return out


def depth_metrics(pred, gt, mask, scale_shift=None, disparity=False, clip=None, aligned=None, metrics=True):
    """[B,H,W] fp32 pred / gt, uint8 mask or None (CUDA) -> fp32 [10] device row of METRICS (None when not `metrics`).
    pred is first mapped as eval.py:173-210 does: * scale + shift, the disparity inversion, clip=(min, max) then
    >= 1e-6; `aligned` ([B,H,W] fp32) receives the mapped prediction."""
    B, H, W = pred.shape
    dev = pred.device
    ws = out = None
    if metrics:
        ws = torch.empty(B * MAX_BLOCKS * _FIELDS["depth"], dtype=torch.float64, device=dev)
        out = torch.empty(len(METRICS), dtype=F32, device=dev)
    lo, hi = clip if clip is not None else (0.0, 0.0)
    _ck(_lib.load().b200_eval_depth_metrics(_p(pred), _p(gt), _p(mask), B, H * W, _p(scale_shift), int(disparity),
                                            int(clip is not None), float(lo), float(hi), _p(aligned), _p(ws), _p(out),
                                            _stream()), "b200_eval_depth_metrics")
    return out


def _strides(t):
    return (ctypes.c_longlong * 4)(*t.stride())


def normal_error(pred, gt, mask=None, err_map=None, buf=None, buf_len=None, sums=None, counts=None):
    """[B,3,H,W] fp32 pred / gt with any element strides, uint8 [B,H,W] mask or None (CUDA).  Writes the angles in
    degrees to err_map ([B,H,W] fp32), appends the masked ones to buf at buf_len (uint64 [1]), and adds (sum e,
    sum e^2) to sums (fp64 [2]) and (n, #< 5, 7.5, 11.25, 22.5, 30) to counts (int64 [6])."""
    B, _, H, W = pred.shape
    ws = torch.empty(B * MAX_BLOCKS * _FIELDS["normal"], dtype=torch.float64, device=pred.device)
    cap = buf.numel() if buf is not None else 0
    _ck(_lib.load().b200_eval_normal_error(_p(pred), _strides(pred), _p(gt), _strides(gt), _p(mask), B, H, W,
                                           _p(err_map), _p(buf), cap, _p(buf_len), _p(ws), _p(sums), _p(counts),
                                           _stream()), "b200_eval_normal_error")


def kth_smallest(x, n, n_max, k=-1):
    """Exact k-th smallest (0-based) of the non-negative fp32 x[:n] with n a uint64 [1] device count (n_max >= n);
    k = -1: the median.  -> fp32 [3] device: (k-th, (k+1)-th, np.median for k = -1 else the k-th)."""
    ws = torch.empty(KTH_WS_WORDS, dtype=torch.int64, device=x.device)
    out = torch.empty(3, dtype=F32, device=x.device)
    _ck(_lib.load().b200_eval_kth_smallest(_p(x), _p(n), int(n_max), int(k), _p(ws), _p(out), _stream()),
        "b200_eval_kth_smallest")
    return out


# ------------------------------------------------------------------------------------ Marigold depth
def align_depth_least_square(gt_arr, pred_arr, valid_mask_arr, return_scale_shift=True, max_resolution=None):
    """Marigold/src/util/alignment.py:8-55.  numpy arrays in -> numpy arrays out (float32; scale and shift of shape
    (1,)), CUDA tensors in -> CUDA tensors out.  The aligned map is pred * scale + shift in fp32."""
    as_numpy = isinstance(pred_arr, np.ndarray)
    if as_numpy:
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
        if dev is None:
            raise ValueError("align_depth_least_square needs a CUDA device (no CPU fallback)")
        gt_arr, pred_arr, valid_mask_arr = (torch.from_numpy(np.ascontiguousarray(a)).to(dev)
                                            for a in (gt_arr, pred_arr, valid_mask_arr))
    _need_cuda(gt_arr, pred_arr, valid_mask_arr)
    ori_shape = pred_arr.shape
    gt, pred, mask = gt_arr.squeeze(), pred_arr.squeeze(), valid_mask_arr.squeeze()
    if pred.dim() != 2 or gt.shape != pred.shape or mask.shape != pred.shape:
        raise ValueError(f"align_depth_least_square: shapes {tuple(gt_arr.shape)}, {tuple(pred_arr.shape)}, "
                         f"{tuple(valid_mask_arr.shape)} do not squeeze to one [H, W]")
    gt = _float_map(gt, "gt_arr").contiguous()[None]
    pred = _float_map(pred, "pred_arr").contiguous()[None]
    mask = _bool_mask(mask, "valid_mask_arr")[None]
    ss = align_scale_shift(gt, pred, mask, max_resolution)
    aligned = torch.empty_like(pred)
    depth_metrics(pred, None, None, scale_shift=ss, aligned=aligned, metrics=False)
    aligned = aligned.reshape(ori_shape)
    scale, shift = ss[0, 0:1], ss[0, 1:2]
    if as_numpy:
        aligned, scale, shift = (t.cpu().numpy() for t in (aligned, scale, shift))
    return (aligned, scale, shift) if return_scale_shift else aligned


def _metric_inputs(output, target, valid_mask):
    _need_cuda(output, target, valid_mask)
    if output.dim() < 2 or target.shape != output.shape:
        raise ValueError(f"output {tuple(output.shape)} and target {tuple(target.shape)} must be the same [..., H, W]")
    if valid_mask is not None and valid_mask.shape != output.shape:
        raise ValueError(f"valid_mask {tuple(valid_mask.shape)} must have the shape of output {tuple(output.shape)}")
    H, W = output.shape[-2:]
    p = _float_map(output, "output").reshape(-1, H, W).contiguous()
    g = _float_map(target, "target").reshape(-1, H, W).contiguous()
    m = _bool_mask(valid_mask, "valid_mask").reshape(-1, H, W) if valid_mask is not None else None
    return p, g, m


def _metric_fn(idx, name, mask_required=False):
    def fn(output, target, valid_mask=None):
        p, g, m = _metric_inputs(output, target, valid_mask)
        return depth_metrics(p, g, m)[idx]
    if mask_required:
        def fn_req(pred, gt, valid_mask):
            return fn(pred, gt, valid_mask)
        fn_req.__name__ = name
        fn_req.__doc__ = f"Marigold/src/util/metric.py {name}: 0-d fp32 CUDA tensor (valid_mask=None: every pixel)."
        return fn_req
    fn.__name__ = name
    fn.__doc__ = f"Marigold/src/util/metric.py {name}: 0-d fp32 CUDA tensor, one kernel launch."
    return fn


metric = types.SimpleNamespace(**{name: _metric_fn(i, name, mask_required=name.startswith("delta"))
                                  for i, name in enumerate(METRICS)})


class DepthEvaluator:
    """The per-sample loop body of Marigold/eval.py:147-220 on the device: optional least-squares alignment (in depth
    or disparity space, on the `alignment_max_res` sampling grid), clipping to [min_depth, max_depth] and >= 1e-6, and
    the ten metrics.  Each `update` returns the fp32 [10] row (order METRICS) and keeps it on the device."""

    def __init__(self, min_depth, max_depth, alignment=None, alignment_max_res=None):
        if alignment not in ALIGNMENTS:
            raise ValueError(f"alignment={alignment!r}: expected one of {ALIGNMENTS}")
        self.min_depth, self.max_depth = float(min_depth), float(max_depth)
        self.alignment, self.alignment_max_res = alignment, alignment_max_res
        self._rows = []

    def update(self, depth_pred, depth_raw, valid_mask):
        _need_cuda(depth_pred, depth_raw, valid_mask)
        pred, gt, mask = depth_pred.squeeze(), depth_raw.squeeze(), valid_mask.squeeze()
        if pred.dim() != 2 or gt.shape != pred.shape or mask.shape != pred.shape:
            raise ValueError(f"depth_pred {tuple(depth_pred.shape)}, depth_raw {tuple(depth_raw.shape)} and valid_mask "
                             f"{tuple(valid_mask.shape)} must squeeze to one [H, W]")
        pred = _float_map(pred, "depth_pred").contiguous()[None]
        gt = _float_map(gt, "depth_raw").contiguous()[None]
        mask = _bool_mask(mask, "valid_mask")[None]
        disparity = self.alignment == "least_square_disparity"
        ss = None
        if self.alignment is not None:
            ss = align_scale_shift(gt, pred, mask, self.alignment_max_res, disparity=disparity)
        row = depth_metrics(pred, gt, mask, scale_shift=ss, disparity=disparity, clip=(self.min_depth, self.max_depth))
        self._rows.append(row)
        return row

    def per_sample(self):
        """float32 [N, 10] host array: the rows of eval.py's per_sample_metrics.csv (one device-to-host copy)."""
        if not self._rows:
            return np.zeros((0, len(METRICS)), dtype=np.float32)
        return torch.stack(self._rows).cpu().numpy()

    def result(self):
        """MetricTracker.result(): {name: average over samples}, summed one sample at a time in float64."""
        per = self.per_sample()
        out = {}
        for j, name in enumerate(METRICS):
            total = 0
            for v in per[:, j]:
                total += float(v)
            out[name] = total / len(per) if len(per) else float("nan")
        return out


# ------------------------------------------------------------------------------------ DSINE normals
def _normal_inputs(pred_norm, gt_norm, mask=None):
    _need_cuda(pred_norm, gt_norm, mask)
    if pred_norm.dim() != 4 or pred_norm.shape[1] != 3 or gt_norm.shape != pred_norm.shape:
        raise ValueError(f"pred_norm {tuple(pred_norm.shape)} and gt_norm {tuple(gt_norm.shape)} must both be "
                         "[B, 3, H, W]")
    B, _, H, W = pred_norm.shape
    m = None
    if mask is not None:
        if mask.shape not in ((B, 1, H, W), (B, H, W)):
            raise ValueError(f"gt_norm_mask {tuple(mask.shape)} must be [B, 1, H, W]")
        m = _bool_mask(mask, "gt_norm_mask")
    p = pred_norm if pred_norm.dtype == F32 else _float_map(pred_norm, "pred_norm")
    g = gt_norm if gt_norm.dtype == F32 else _float_map(gt_norm, "gt_norm")
    return p, g, m


def compute_normal_error(pred_norm, gt_norm):
    """DSINE/utils/utils.py:150-159: per-pixel angle in degrees, [B, 1, H, W] fp32.  pred_norm / gt_norm are
    [B, 3, H, W] views with any strides (a permuted [H, W, 3] map is read in place)."""
    p, g, _ = _normal_inputs(pred_norm, gt_norm)
    B, _, H, W = p.shape
    err = torch.empty((B, 1, H, W), dtype=F32, device=p.device)
    normal_error(p, g, None, err_map=err)
    return err


class NormalEvaluator:
    """DSINE/projects/dsine/test.py:100-130 on the device.  `update` appends the masked pixels' angles to a growing
    device buffer and accumulates their sum, sum of squares and threshold counts; `result` is compute_normal_metrics
    (utils.py:162-180) with the exact median of the pooled angles, copied to the host once."""

    def __init__(self):
        self._dev = None
        self._buf = None
        self._bound = 0            # host-known upper bound of the pooled count: sum of B*H*W over the updates

    def _state(self, dev, extra):
        if self._dev is None:
            self._dev = dev
            self._len = torch.zeros(1, dtype=torch.int64, device=dev)
            self._sums = torch.zeros(2, dtype=torch.float64, device=dev)
            self._counts = torch.zeros(6, dtype=torch.int64, device=dev)
            self._buf = torch.empty(0, dtype=F32, device=dev)
        elif dev != self._dev:
            raise ValueError(f"NormalEvaluator holds state on {self._dev}, got tensors on {dev}")
        need = self._bound + extra
        if need > self._buf.numel():
            grown = torch.empty(max(need, 2 * self._buf.numel()), dtype=F32, device=dev)
            grown[:self._bound].copy_(self._buf[:self._bound])
            self._buf = grown
        self._bound = need

    def update(self, pred_norm, gt_norm, gt_norm_mask):
        p, g, m = _normal_inputs(pred_norm, gt_norm, gt_norm_mask)
        B, _, H, W = p.shape
        self._state(p.device, B * H * W)
        normal_error(p, g, m, buf=self._buf, buf_len=self._len, sums=self._sums, counts=self._counts)

    def errors(self):
        """The pooled angles (fp32 CUDA tensor, in no particular order); reads the count back."""
        if self._buf is None:
            return torch.empty(0, dtype=F32)
        return self._buf[:int(self._len.item())]

    def result(self):
        """{mean, median, rmse, a1..a5} as compute_normal_metrics gives them; None before any update."""
        if self._buf is None:
            return None
        med = kth_smallest(self._buf, self._len, self._bound)
        host = torch.cat((self._sums, self._counts.double(), med.double())).cpu().numpy()
        s, s2, counts, median = host[0], host[1], host[2:8], np.float32(host[10])
        n = counts[0]
        out = dict(mean=s / n, median=float(median), rmse=math.sqrt(s2 / n) if n else float("nan"))
        for i in range(5):
            out[f"a{i + 1}"] = 100.0 * (counts[1 + i] / n)
        return {k: float(out[k]) for k in NORMAL_METRICS}
