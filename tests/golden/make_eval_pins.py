"""Generate tests/golden/eval_pins.pt by RUNNING THE REFERENCE'S OWN EVALUATION CODE (imported by path from a checkout of
VisualComputingInstitute/diffusion-e2e-ft, read-only) on seeded inputs:

    Marigold/src/util/alignment.py   align_depth_least_square, depth2disparity, disparity2depth
    Marigold/src/util/metric.py      the ten depth metrics (MetricTracker's averaging is restated below)
    DSINE/utils/utils.py             compute_normal_error, compute_normal_metrics

Marigold/eval.py imports omegaconf and its dataset readers, so its per-sample loop body (:172-220) cannot be imported:
`eval_one` below restates those lines, the disparity branch (:182-202) included, calling the reference functions.
The pooled normal errors are the torch.cat accumulation of DSINE/projects/dsine/test.py:105-113.

    python tests/golden/make_eval_pins.py <path to the reference checkout>
"""
import importlib.util
import os
import sys

import numpy as np
import torch

REF = sys.argv[1] if len(sys.argv) > 1 else ""
HERE = os.path.dirname(os.path.abspath(__file__))
EVAL_METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10",
                "delta1_acc", "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")          # Marigold/eval.py:46-57


def load_ref(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def depth_case(seed, H, W, lo, hi, p_invalid=0.15):
    """gt in [lo, hi] with invalid pixels set to 0, an affine-invariant prediction in about [0, 1], the valid mask."""
    rs = np.random.RandomState(seed)
    gt = (lo + (hi - lo) * rs.rand(H, W) ** 1.5).astype(np.float32)
    pred = ((gt - lo) / (hi - lo) * 0.9 + 0.05 + 0.03 * rs.randn(H, W)).astype(np.float32)
    mask = rs.rand(H, W) > p_invalid
    gt[~mask & (rs.rand(H, W) > 0.5)] = 0.0
    return gt, pred, mask


class Tracker:
    """MetricTracker of Marigold/src/util/metric.py:10-31 without its pandas frame (pandas >= 3 makes the frame's
    column arrays read-only, so its reset() raises): total += value * n, counts += n, average = total / counts."""

    def __init__(self, keys):
        self.total, self.counts = dict.fromkeys(keys, 0), dict.fromkeys(keys, 0)

    def update(self, key, value, n=1):
        self.total[key] += value * n
        self.counts[key] += n

    def result(self):
        return {k: self.total[k] / self.counts[k] for k in self.total}


def eval_one(align, metric, alignment, gt, pred, mask, min_depth, max_depth, max_res):
    """Marigold/eval.py:172-220 for one sample (depth_raw = gt, depth_pred = pred, valid_mask = mask)."""
    depth_pred = pred
    if "least_square" == alignment:
        depth_pred, scale, shift = align.align_depth_least_square(
            gt_arr=gt, pred_arr=depth_pred, valid_mask_arr=mask, return_scale_shift=True, max_resolution=max_res)
    elif "least_square_disparity" == alignment:
        gt_disparity, gt_non_neg_mask = align.depth2disparity(depth=gt, return_mask=True)
        pred_non_neg_mask = depth_pred > 0
        valid_nonnegative_mask = mask & gt_non_neg_mask & pred_non_neg_mask
        disparity_pred, scale, shift = align.align_depth_least_square(
            gt_arr=gt_disparity, pred_arr=depth_pred, valid_mask_arr=valid_nonnegative_mask, return_scale_shift=True,
            max_resolution=max_res)
        disparity_pred = np.clip(disparity_pred, a_min=1e-3, a_max=None)
        depth_pred = align.disparity2depth(disparity_pred)
    else:
        scale = shift = np.zeros(1, np.float32)
    depth_pred = np.clip(depth_pred, a_min=min_depth, a_max=max_depth)
    depth_pred = np.clip(depth_pred, a_min=1e-6, a_max=None)
    depth_pred_ts = torch.from_numpy(depth_pred)
    row = [getattr(metric, m)(depth_pred_ts, torch.from_numpy(gt), torch.from_numpy(mask)).item() for m in EVAL_METRICS]
    return dict(aligned=torch.from_numpy(depth_pred.copy()), metrics=torch.tensor(row, dtype=torch.float64),
                scale=float(np.asarray(scale).reshape(-1)[0]), shift=float(np.asarray(shift).reshape(-1)[0]))


def main():
    torch.set_num_threads(4)
    align = load_ref("Marigold/src/util/alignment.py", "ref_alignment")
    metric = load_ref("Marigold/src/util/metric.py", "ref_metric")
    dsine = load_ref("DSINE/utils/utils.py", "ref_dsine_utils")
    out = {}

    # ---- least-squares alignment: full grid, a non-square max_resolution grid whose source step 1/s differs from
    # W/OW, and the ETH3D aspect ratio (4032 x 6048 / 64) at max_res 16.  The maps are small: the fixture is committed.
    al = {}
    for name, (seed, H, W, lo, hi, max_res) in dict(full=(1, 32, 40, 0.5, 10.0, None),
                                                    portrait=(2, 90, 60, 0.5, 10.0, 20),
                                                    eth3d=(3, 63, 94, 0.1, 60.0, 16)).items():
        gt, pred, mask = depth_case(seed, H, W, lo, hi)
        a, s, t = align.align_depth_least_square(gt, pred, mask, return_scale_shift=True, max_resolution=max_res)
        al[name] = dict(gt=torch.from_numpy(gt), pred=torch.from_numpy(pred), mask=torch.from_numpy(mask),
                        max_res=max_res, aligned=torch.from_numpy(np.asarray(a, np.float32)),
                        scale=float(s.reshape(-1)[0]), shift=float(t.reshape(-1)[0]))
    gt, pred, mask = depth_case(4, 20, 28, 0.5, 10.0)
    const = np.full_like(pred, 0.37)
    for name, (p, m) in dict(constant=(const, mask), empty=(pred, np.zeros_like(mask))).items():
        a, s, t = align.align_depth_least_square(gt, p, m, return_scale_shift=True)
        al[name] = dict(gt=torch.from_numpy(gt), pred=torch.from_numpy(p), mask=torch.from_numpy(m), max_res=None,
                        aligned=torch.from_numpy(np.asarray(a, np.float32)), scale=float(s.reshape(-1)[0]),
                        shift=float(t.reshape(-1)[0]))
    out["align"] = al

    # ---- the per-sample protocol (eval.py:172-220) and MetricTracker averages, per alignment mode.  The inputs are
    # stored once; each mode stores its per-sample results in input order.  Without alignment the prediction is an
    # already metric one (`metric_pred`).
    inputs = []
    for seed, H, W, lo, hi in [(11, 24, 32, 1e-3, 10.0), (12, 24, 32, 1e-5, 80.0), (13, 30, 22, 0.5, 3.0),
                               (14, 26, 35, 0.2, 30.0)]:
        gt, pred, mask = depth_case(seed, H, W, lo, hi)
        inputs.append(dict(gt=torch.from_numpy(gt), pred=torch.from_numpy(pred), mask=torch.from_numpy(mask),
                           metric_pred=torch.from_numpy((pred * (hi - lo) + lo).astype(np.float32)), min_depth=lo,
                           max_depth=hi))
    modes = {}
    for alignment, max_res in (("least_square", None), ("least_square", 20), ("least_square_disparity", None),
                               (None, None)):
        results = []
        tracker = Tracker(EVAL_METRICS)
        for x in inputs:
            pred = x["pred" if alignment else "metric_pred"].numpy()
            r = eval_one(align, metric, alignment, x["gt"].numpy(), pred, x["mask"].numpy(), x["min_depth"],
                         x["max_depth"], max_res)
            for m, v in zip(EVAL_METRICS, r["metrics"].tolist()):
                tracker.update(m, v)
            results.append(r)
        key = f"{alignment}" + (f"@{max_res}" if max_res else "")
        modes[key] = dict(alignment=alignment, max_res=max_res, results=results,
                          result={k: float(v) for k, v in tracker.result().items()})
    out["protocol"] = dict(inputs=inputs, modes=modes)

    # ---- batch-2 metrics with and without a mask (metric.py batch semantics); the delta metrics need the mask
    g2, p2, m2 = zip(*(depth_case(s, 24, 30, 0.5, 10.0) for s in (21, 22)))
    gt2 = torch.from_numpy(np.stack(g2)).clamp_min(0.5)
    pr2 = torch.from_numpy(np.stack(p2)) * 9.5 + 0.5
    vm2 = torch.from_numpy(np.stack(m2))
    vals = {}
    for fn in EVAL_METRICS:
        vals[fn] = dict(masked=float(getattr(metric, fn)(pr2.clone(), gt2.clone(), vm2.clone())))
        if not fn.startswith("delta"):
            vals[fn]["full"] = float(getattr(metric, fn)(pr2.clone(), gt2.clone()))
    out["batch"] = dict(pred=pr2, gt=gt2, mask=vm2, values=vals)

    # ---- DSINE normal errors: maps and the pooled metrics of test.py:100-130
    rs = np.random.RandomState(31)

    def unit(shape):
        v = rs.randn(*shape).astype(np.float32)
        return v / np.linalg.norm(v, axis=1, keepdims=True)

    samples = []
    shapes = [(1, 24, 32), (2, 17, 23), (1, 30, 20)]
    for i, (B, H, W) in enumerate(shapes):
        gt_n = unit((B, 3, H, W))
        pred_n = (gt_n + 0.25 * rs.randn(B, 3, H, W).astype(np.float32)).astype(np.float32)
        mask = rs.rand(B, 1, H, W) > 0.2
        pred_n[:, :, :3, :4] = gt_n[:, :, :3, :4]                  # zero-angle pixels (pred == gt)
        pred_n[:, :, 5, :6] = 0.0                                  # zero-vector predictions: 90 degrees
        pred_n[:, :, 7, 1:8] = pred_n[:, :, 7, :1]                 # exact duplicate angles
        gt_n[:, :, 7, 1:8] = gt_n[:, :, 7, :1]
        samples.append(dict(pred=torch.from_numpy(pred_n), gt=torch.from_numpy(gt_n), mask=torch.from_numpy(mask)))
    pooled, prefix = None, []
    for s in samples:
        err = dsine.compute_normal_error(s["pred"], s["gt"])
        s["error"] = err
        sel = err[s["mask"]]
        pooled = sel if pooled is None else torch.cat((pooled, sel), dim=0)
        m = dsine.compute_normal_metrics(pooled)
        prefix.append(dict(count=int(pooled.shape[0]), **{k: float(v) for k, v in m.items()}))
    out["normals"] = dict(samples=samples, pooled=prefix)
    assert len({p["count"] % 2 for p in prefix}) == 2, "want both odd and even pooled counts"

    path = os.path.join(HERE, "eval_pins.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("usage: make_eval_pins.py <path to the diffusion-e2e-ft reference checkout>")
    main()
