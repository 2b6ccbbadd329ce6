"""Evaluation on the CPU: plain-torch / numpy restatements of the four ABI-13 evaluation kernels
(include/b200_e2eft.h) reproduce tests/golden/eval_pins.pt (made by running the reference's evaluation code), and
the evaluators' host logic runs on those restatements: bookkeeping, MetricTracker averaging, the even / odd median,
and argument errors raised before any launch."""
import os

import numpy as np
import pytest
import torch

from diffusion_e2e_ft_b200 import evaluation as ev, lib

PINS = torch.load(os.path.join(os.path.dirname(__file__), "golden", "eval_pins.pt"), weights_only=False)
THRESH = (1.25, 1.25 ** 2, 1.25 ** 3)


def protocol_modes(pins):
    """Each alignment mode of the fixture's eval.py protocol with its samples: the shared inputs merged with that
    mode's per-sample results (without alignment the prediction is the metric one)."""
    P = pins["protocol"]
    return {key: dict(m, samples=[dict(x, **r, pred=x["pred" if m["alignment"] else "metric_pred"])
                                  for x, r in zip(P["inputs"], m["results"])])
            for key, m in P["modes"].items()}


PROTOCOL = protocol_modes(PINS)


# ---- the kernel contracts, restated
def align_scale_shift(gt, pred, mask, max_resolution=None, disparity=False):
    """np.linalg.lstsq of [p 1] x = g over the mask on the sampled columns, computed in fp64, rounded to fp32."""
    B, H, W = pred.shape
    ow, col_scale = ev.sampling_columns(H, W, max_resolution)
    cols = np.minimum(np.floor(np.arange(ow, dtype=np.float32) * np.float32(col_scale)).astype(np.int64), W - 1)
    out = torch.empty((B, 2), dtype=torch.float32)
    for b in range(B):
        g, p, m = gt[b][:, cols].numpy(), pred[b][:, cols].numpy(), mask[b][:, cols].numpy().astype(bool)
        if disparity:
            m = m & (g > 0) & (p > 0)
            g = np.where(g > 0, np.float32(1.0) / np.where(g > 0, g, 1), 0).astype(np.float32)
        A = np.stack([p[m], np.ones(int(m.sum()), np.float32)], 1).astype(np.float64)
        x = np.linalg.lstsq(A, g[m].astype(np.float64), rcond=None)[0] if m.any() else np.zeros(2)
        out[b] = torch.from_numpy(x.astype(np.float32))
    return out


def map_prediction(pred, scale_shift=None, disparity=False, clip=None):
    p = pred.clone()
    if scale_shift is not None:
        p = p * scale_shift[:, 0, None, None] + scale_shift[:, 1, None, None]
    if disparity:
        p = torch.where(p < 1e-3, torch.tensor(1e-3, dtype=torch.float32), p)
        p = torch.where(p > 0, 1.0 / p, torch.zeros_like(p))
    if clip is not None:
        lo, hi = (torch.tensor(v, dtype=torch.float32) for v in clip)
        p = torch.where(p < lo, lo, p)
        p = torch.where(p > hi, hi, p)
        p = torch.where(p < 1e-6, torch.tensor(1e-6, dtype=torch.float32), p)
    return p


def depth_metrics(pred, gt, mask, scale_shift=None, disparity=False, clip=None, aligned=None, metrics=True):
    """fp32 per-pixel terms, fp64 per-sample sums, metric.py's batch semantics."""
    p = map_prediction(pred, scale_shift, disparity, clip)
    if aligned is not None:
        aligned.copy_(p)
    if not metrics:
        return None
    g = gt
    m = mask.bool() if mask is not None else torch.ones_like(p, dtype=torch.bool)

    def s(x):
        return torch.where(m, x.double(), torch.zeros((), dtype=torch.float64)).sum((-1, -2))
    n = m.sum((-1, -2)).double()
    d = p - g
    dl = torch.log(p) - torch.log(g)
    l10 = (torch.log10(p) - torch.log10(g)).abs()
    r1, r2 = p / g, g / p
    di = 1.0 / p - 1.0 / g
    row = [(s(d.abs() / g) / n).mean(), (s(d.abs() * d.abs() / g) / n).mean(), (s(d * d) / n).sqrt().mean(),
           (s(dl * dl) / n).sqrt().mean(), s(l10).sum() / n.sum()]
    row += [(s(((r1 < t) & (r2 < t)).float()) / n).mean() for t in THRESH]
    row += [(s(di * di) / n).sqrt().mean(), (s(dl * dl) / n - s(dl) ** 2 / n ** 2).mean().sqrt() * 100]
    return torch.stack(row).float()


def normal_error(pred, gt, mask=None, err_map=None, buf=None, buf_len=None, sums=None, counts=None):
    e = torch.acos(torch.clamp(torch.cosine_similarity(pred, gt, dim=1), -1.0, 1.0)) * 180.0 / np.pi
    if err_map is not None:
        err_map.copy_(e.reshape(err_map.shape))
    sel = e[mask.bool().reshape(e.shape)] if mask is not None else e.reshape(-1)
    if buf is not None:
        n0 = int(buf_len[0])
        buf[n0:n0 + sel.numel()] = sel
        buf_len += sel.numel()
    if sums is not None:
        sums += torch.stack([sel.double().sum(), (sel.double() ** 2).sum()])
        counts += torch.tensor([sel.numel()] + [int((sel < t).sum()) for t in (5, 7.5, 11.25, 22.5, 30)])


def kth_smallest(x, n, n_max, k=-1):
    n = int(n[0])
    assert n <= n_max
    if n == 0 or k >= n:
        return torch.full((3,), float("nan"))
    v = x[:n].sort().values
    kk = (n - 1) // 2 if k < 0 else k
    a, b = v[kk], v[min(kk + 1, n - 1)]
    return torch.stack([a, b, (a + b) / 2 if k < 0 and n % 2 == 0 else a])


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(ev, "_need_cuda", lambda *a: None)
    for name, fn in dict(align_scale_shift=align_scale_shift, depth_metrics=depth_metrics, normal_error=normal_error,
                         kth_smallest=kth_smallest).items():
        monkeypatch.setattr(ev, name, fn)


@pytest.fixture
def no_launch(monkeypatch):
    def load(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(lib, "load", load)


def batch1(*ts):
    return [t[None] for t in ts]


# ---- the restatements reproduce the reference
def test_sampling_columns_match_torch_upsample_on_the_reference_input():
    """alignment.py:25-32 hands nn.Upsample a [1, H, W] tensor: a 1-D nearest interpolation along W with the source
    step 1/s, which is not W / OW (the size-based grid of b200_resize_nearest)."""
    for (H, W), max_res in (((4032, 6048), 1024), ((300, 200), 70), ((126, 189), 32), ((480, 640), 1024),
                            ((1242, 375), 512)):
        ow, col_scale = ev.sampling_columns(H, W, max_res)
        s = float(np.min(max_res / np.array((H, W))))
        ramp = torch.arange(W, dtype=torch.float32).expand(1, 3, W)
        up = torch.nn.Upsample(scale_factor=s, mode="nearest")(ramp) if s < 1 else ramp
        cols = np.minimum(np.floor(np.arange(ow, dtype=np.float32) * np.float32(col_scale)).astype(np.int64), W - 1)
        assert up.shape[-1] == ow and np.array_equal(up[0, 0].numpy().astype(np.int64), cols), (H, W)
    ow, col_scale = ev.sampling_columns(300, 200, 70)
    scale_grid = np.floor(np.arange(ow, dtype=np.float32) * np.float32(col_scale)).astype(np.int64)
    size_grid = np.floor(np.arange(ow) * (200 / ow)).astype(np.int64)
    assert int((scale_grid != size_grid).sum()) > ow // 2


@pytest.mark.parametrize("case", list(PINS["align"]))
def test_align_restatement_reproduces_the_reference(case):
    c = PINS["align"][case]
    gt, pred, mask = batch1(c["gt"], c["pred"], c["mask"])
    ss = align_scale_shift(gt, pred, mask.to(torch.uint8), c["max_res"])
    assert float(ss[0, 0]) == c["scale"] and float(ss[0, 1]) == c["shift"]
    aligned = torch.empty_like(pred)
    depth_metrics(pred, None, None, ss, aligned=aligned, metrics=False)
    assert torch.equal(aligned[0], c["aligned"])


@pytest.mark.parametrize("mode", list(PROTOCOL))
def test_protocol_restatement_reproduces_the_reference(mode):
    P = PROTOCOL[mode]
    disparity = P["alignment"] == "least_square_disparity"
    for s in P["samples"]:
        gt, pred, mask = batch1(s["gt"], s["pred"], s["mask"])
        ss = align_scale_shift(gt, pred, mask, P["max_res"], disparity) if P["alignment"] else None
        if ss is not None:
            assert float(ss[0, 0]) == s["scale"] and float(ss[0, 1]) == s["shift"]
        aligned = torch.empty_like(pred)
        row = depth_metrics(pred, gt, mask, ss, disparity, (s["min_depth"], s["max_depth"]), aligned=aligned)
        assert torch.equal(aligned[0], s["aligned"])
        torch.testing.assert_close(row.double(), s["metrics"], rtol=1e-5, atol=0)


def test_batch_metric_restatement_reproduces_the_reference():
    B = PINS["batch"]
    for i, name in enumerate(ev.METRICS):
        for kind, m in (("masked", B["mask"]), ("full", None)):
            if kind in B["values"][name]:
                got = float(depth_metrics(B["pred"], B["gt"], m)[i])
                assert got == pytest.approx(B["values"][name][kind], rel=1e-5), (name, kind)


def test_normal_restatements_reproduce_the_reference():
    N = PINS["normals"]
    pooled = []
    for s, ref in zip(N["samples"], N["pooled"]):
        err = torch.empty_like(s["error"])
        normal_error(s["pred"], s["gt"], None, err_map=err)
        assert torch.equal(err, s["error"])
        pooled.append(err[s["mask"]])
        v = torch.cat(pooled)
        n = torch.tensor([v.numel()])
        assert float(kth_smallest(v, n, v.numel())[2]) == ref["median"] == np.median(v.numpy())


# ---- the evaluators' host logic on the restatements
@pytest.mark.parametrize("mode", list(PROTOCOL))
def test_depth_evaluator_rows_and_tracker_average(emulated, mode):
    P = PROTOCOL[mode]
    e = ev.DepthEvaluator(P["samples"][0]["min_depth"], P["samples"][0]["max_depth"], P["alignment"], P["max_res"])
    rows = []
    for s in P["samples"]:
        e.min_depth, e.max_depth = s["min_depth"], s["max_depth"]
        rows.append(e.update(s["pred"][None, None], s["gt"], s["mask"][None]))
        torch.testing.assert_close(rows[-1].double(), s["metrics"], rtol=1e-5, atol=0)
    per = e.per_sample()
    assert per.shape == (len(P["samples"]), 10) and per.dtype == np.float32
    assert np.array_equal(per, torch.stack(rows).numpy())
    res = e.result()
    assert list(res) == list(ev.METRICS)
    for k, v in P["result"].items():
        assert res[k] == pytest.approx(v, rel=1e-5), k


def test_metric_namespace_matches_eval_py_loop(emulated):
    B = PINS["batch"]
    for i, name in enumerate(ev.METRICS):
        fn = getattr(ev.metric, name)
        assert fn.__name__ == name
        assert float(fn(B["pred"], B["gt"], B["mask"])) == pytest.approx(B["values"][name]["masked"], rel=1e-5)
        if "full" in B["values"][name]:
            assert float(fn(B["pred"], B["gt"])) == pytest.approx(B["values"][name]["full"], rel=1e-5)


def test_align_depth_least_square_tensor_convention(emulated):
    c = PINS["align"]["portrait"]
    a, s, t = ev.align_depth_least_square(c["gt"][None], c["pred"][None], c["mask"][None],
                                          max_resolution=c["max_res"])
    assert a.shape == (1, *c["pred"].shape) and s.shape == (1,) and t.shape == (1,)
    assert float(s) == c["scale"] and float(t) == c["shift"] and torch.equal(a[0], c["aligned"])
    assert torch.equal(ev.align_depth_least_square(c["gt"], c["pred"], c["mask"], False, c["max_res"]), c["aligned"])


def test_normal_evaluator_pooling_and_median(emulated):
    N = PINS["normals"]
    e = ev.NormalEvaluator()
    assert e.result() is None
    for s, ref in zip(N["samples"], N["pooled"]):
        e.update(s["pred"], s["gt"], s["mask"])
        r = e.result()
        assert list(r) == list(ev.NORMAL_METRICS)
        assert r["median"] == ref["median"]
        for k in ("mean", "rmse"):
            assert r[k] == pytest.approx(ref[k], rel=1e-4)
        for k in ("a1", "a2", "a3", "a4", "a5"):
            assert r[k] == pytest.approx(ref[k], rel=1e-12)
        assert e.errors().numel() == ref["count"] and e._bound >= ref["count"]
    # a [H, W, 3] map read through a permuted view (torch's CPU cosine_similarity rounds by layout)
    e2 = ev.NormalEvaluator()
    for s in N["samples"]:
        hwc = s["pred"].permute(0, 2, 3, 1).contiguous()
        e2.update(hwc.permute(0, 3, 1, 2), s["gt"], s["mask"])
    r2, r = e2.result(), e.result()
    assert r2 == pytest.approx(r, rel=1e-6)


@pytest.mark.parametrize("vals", [[3.0], [2.0, 1.0], [5.0, 1.0, 3.0], [4.0, 1.0, 3.0, 2.0], [7.0] * 6,
                                  [0.0, 0.0, 1.5, 0.0], [0.1, 0.2]])
def test_median_even_and_odd(vals):
    x = torch.tensor(vals, dtype=torch.float32)
    got = kth_smallest(x, torch.tensor([len(vals)]), len(vals))
    assert float(got[2]) == float(np.median(x.numpy()))
    k = len(vals) // 3
    assert float(kth_smallest(x, torch.tensor([len(vals)]), len(vals), k)[0]) == float(torch.kthvalue(x, k + 1).values)


# ---- argument errors before any launch
def test_argument_errors_raise_before_launch(no_launch):
    with pytest.raises(ValueError, match="alignment"):
        ev.DepthEvaluator(0.1, 10, alignment="median")
    with pytest.raises(ValueError, match="no CPU fallback"):
        ev.DepthEvaluator(0.1, 10).update(torch.ones(4, 4), torch.ones(4, 4), torch.ones(4, 4, dtype=torch.bool))
    with pytest.raises(ValueError, match="no CPU fallback"):
        ev.NormalEvaluator().update(torch.ones(1, 3, 4, 4), torch.ones(1, 3, 4, 4), torch.ones(1, 1, 4, 4) > 0)
    with pytest.raises(ValueError, match="no CPU fallback"):
        ev.metric.rmse_linear(torch.ones(4, 4), torch.ones(4, 4))


def test_shape_and_dtype_errors_raise_before_launch(no_launch, monkeypatch):
    monkeypatch.setattr(ev, "_need_cuda", lambda *a: None)
    m = torch.ones(4, 5, dtype=torch.bool)
    d = ev.DepthEvaluator(0.1, 10, "least_square")
    with pytest.raises(ValueError, match="squeeze"):
        d.update(torch.ones(4, 5), torch.ones(4, 6), m)
    with pytest.raises(ValueError, match="bool"):
        d.update(torch.ones(4, 5), torch.ones(4, 5), torch.ones(4, 5))
    with pytest.raises(ValueError, match="floating"):
        d.update(torch.ones(4, 5, dtype=torch.int32), torch.ones(4, 5), m)
    with pytest.raises(ValueError, match="same"):
        ev.metric.abs_relative_difference(torch.ones(2, 4, 5), torch.ones(4, 5))
    with pytest.raises(ValueError, match="valid_mask"):
        ev.metric.delta1_acc(torch.ones(4, 5), torch.ones(4, 5), torch.ones(4, 4, dtype=torch.bool))
    n = ev.NormalEvaluator()
    with pytest.raises(ValueError, match=r"\[B, 3, H, W\]"):
        n.update(torch.ones(1, 4, 4, 4), torch.ones(1, 4, 4, 4), torch.ones(1, 1, 4, 4) > 0)
    with pytest.raises(ValueError, match="gt_norm_mask"):
        n.update(torch.ones(1, 3, 4, 4), torch.ones(1, 3, 4, 4), torch.ones(1, 1, 4, 5) > 0)
    with pytest.raises(ValueError, match="squeeze"):
        ev.align_depth_least_square(torch.ones(4, 5), torch.ones(3, 4, 5), m)
    with pytest.raises(ValueError, match="no column"):
        ev.sampling_columns(4000, 3, 2)
