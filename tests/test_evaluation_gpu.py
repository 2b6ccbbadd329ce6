"""-m gpu: the ABI-13 evaluation kernels and evaluators against tests/golden/eval_pins.pt (the reference's own
evaluation code run on seeded inputs), an fp64 restatement, np.median on the kernel's own pooled angles, determinism,
no host synchronisation in update(), and one end-to-end pass over the tiny engine pipeline's outputs."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from diffusion_e2e_ft_b200 import evaluation as ev  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PINS = torch.load(os.path.join(HERE, "golden", "eval_pins.pt"), weights_only=False)
THRESH = (1.25, 1.25 ** 2, 1.25 ** 3)
ANGLE_TOL = 0.03                # degrees: fp32 acos next to 0 degrees resolves no better


def protocol_modes(pins):
    """Each alignment mode of the fixture's eval.py protocol with its samples: the shared inputs merged with that
    mode's per-sample results (without alignment the prediction is the metric one)."""
    P = pins["protocol"]
    return {key: dict(m, samples=[dict(x, **r, pred=x["pred" if m["alignment"] else "metric_pred"])
                                  for x, r in zip(P["inputs"], m["results"])])
            for key, m in P["modes"].items()}


PROTOCOL = protocol_modes(PINS)


def cuda(*ts):
    return [t.to(DEV) for t in ts]


def ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(int(a.view(np.int32)) - int(b.view(np.int32)))


def metrics_fp64(p, g, m):
    """metric.py's ten metrics of one [H, W] map in float64 numpy; returns the values and the delta counts."""
    p, g = p.astype(np.float64)[m], g.astype(np.float64)[m]
    n = p.size
    d, dl = p - g, np.log(p) - np.log(g)
    mx = np.maximum(p / g, g / p)
    cnt = [int((mx < t).sum()) for t in THRESH]
    vals = [np.mean(np.abs(d) / g), np.mean(d * d / g), np.sqrt(np.mean(d * d)), np.sqrt(np.mean(dl * dl)),
            np.mean(np.abs(np.log10(p) - np.log10(g)))] + [c / n for c in cnt] + [
        np.sqrt(np.mean((1 / p - 1 / g) ** 2)), np.sqrt(np.mean(dl * dl) - np.mean(dl) ** 2) * 100]
    return np.array(vals), cnt


def check_row(row, ref_row, aligned, gt, mask):
    """delta counts equal; the rest within 1e-5 of the reference's fp32 values and 1e-6 of fp64 on the same map."""
    row = row.cpu().double().numpy()
    ref_row = np.asarray(ref_row, np.float64)
    n = int(mask.sum())
    f64, cnt = metrics_fp64(aligned, gt, mask)
    for j in range(10):
        if 5 <= j <= 7:
            assert round(row[j] * n) == round(ref_row[j] * n) == cnt[j - 5], (j, row[j], ref_row[j])
        else:
            assert row[j] == pytest.approx(ref_row[j], rel=1e-5), (ev.METRICS[j], row[j], ref_row[j])
            assert row[j] == pytest.approx(f64[j], rel=1e-6, abs=1e-7), (ev.METRICS[j], row[j], f64[j])


# ------------------------------------------------------------------------------------ depth
@pytest.mark.parametrize("case", list(PINS["align"]))
def test_align_depth_least_square_vs_reference(case):
    c = PINS["align"][case]
    a, s, t = ev.align_depth_least_square(c["gt"].numpy(), c["pred"].numpy(), c["mask"].numpy(),
                                          max_resolution=c["max_res"])
    assert isinstance(a, np.ndarray) and a.dtype == np.float32 and s.shape == (1,) and t.shape == (1,)
    print("align", case, "scale ulps", ulps(s[0], c["scale"]), "shift ulps", ulps(t[0], c["shift"]))
    assert ulps(s[0], c["scale"]) <= 1 and ulps(t[0], c["shift"]) <= 1
    if s[0] == np.float32(c["scale"]) and t[0] == np.float32(c["shift"]):
        np.testing.assert_array_equal(a, c["aligned"].numpy())
    a2 = ev.align_depth_least_square(*cuda(c["gt"], c["pred"], c["mask"]), return_scale_shift=False,
                                     max_resolution=c["max_res"])
    assert a2.is_cuda and np.array_equal(a2.cpu().numpy(), a)


@pytest.mark.parametrize("mode", list(PROTOCOL))
def test_depth_evaluator_vs_reference_protocol(mode):
    P = PROTOCOL[mode]
    disparity = P["alignment"] == "least_square_disparity"
    e = ev.DepthEvaluator(0, 1, P["alignment"], P["max_res"])
    for s in P["samples"]:
        gt, pred, mask = cuda(s["gt"], s["pred"], s["mask"])
        e.min_depth, e.max_depth = s["min_depth"], s["max_depth"]
        row = e.update(pred, gt, mask)
        ss = ev.align_scale_shift(gt[None], pred[None], mask.view(torch.uint8)[None], P["max_res"], disparity) \
            if P["alignment"] else None
        aligned = torch.empty_like(pred)[None]
        ev.depth_metrics(pred[None], None, None, ss, disparity, (s["min_depth"], s["max_depth"]), aligned=aligned,
                         metrics=False)
        if ss is not None:
            assert ulps(ss[0, 0].item(), s["scale"]) <= 1 and ulps(ss[0, 1].item(), s["shift"]) <= 1
            exact = ss[0, 0].item() == np.float32(s["scale"]) and ss[0, 1].item() == np.float32(s["shift"])
        else:
            exact = True
        if exact:
            assert torch.equal(aligned[0].cpu(), s["aligned"])
        check_row(row, s["metrics"], aligned[0].cpu().numpy(), s["gt"].numpy(), s["mask"].numpy())
    res = e.result()
    for k, v in P["result"].items():
        assert res[k] == pytest.approx(v, rel=1e-5), k
    assert e.per_sample().shape == (len(P["samples"]), 10)


def test_batch_metrics_vs_reference():
    B = PINS["batch"]
    pred, gt, mask = cuda(B["pred"], B["gt"], B["mask"])
    for name in ev.METRICS:
        fn = getattr(ev.metric, name)
        got = fn(pred, gt, mask)
        assert got.is_cuda and got.dim() == 0
        assert float(got) == pytest.approx(B["values"][name]["masked"], rel=1e-5), name
        if "full" in B["values"][name]:
            assert float(fn(pred, gt)) == pytest.approx(B["values"][name]["full"], rel=1e-5), name


def test_empty_mask_gives_nan():
    g = torch.rand(1, 8, 9, device=DEV) + 0.5
    row = ev.depth_metrics(g.clone(), g, torch.zeros(1, 8, 9, dtype=torch.uint8, device=DEV))
    assert torch.isnan(row).all()


# ------------------------------------------------------------------------------------ normals
def test_normal_error_maps_and_pooled_metrics_vs_reference():
    N = PINS["normals"]
    e = ev.NormalEvaluator()
    for s, ref in zip(N["samples"], N["pooled"]):
        pred, gt, mask = cuda(s["pred"], s["gt"], s["mask"])
        err = ev.compute_normal_error(pred, gt).cpu()
        assert err.shape == s["error"].shape
        diff = (err - s["error"]).abs().max().item()
        assert diff <= ANGLE_TOL, diff
        zero = (s["pred"] == s["gt"]).all(1, keepdim=True)
        assert (err[zero] <= ANGLE_TOL).all()
        e.update(pred, gt, mask)
        r = e.result()
        for k in ("mean", "rmse"):
            assert r[k] == pytest.approx(ref[k], rel=1e-4), k
        pooled = e.errors().cpu().numpy()
        assert pooled.size == ref["count"]
        assert r["median"] == float(np.median(pooled))                         # selection: bit-exact
        assert r["median"] == pytest.approx(ref["median"], abs=ANGLE_TOL)
    # threshold counts, away from pixels whose angle lies within the tolerance of a threshold
    ref_pool = torch.cat([s["error"][s["mask"]] for s in N["samples"]]).numpy()
    got_pool = torch.cat([ev.compute_normal_error(*cuda(s["pred"], s["gt"])).cpu()[s["mask"]]
                          for s in N["samples"]]).numpy()
    for t in (5, 7.5, 11.25, 22.5, 30):
        far = np.abs(ref_pool - t) > ANGLE_TOL
        assert ((got_pool < t) == (ref_pool < t))[far].all()


def test_normal_maps_read_in_place_from_hwc():
    s = PINS["normals"]["samples"][1]
    pred, gt = cuda(s["pred"], s["gt"])
    hwc = pred.permute(0, 2, 3, 1).contiguous()
    assert torch.equal(ev.compute_normal_error(hwc.permute(0, 3, 1, 2), gt), ev.compute_normal_error(pred, gt))


def _median_check(x):
    n = torch.tensor([x.numel()], dtype=torch.int64, device=DEV)
    got = ev.kth_smallest(x, n, x.numel()).cpu().numpy()
    return got


@pytest.mark.parametrize("kind", ["n1", "n2", "odd", "even", "all_equal", "zeros", "nyuv2"])
def test_median_bit_exact_vs_numpy(kind):
    g = torch.Generator(device=DEV).manual_seed(3)
    n = dict(n1=1, n2=2, odd=100_001, even=100_000, all_equal=4096, zeros=5000, nyuv2=654 * 480 * 640)[kind]
    x = torch.rand(n, generator=g, device=DEV) * 180
    if kind == "all_equal":
        x.fill_(12.5)
    if kind == "zeros":
        x[: n // 2 + 3] = 0.0
    if kind in ("odd", "even"):
        x[::7] = x[3]                                                           # exact duplicates around the middle
    got = _median_check(x)
    host = x.cpu().numpy()
    assert got[2] == np.median(host), (kind, got, np.median(host))
    k = n // 3
    kv = ev.kth_smallest(x, torch.tensor([n], dtype=torch.int64, device=DEV), n, k).cpu().numpy()
    assert kv[0] == torch.kthvalue(x.cpu(), k + 1).values.item()


def test_median_over_two_to_the_31_values():
    """A pool just over 2^31 values: integer-valued angles, checked against exact counts (the pool is too large for a
    host copy plus np.partition to be worth it; the selection rule is the one checked against np.median above)."""
    free, _ = torch.cuda.mem_get_info()
    n = 2 ** 31 + 3
    if free < n * 4 + (4 << 30):
        pytest.skip("needs about 12 GB of free device memory")
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.empty(n, dtype=torch.float32, device=DEV)
    hist = torch.zeros(4096, dtype=torch.int64, device=DEV)
    step = 1 << 28
    for i in range(0, n, step):
        c = torch.randint(0, 4096, (min(step, n - i),), generator=g, device=DEV)
        hist += torch.bincount(c, minlength=4096)
        x[i:i + c.numel()] = c.float() / 16
        del c
    cum = torch.cumsum(hist, 0)
    k = (n - 1) // 2                                                            # n odd: the median is the k-th
    want = int(torch.searchsorted(cum, torch.tensor(k + 1, device=DEV)).item()) / 16
    got = _median_check(x)
    assert float(got[2]) == want and float(got[0]) == want
    del x


# ------------------------------------------------------------------------------------ determinism, no host sync
def _full_run():
    P = PROTOCOL["least_square@20"]
    d = ev.DepthEvaluator(1e-3, 80.0, "least_square", 40)
    for s in P["samples"]:
        d.update(*cuda(s["pred"], s["gt"], s["mask"]))
    n = ev.NormalEvaluator()
    for s in PINS["normals"]["samples"]:
        n.update(*cuda(s["pred"], s["gt"], s["mask"]))
    return d.per_sample(), n.result(), torch.cat((n._sums.view(torch.int64), n._counts)).cpu()


def test_two_runs_are_bitwise_equal():
    a, b = _full_run(), _full_run()
    assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1] and torch.equal(a[2], b[2])


def test_update_does_not_sync_the_host():
    s = PROTOCOL["least_square_disparity"]["samples"][0]
    t = PINS["normals"]["samples"][1]
    dp, dg, dm = cuda(s["pred"], s["gt"], s["mask"])
    npred, ngt, nm = cuda(t["pred"], t["gt"], t["mask"])
    d = ev.DepthEvaluator(1e-3, 80.0, "least_square_disparity", 32)
    n = ev.NormalEvaluator()
    d.update(dp, dg, dm)                         # library load outside the checked region
    n.update(npred, ngt, nm)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            d.update(dp, dg, dm)
            n.update(npred, ngt, nm)             # also grows the pooled buffer
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(d.per_sample()) == 4 and n.errors().numel() == 4 * int(t["mask"].sum())


# ------------------------------------------------------------------------------------ end to end
def test_end_to_end_tiny_pipeline_outputs():
    """The tiny Marigold pipeline's depth_np / normal_np on a seeded image go through the evaluators and match the
    reference's evaluation arithmetic run on the same arrays on the CPU (numpy lstsq, fp32 alignment and clipping,
    torch.cosine_similarity, np.median)."""
    import engine_checks as E
    import make_golden as MG
    from diffusion_e2e_ft_b200 import DDIMScheduler, MarigoldPipeline
    unet_ref, vae_ref = MG.build_tiny()
    unet, vae = E.engine_from_oracle(unet_ref, vae_ref, DEV)
    pipe = MarigoldPipeline(unet, vae, DDIMScheduler(), empty_text_embed=MG.inputs(5, 1, 2, 128, scale=0.5).to(DEV))
    img = (torch.rand(3, 60, 100, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)
    depth = pipe(img, denoising_steps=1, ensemble_size=1, processing_res=80, noise="zeros").depth_np
    normal = pipe(img, denoising_steps=1, ensemble_size=1, processing_res=80, noise="zeros", normals=True).normal_np
    rs = np.random.RandomState(0)
    gt = (0.5 + 9.5 * rs.rand(*depth.shape)).astype(np.float32)
    mask = rs.rand(*depth.shape) > 0.1

    # depth: host lstsq + fp32 arithmetic + torch metrics, as Marigold/eval.py:172-220 runs them
    A = np.stack([depth[mask], np.ones(int(mask.sum()), np.float32)], 1)
    scale, shift = np.linalg.lstsq(A, gt[mask].reshape(-1, 1), rcond=None)[0]
    want_pred = np.clip(np.clip(depth * scale + shift, 0.5, 10.0), 1e-6, None)
    d = ev.DepthEvaluator(0.5, 10.0, "least_square")
    row = d.update(*cuda(torch.from_numpy(depth), torch.from_numpy(gt), torch.from_numpy(mask)))
    check_row(row, metrics_fp64(want_pred, gt, mask)[0], want_pred, gt, mask)

    # normals: torch.cosine_similarity on the CPU + the pooled statistics of compute_normal_metrics
    gt_n = rs.randn(3, *normal.shape[1:]).astype(np.float32)
    gt_n /= np.linalg.norm(gt_n, axis=0, keepdims=True)
    nmask = rs.rand(1, 1, *normal.shape[1:]) > 0.2
    p_t, g_t = torch.from_numpy(normal)[None], torch.from_numpy(gt_n)[None]
    want_err = torch.acos(torch.clamp(torch.cosine_similarity(p_t, g_t, dim=1), -1, 1)) * 180.0 / np.pi
    pooled = want_err.unsqueeze(1)[torch.from_numpy(nmask)].numpy()
    n = ev.NormalEvaluator()
    n.update(*cuda(p_t, g_t, torch.from_numpy(nmask)))
    r = n.result()
    assert r["mean"] == pytest.approx(float(np.mean(pooled.astype(np.float64))), rel=1e-4)
    assert r["rmse"] == pytest.approx(float(np.sqrt(np.mean(pooled.astype(np.float64) ** 2))), rel=1e-4)
    assert r["median"] == pytest.approx(float(np.median(pooled)), abs=ANGLE_TOL)
    assert r["median"] == float(np.median(n.errors().cpu().numpy()))
