"""GPU tests of the Hypersim preprocessing (b200_data_hypersim_frames in csrc/data.cu): bitwise equality with the
reference run of tests/golden/hypersim_pins.npz on every case at B = 1 and B = 8, with the oracle
(tests/hypersim_oracle.py) at other sizes and focal lengths, the tone map's double-double power against `decimal`,
preprocess_hypersim end to end into the training loader, and a run on a device that is not the current one."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import hypersim_oracle as oracle  # noqa: E402
import make_hypersim_pins as mk  # noqa: E402
from diffusion_e2e_ft_b200 import data  # noqa: E402
from diffusion_e2e_ft_b200 import lib as _lib  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PINS = dict(np.load(os.path.join(HERE, "golden", "hypersim_pins.npz")))
OUT_CASES = [c for c in mk.CASES if f"out_sha/{c}/0" in PINS]


def _run(frames, device=DEV, focal=oracle.FOCAL):
    rgb, dist, eid = (torch.from_numpy(np.stack(a)).to(device) for a in zip(*frames))
    bgr, depth = data.hypersim_frames(rgb, dist, eid, focal)
    assert bgr.dtype == torch.uint8 and depth.dtype == torch.uint16 and bgr.device == rgb.device
    return bgr.cpu().numpy(), depth.cpu().numpy()


def _run_with_stats(frames, focal=oracle.FOCAL):
    """The raw C-ABI call with its per-frame (p90, scale) readout: (bgr, depth, stats [B][2]) as numpy arrays."""
    rgb, dist, eid = (torch.from_numpy(np.stack(a)).to(DEV) for a in zip(*frames))
    B, H, W = dist.shape
    L = _lib.load()
    bgr = torch.empty((B, H, W, 3), dtype=torch.uint8, device=DEV)
    depth = torch.empty((B, H, W), dtype=torch.uint16, device=DEV)
    err = torch.empty(B, dtype=torch.int32, device=DEV)
    stats = torch.empty((B, 2), dtype=torch.float64, device=DEV)
    ws = torch.empty(L.b200_data_hypersim_workspace_bytes(B, H, W) // 8 + 1, dtype=torch.float64, device=DEV)
    half = {torch.float16: 1, torch.float32: 0}
    _lib.check(L.b200_data_hypersim_frames(rgb.data_ptr(), half[rgb.dtype], dist.data_ptr(), half[dist.dtype],
                                           eid.data_ptr(), B, H, W, focal, data._tone_map_numerator(), bgr.data_ptr(),
                                           depth.data_ptr(), err.data_ptr(), stats.data_ptr(), ws.data_ptr(),
                                           ws.numel() * 8, torch.cuda.current_stream().cuda_stream),
               "b200_data_hypersim_frames")
    return bgr.cpu().numpy(), depth.cpu().numpy(), stats.cpu().numpy()


def _same_dtype_groups():
    groups = {}
    for c in OUT_CASES:
        a = mk.case_arrays(c)
        groups.setdefault((a[0].dtype, a[1].dtype), []).append(c)
    return groups


@pytest.mark.parametrize("case", OUT_CASES)
def test_kernel_equals_the_pinned_reference_one_frame(case):
    bgr, depth = _run([mk.case_arrays(case)])
    assert mk.sha256(bgr[0]) == str(PINS[f"out_sha/{case}/0"]), case
    assert mk.sha256(depth[0]) == str(PINS[f"out_sha/{case}/1"]), case


def test_kernel_equals_the_pinned_reference_in_batches_of_eight():
    for (rt, dt), cases in _same_dtype_groups().items():
        batch = (cases * 8)[:8]                       # every case of these dtypes, at several batch positions
        bgr, depth = _run([mk.case_arrays(c) for c in batch])
        for i, c in enumerate(batch):
            assert mk.sha256(bgr[i]) == str(PINS[f"out_sha/{c}/0"]), (c, i, rt, dt)
            assert mk.sha256(depth[i]) == str(PINS[f"out_sha/{c}/1"]), (c, i, rt, dt)


def test_entity_id_zero_raises():
    assert str(PINS["entity_zero_error"]) == "AssertionError"
    frames = [mk.case_arrays("random_hdr"), mk.case_arrays("entity_zero")]
    with pytest.raises(data.HypersimEntityIdError, match=r"frame\(s\) \[1\]") as e:
        _run(frames)
    assert e.value.frames == [1]


def test_percentile_and_scale_equal_the_pinned_reference():
    """The kernel's per-frame 90th percentile is the one the script's np.percentile returned, bit for bit, and its
    scale the script's expression on it."""
    for (rt, dt), cases in _same_dtype_groups().items():
        arrays = [mk.case_arrays(c) for c in cases]
        bgr, depth, stats = _run_with_stats(arrays)
        for c, a, st in zip(cases, arrays, stats):
            assert np.array_equal(st[0], PINS[f"p90/{c}"], equal_nan=True), (c, st[0], PINS[f"p90/{c}"])
            want = oracle.tone_scale(a[0].astype(np.float64), a[2] != -1)
            assert np.array_equal(st[1], want, equal_nan=True), (c, st[1], want)
    assert np.isfinite(PINS["p90/inf_negative"]) and np.isnan(PINS["p90/nan_valid"])


def test_percentile_lerp_both_branches_equal_numpy():
    """Valid counts 1 .. 64 and a few larger ones: the virtual index is integral, below and at or above .5 past an
    integer, so both of _lerp's branches and the n = 1 case run; p90 equals np.percentile bit for bit."""
    rng = np.random.default_rng(21)
    branches = set()
    for n in list(range(1, 65)) + [101, 1000, 4097, 65537]:
        rgb = np.exp(rng.normal(-1.0, 2.0, (1, n, 3))).astype(np.float32)
        eid = np.ones((1, n), np.int32)
        extra = rng.integers(0, n + 1)               # invalid pixels mixed in
        rgb = np.concatenate([rgb, np.full((1, extra, 3), 50.0, np.float32)], 1)
        eid = np.concatenate([eid, -np.ones((1, extra), np.int32)], 1)
        dist = np.ones(eid.shape, np.float32)
        _, _, st = _run_with_stats([(rgb, dist, eid)])
        r64 = rgb.astype(np.float64)                  # the script's astype(float) first: fp64 products
        br = (0.3 * r64[..., 0] + 0.59 * r64[..., 1] + 0.11 * r64[..., 2])[eid != -1]
        assert st[0, 0] == np.percentile(br, 90) == oracle.percentile90(br), n
        assert st[0, 1] == oracle.tone_scale(rgb.astype(np.float64), eid != -1), n
        v = (n - 1) * 0.9
        branches.add("n1" if n == 1 else "int" if v == int(v) else "hi" if v - int(v) >= 0.5 else "lo")
    assert branches == {"n1", "int", "hi", "lo"}


@pytest.mark.parametrize("H,W,focal,seed", [(1, 1, 886.81, 0), (3, 5, 10.0, 1), (37, 53, 500.25, 2),
                                            (480, 640, 886.81, 3), (129, 257, 1234.5, 4)])
def test_kernel_equals_oracle_at_other_sizes(H, W, focal, seed):
    rng = np.random.default_rng(seed)
    frames = []
    for b in range(3):
        rgb = np.exp(rng.normal(-1.0, 2.0, (H, W, 3))).astype(np.float32 if b % 2 else np.float16)
        dist = (rng.random((H, W)) * 90).astype(np.float16 if b % 2 else np.float32)
        eid = rng.integers(-1, 5, (H, W)).astype(np.int32)
        eid[eid == 0] = 2
        if b == 2:
            rgb[rng.random((H, W, 3)) < 0.05] = -1.0
            if H * W >= 4:                                   # +inf and -inf radiance under a finite scale
                rgb[0, 0, 0], rgb[-1, -1, 1] = np.inf, -np.inf
        frames.append((rgb, dist, eid))
    for fr in ([frames[0], frames[2]], [frames[1]]):         # one dtype combination per launch
        bgr, depth = _run(fr, focal=focal)
        for i, (rgb, dist, eid) in enumerate(fr):
            ob, od = oracle.frame(rgb, dist, eid, focal)
            assert np.array_equal(bgr[i], ob) and np.array_equal(depth[i], od), (H, W, i)


def _debug_pow(m, force_slow):
    L = _lib.load()
    x = torch.from_numpy(np.asarray(m, np.float64)).to(DEV)
    p = torch.empty_like(x)
    lev = torch.empty(x.shape, dtype=torch.uint8, device=DEV)
    slow = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(L.b200_debug_hypersim_pow(x.data_ptr(), x.numel(), int(force_slow), p.data_ptr(), lev.data_ptr(),
                                         slow.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "b200_debug_hypersim_pow")
    return p.cpu().numpy(), lev.cpu().numpy(), int(slow.item())


def test_pow_near_level_boundaries_equals_decimal():
    m = oracle.boundary_args()
    p, lev, slow = _debug_pow(m, False)
    assert slow > 0
    want = np.array([oracle.level_decimal(v) for v in m], np.uint8)
    assert np.array_equal(lev, want)
    p_slow, lev_slow, n = _debug_pow(m, True)
    assert n == len(m)
    assert np.array_equal(p_slow, np.array([oracle.pow_decimal(v, oracle.GAMMA) for v in m]))
    assert np.array_equal(lev_slow, want)


def test_pow_forced_double_double_is_correctly_rounded():
    rng = np.random.default_rng(11)
    m = np.concatenate([rng.uniform(0, 1, 2000), np.exp(rng.uniform(-700, 700, 500)), [5e-324, 1e-310, 1.0, 2.0]])
    p, _, n = _debug_pow(m, True)
    assert n == len(m)
    assert np.array_equal(p, np.array([oracle.pow_decimal(v, oracle.GAMMA) for v in m]))


@pytest.fixture
def raw_tree(tmp_path, monkeypatch):
    raw, csv = str(tmp_path / "raw"), str(tmp_path / "split.csv")
    registry = mk.write_raw_tree(raw, csv)
    monkeypatch.setitem(sys.modules, "h5py", mk.h5py_stub(registry))
    return raw, csv, str(tmp_path / "processed")


def _check_outputs(out):
    imgs, texts = mk.read_outputs(out)
    for c in OUT_CASES:
        for k in (0, 1):
            assert mk.sha256(imgs[c][k]) == str(PINS[f"out_sha/{c}/{k}"]), (c, k)
    for name, text in texts.items():
        assert text == str(PINS[f"text/{name}"]), name


def test_preprocess_writes_the_pinned_files_and_the_loader_reads_them(raw_tree, tmp_path, monkeypatch):
    import cv2
    raw, csv, out = raw_tree
    n = data.preprocess_hypersim(csv, raw, out, batch_size=3, num_workers=0, device=DEV)
    assert n == len(OUT_CASES)
    _check_outputs(out)
    # data.Hypersim reads data/hypersim/processed/train/filename_meta_train.csv from the working directory, and the
    # normals from <root>/../normals (a separate download): give it both
    work = tmp_path / "work"
    (work / "data" / "hypersim").mkdir(parents=True)
    os.symlink(out, work / "data" / "hypersim" / "processed")
    monkeypatch.chdir(work)
    for c, scene, cam, fid, split, inc in mk.FRAMES:
        if inc and split == "train":
            d = os.path.join(out, "normals", scene, "images", f"scene_{cam}_geometry_preview")
            os.makedirs(d, exist_ok=True)
            cv2.imwrite(os.path.join(d, f"frame.{fid:04d}.normal_cam.png"), np.full((mk.H, mk.W, 3), 128, np.uint8))
    ds = data.Hypersim(os.path.join("data", "hypersim", "processed"), transform=False)
    assert len(ds) == sum(1 for f in mk.FRAMES if f[5] and f[4] == "train")
    batch = torch.utils.data.default_collate([ds[i] for i in range(2)])
    prepared = data.prepare_batch(batch, DEV)
    assert prepared["rgb"].shape == (2, 3, mk.H, mk.W) and torch.isfinite(prepared["rgb"]).all()


def test_preprocess_with_workers_and_an_existing_split(raw_tree):
    raw, csv, out = raw_tree
    assert data.preprocess_hypersim(csv, raw, out, batch_size=8, num_workers=2, device=DEV) == len(OUT_CASES)
    _check_outputs(out)
    with pytest.raises(FileExistsError):
        data.preprocess_hypersim(csv, raw, out, device=DEV)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_runs_on_a_device_that_is_not_current():
    frames = [mk.case_arrays("random_hdr")]
    with torch.cuda.device(0):
        bgr, depth = _run(frames, device="cuda:1")
    assert mk.sha256(bgr[0]) == str(PINS["out_sha/random_hdr/0"])
    assert mk.sha256(depth[0]) == str(PINS["out_sha/random_hdr/1"])
