"""CPU tests of the Virtual KITTI 2 normal generation (diffusion_e2e_ft_b200.data.vkitti_normals /
generate_vkitti_normals): the numpy oracle against the reference-run fixture tests/golden/vkitti_normals_pins.npz, the
power pin against `decimal`, the filters against cv2, the script's file walk, argument errors, the device context, and
the generator's host logic with the device step emulated."""
import ast
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import vkitti_normals_oracle as oracle  # noqa: E402
import make_vkitti_normals_pins as mk  # noqa: E402
from diffusion_e2e_ft_b200 import data  # noqa: E402

PINS = dict(np.load(os.path.join(HERE, "golden", "vkitti_normals_pins.npz")))
CASES = [str(c) for c in PINS["cases"]]


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("vkitti") / "virtual_kitti_2"
    files = mk.write_normals_tree(str(root))
    return str(root), files


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_the_pinned_reference_run(case):
    d = mk.case_depth(case)
    assert mk.sha256(d) == str(PINS[f"depth_sha/{case}"])
    got = oracle.normals_frame(d)
    if f"out/{case}" in PINS:
        assert np.array_equal(PINS[f"depth/{case}"], d)
        assert got.dtype == np.uint16 and np.array_equal(got, PINS[f"out/{case}"])
    assert mk.sha256(got) == str(PINS[f"out_sha/{case}"])


def test_fixture_covers_every_case_and_full_size_frames():
    assert set(CASES) == set(mk.SMALL + mk.FULL_CASES)
    assert {mk.case_depth(c).shape for c in mk.FULL_CASES} == {(375, 1242)}
    sky = mk.case_depth("full_road")
    assert (sky == 65535).any() and (sky == 0).any() and (mk.case_depth("zeros") == 0).any()


def test_unpinned_reference_differences_are_explained():
    """The reference's own fp32 np.power is not correctly rounded.  Where that changes an output it moves it by one
    quantisation level, except where one of get_DAG_filter's ratios lies within ~1.4e-7 of e: there the other power
    flips the threshold comparison and the whole normal moves (a few pixels of the smooth full-size frame)."""
    diff = PINS["unpinned_diff"]
    assert diff.shape[1] == 6 and len(diff) > 0
    step = np.abs(diff[:, 4] - diff[:, 5])
    assert step.min() == 1 and (step == 1).mean() > 0.5
    for case_i in np.unique(diff[:, 0]):
        c = CASES[case_i]
        rows = diff[diff[:, 0] == case_i]
        big = np.abs(rows[:, 4] - rows[:, 5]) > 1
        if big.any():
            assert np.all(oracle.threshold_margin(mk.case_depth(c))[rows[big, 1], rows[big, 2]] < 2e-7), c
        if f"out/{c}" in PINS:
            assert np.array_equal(PINS[f"out/{c}"][rows[:, 1], rows[:, 2], rows[:, 3]], rows[:, 5])


@pytest.mark.parametrize("case", ["random", "planes", "sky", "tiny_3x3", "tiny_3x4", "tiny_4x3", "tiny_5x7"])
def test_oracle_filters_equal_cv2_filter2d(case):
    cv2 = pytest.importorskip("cv2")
    Z = oracle.depth_m100(mk.case_depth(case))
    kernels = [np.array([[-1, 1, 0]]), np.array([[0, -1, 1]]), np.array([[-1], [1], [0]]), np.array([[0], [-1], [1]])]
    for got, k in zip(oracle.dag_gradients(Z), kernels):
        assert np.array_equal(got, cv2.filter2D(Z, -1, k))
    lap = np.array([[0, -1, 0], [-1, 4, -1], [0, -1, 0]])
    assert np.array_equal(oracle.mrf_laplacian(Z), np.abs(cv2.filter2D(Z, -1, lap)))


def _decimal(xs):
    return np.array([oracle.pow_e32_decimal(x) for x in xs], np.float32)


@pytest.mark.parametrize("args", ["grid", "subnormal", "random"])
def test_power_pin_is_correctly_rounded(args):
    if args == "grid":                 # integer and half-integer laplacians, 0 .. 110
        x = np.arange(0, 220.5, 1, dtype=np.float32) / np.float32(2)
    elif args == "subnormal":          # results below 2^-126 down to the last that rounds to 2^-149
        x = np.linspace(87.0, 104.5, 4000, dtype=np.float32)
    else:
        rng = np.random.default_rng(7)
        x = np.concatenate([rng.uniform(0, 110, 3000), rng.uniform(0, 2, 1000)]).astype(np.float32)
    got = oracle.pow_e32_neg(x)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), _decimal(x).view(np.uint32))
    if args == "subnormal":
        assert ((got > 0) & (got < np.finfo(np.float32).tiny)).any() and (got == 0).any()


def test_discovery_is_the_scripts_ten_variant_walk(tree):
    root, files = tree
    frames = data._VKITTIDepthFrames(root)
    got = [tuple(os.path.relpath(p, root) for p in t) for t in frames.pairs]
    want = [tuple(str(s) for s in t) for t in PINS["pairs"]]
    # the order of files within one directory is the file system's; the walk order of the directories is fixed
    assert [os.path.dirname(t[1]) for t in got] == [os.path.dirname(t[1]) for t in want]
    assert sorted(got) == sorted(want) and len(got) == len(files)
    train = data.VirtualKITTI2(root)
    assert len(train) == len(mk.FULL_CASES)


def _cuda_tensor_free(monkeypatch):
    def load(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(data._lib, "load", load)


@pytest.mark.parametrize("bad", ["dtype", "rank", "cpu", "list"])
def test_vkitti_normals_rejects_bad_inputs_before_launch(bad, monkeypatch):
    _cuda_tensor_free(monkeypatch)
    x = {"dtype": torch.zeros(1, 8, 8, dtype=torch.int32), "rank": torch.zeros(8, 8, dtype=torch.uint16),
         "cpu": torch.zeros(1, 8, 8, dtype=torch.uint16), "list": [[[0]]]}[bad]
    with pytest.raises(ValueError):
        data.vkitti_normals(x)


@pytest.mark.parametrize("bad", ["small", "fx", "v0"])
def test_vkitti_normals_rejects_bad_shape_and_intrinsics(bad, monkeypatch):
    """Checked on a stand-in that passes the device check, so the shape and intrinsics checks themselves raise."""
    _cuda_tensor_free(monkeypatch)

    class CudaLike(torch.Tensor):
        @property
        def is_cuda(self):
            return True
    x = torch.zeros(2, 2 if bad == "small" else 8, 8, dtype=torch.uint16).as_subclass(CudaLike)
    kw = {"fx": {"fx": math.inf}, "v0": {"v0": float("nan")}}.get(bad, {})
    with pytest.raises(ValueError, match="H, W >= 3" if bad == "small" else "finite"):
        data.vkitti_normals(x, **kw)
    with pytest.raises(ValueError, match="finite"):
        data.vkitti_normals(torch.zeros(1, 8, 8, dtype=torch.uint16).as_subclass(CudaLike), fx=1e39)


class _Entered(Exception):
    pass


def test_generate_enters_the_device_before_any_copy_or_launch(tree, monkeypatch):
    entered = []

    class FakeDevice:
        def __init__(self, d):
            self.d = torch.device(d)

        def __enter__(self):
            entered.append(self.d)
            raise _Entered

        def __exit__(self, *a):
            return False

    def touched(*a, **k):
        raise AssertionError("device work outside the device context")
    monkeypatch.setattr(torch.cuda, "device", FakeDevice)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(data._lib, "load", touched)
    monkeypatch.setattr(data, "_normals_on_host", touched)
    for device, want in (("cuda:1", "cuda:1"), (None, "cuda:0"), (torch.device("cuda", 2), "cuda:2")):
        with pytest.raises(_Entered):
            data.generate_vkitti_normals(tree[0], num_workers=0, device=device)
        assert entered[-1] == torch.device(want)
    with pytest.raises(ValueError):
        data.generate_vkitti_normals(tree[0], device="cpu")
    with pytest.raises(ValueError):
        data.generate_vkitti_normals(tree[0], batch_size=0, device="cuda:0")


class _NoDevice:
    def __init__(self, d):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@pytest.fixture
def emulated(monkeypatch):
    calls = []

    def normals_on_host(depth, dev):
        calls.append(tuple(depth.shape))
        return oracle.emulated_normals_on_host(depth, dev)
    monkeypatch.setattr(data, "_normals_on_host", normals_on_host)
    monkeypatch.setattr(torch.cuda, "device", _NoDevice)
    return calls


@pytest.mark.parametrize("workers", [0, 2])
def test_generate_writes_the_pinned_pngs(tmp_path, emulated, workers):
    import cv2
    root = str(tmp_path / "virtual_kitti_2")
    files = mk.write_normals_tree(root)
    n = data.generate_vkitti_normals(root, batch_size=3, num_workers=workers, device="cuda:0")
    assert n == len(files) == len(PINS["pairs"])
    # runs of equal-size frames, at most batch_size each
    assert all(b <= 3 for b, *_ in emulated) and sum(b for b, *_ in emulated) == len(files)
    for case, (_, normal) in files.items():
        img = cv2.imread(os.path.join(root, normal), cv2.IMREAD_UNCHANGED)
        assert img.dtype == np.uint16 and img.shape == mk.case_depth(case).shape + (3,)
        assert mk.sha256(img) == str(PINS[f"out_sha/{case}"]), case


def test_generate_bounds_the_frames_waiting_for_their_write(tmp_path, monkeypatch):
    """With encoding much slower than decoding, the frames computed but not yet written stay under the cap of
    2 * max(batch_size, num_workers): the generator waits on old writes instead of queueing the whole run."""
    import threading
    import time
    import cv2
    root = tmp_path / "virtual_kitti_2"
    n, batch_size, workers = 400, 8, 2
    for i in range(n):
        scene, variant = data.VKITTI_SCENES[i % 5], data.VKITTI_NORMAL_VARIANTS[(i // 5) % 10]
        rgb_dir = root / "vkitti_2.0.3_rgb" / scene / variant / "frames" / "rgb" / "Camera_0"
        depth_dir = root / "vkitti_2.0.3_depth" / scene / variant / "frames" / "depth" / "Camera_0"
        rgb_dir.mkdir(parents=True, exist_ok=True)
        depth_dir.mkdir(parents=True, exist_ok=True)
        (rgb_dir / f"rgb_{i:05d}.jpg").write_bytes(b"")
        cv2.imwrite(str(depth_dir / f"depth_{i:05d}.png"), np.full((8, 8), i, np.uint16))
    lock = threading.Lock()
    count = {"computed": 0, "written": 0, "peak": 0}

    def normals_on_host(depth, dev):
        with lock:
            count["peak"] = max(count["peak"], count["computed"] - count["written"])
            count["computed"] += depth.shape[0]
        return np.zeros(tuple(depth.shape) + (3,), np.uint16)

    def write_png(path, arr):
        time.sleep(0.01)
        with lock:
            count["written"] += 1
    monkeypatch.setattr(data, "_normals_on_host", normals_on_host)
    monkeypatch.setattr(data, "_write_png", write_png)
    monkeypatch.setattr(torch.cuda, "device", _NoDevice)
    assert data.generate_vkitti_normals(str(root), batch_size=batch_size, num_workers=workers, device="cuda:0") == n
    assert count["computed"] == count["written"] == n
    assert 0 < count["peak"] <= 2 * max(batch_size, workers), count


def test_generate_names_a_bad_depth_file(tmp_path, emulated):
    import cv2
    root = str(tmp_path / "virtual_kitti_2")
    files = mk.write_normals_tree(root)
    bad = os.path.join(root, files["planes"][0])
    cv2.imwrite(bad, np.zeros((4, 4), np.uint8))
    with pytest.raises(ValueError, match=os.path.basename(bad)):
        data.generate_vkitti_normals(root, num_workers=0, device="cuda:0")
    os.remove(bad)
    with pytest.raises(ValueError, match=os.path.basename(bad)):
        data.generate_vkitti_normals(root, num_workers=1, device="cuda:0")


def test_product_package_never_imports_the_normals_oracle():
    pkg = os.path.join(os.path.dirname(HERE), "diffusion_e2e_ft_b200")
    for name in sorted(os.listdir(pkg)):
        if name.endswith(".py"):
            for node in ast.walk(ast.parse(open(os.path.join(pkg, name)).read())):
                if isinstance(node, (ast.Import, ast.ImportFrom)):
                    mods = [a.name for a in node.names] if isinstance(node, ast.Import) else [node.module or ""]
                    assert not any(m.split(".")[0] in ("vkitti_normals_oracle", "make_vkitti_normals_pins")
                                   for m in mods), (name, mods)
