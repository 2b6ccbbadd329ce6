"""CPU tests of the Hypersim preprocessing (diffusion_e2e_ft_b200.data.hypersim_frames / preprocess_hypersim): the numpy
oracle against the reference-run fixture tests/golden/hypersim_pins.npz, the power pin against `decimal`, the oracle's
pieces against NumPy's own calls, the driver's host logic with the device step emulated, argument errors, the device
context and the C ABI table."""
import os
import re
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

PINS = dict(np.load(os.path.join(HERE, "golden", "hypersim_pins.npz")))
OUT_CASES = [c for c in mk.CASES if f"out_sha/{c}/0" in PINS]


@pytest.mark.parametrize("case", OUT_CASES)
def test_oracle_matches_the_pinned_reference_run(case):
    arrays = mk.case_arrays(case)
    assert mk.sha256(np.concatenate([a.reshape(-1).view(np.uint8) for a in arrays])) == str(PINS[f"in_sha/{case}"])
    bgr, depth = oracle.frame(*arrays)
    assert bgr.dtype == np.uint8 and depth.dtype == np.uint16
    assert mk.sha256(bgr) == str(PINS[f"out_sha/{case}/0"]) and mk.sha256(depth) == str(PINS[f"out_sha/{case}/1"])


@pytest.mark.parametrize("case", OUT_CASES)
def test_oracle_percentile_equals_the_reference_runs(case):
    rgb, _, eid = mk.case_arrays(case)
    valid = eid != -1
    with np.errstate(invalid="ignore", over="ignore"):
        rgb = rgb.astype(np.float64)
        br = 0.3 * rgb[..., 0] + 0.59 * rgb[..., 1] + 0.11 * rgb[..., 2]
    got = oracle.percentile90(br[valid]) if valid.any() else np.nan
    assert np.array_equal(got, PINS[f"p90/{case}"], equal_nan=True), (case, got, PINS[f"p90/{case}"])


def test_inf_case_keeps_a_finite_scale():
    """+inf and -inf radiance sit in different pixels, so no brightness is inf - inf: the select sees +-inf keys and
    the tone map a finite scale, under which +inf radiance gives 255 and -inf gives 0."""
    rgb, dist, eid = mk.case_arrays("inf_negative")
    valid = eid != -1
    assert np.isposinf(rgb[valid]).any() and np.isneginf(rgb[valid]).any()
    assert not (np.isposinf(rgb).any(-1) & np.isneginf(rgb).any(-1)).any()
    scale = oracle.tone_scale(rgb.astype(np.float64), valid)
    assert np.isfinite(scale) and scale > 0
    bgr, _ = oracle.frame(rgb, dist, eid)
    rgb_out = bgr[..., ::-1]
    assert (rgb_out[np.isposinf(rgb)] == 255).all() and (rgb_out[np.isneginf(rgb)] == 0).all()


def test_fixture_covers_the_cases_and_the_csv_walk():
    assert set(OUT_CASES) == {f[0] for f in mk.FRAMES if f[5]} and "excluded" not in OUT_CASES
    assert str(PINS["entity_zero_error"]) == "AssertionError"
    with pytest.raises(ValueError):
        oracle.frame(*mk.case_arrays("entity_zero"))
    for split in ("train", "val", "test"):
        csv = str(PINS[f"text/filename_meta_{split}.csv"])
        assert csv.count("\n") - 1 == sum(1 for f in mk.FRAMES if f[4] == split and f[5])
    n_valid = int((mk.case_arrays("index_integral")[2] != -1).sum())
    assert ((n_valid - 1) * 0.9).is_integer()
    assert not ((int((mk.case_arrays("random_hdr")[2] != -1).sum()) - 1) * 0.9).is_integer()
    assert (np.asarray(mk.case_arrays("far_depth")[1], np.float64) / 886.81 * 886.81 * 1000 > 65535).any()


def test_unpinned_reference_differences_are_as_stored():
    """NumPy's own np.power changes no output pixel of these frames.  A level can only move where
    255 * pow(m, 1 / 2.2) lies within a few ulp of an integer.  Random radiance rarely gets there, but a channel equal
    to the frame's 90th-percentile brightness does: there m = pow(0.8, 2.2) and the level sits exactly on 204.0.  The
    constant frame is such a case; NumPy's power happens to round it correctly on this CPU."""
    assert PINS["unpinned_diff"].shape == (0, 5)
    assert bool(PINS["unpinned_text_equal"])
    rgb, _, eid = mk.case_arrays("constant")
    rgb = rgb.astype(np.float64)
    m = oracle.tone_scale(rgb, eid != -1) * rgb[0, 0, 0]
    assert m == oracle.pow_cr(0.8, oracle.INV_GAMMA) and oracle.pow_cr(m, oracle.GAMMA) * 255 == 204.0
    assert oracle.level_decimal(np.nextafter(m, 0)) == 203 and oracle.level_decimal(m) == 204


def test_pow_pin_is_correctly_rounded():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(0, 1, 300), np.exp(rng.uniform(-700, 700, 200)), oracle.boundary_args(400),
                        [5e-324, 1.0, 0.8]])
    got = oracle.pow_cr(x, oracle.GAMMA)
    assert np.array_equal(got, np.array([oracle.pow_decimal(v, oracle.GAMMA) for v in x]))
    assert oracle.pow_cr(0.8, oracle.INV_GAMMA) == data._tone_map_numerator() == oracle.pow_decimal(0.8, 2.2)


@pytest.mark.parametrize("H,W,focal", [(768, 1024, 886.81), (5, 7, 10.0), (480, 640, 500.5), (1, 1, 886.81)])
def test_plane_norm_equals_numpy_linalg_norm_of_the_scripts_plane(H, W, focal):
    x = np.linspace(-0.5 * W + 0.5, 0.5 * W - 0.5, W).reshape(1, W).repeat(H, 0).astype(np.float32)[:, :, None]
    y = np.linspace(-0.5 * H + 0.5, 0.5 * H - 0.5, H).reshape(H, 1).repeat(W, 1).astype(np.float32)[:, :, None]
    z = np.full([H, W, 1], focal, np.float32)
    want = np.linalg.norm(np.concatenate([x, y, z], 2), 2, 2)
    assert want.dtype == np.float32 and np.array_equal(oracle.plane_norm(H, W, focal), want)


def test_percentile_and_casts_equal_numpy():
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 10, 11, 101, 1000, 4097):
        v = rng.normal(0, 3, n)
        assert oracle.percentile90(v) == np.percentile(v, 90), n
        v[rng.integers(0, n)] = np.inf
        with np.errstate(invalid="ignore"):
            assert np.array_equal(oracle.percentile90(v), np.percentile(v, 90), equal_nan=True), n
    v = np.array([65536.7, 70000.2, -3.7, np.nan, np.inf, -np.inf, 3e9, 2.0 ** 31 - 1, 300.0])
    with np.errstate(invalid="ignore"):
        assert np.array_equal(oracle.wrap_cast(v, 16), v.astype(np.uint16))
        assert np.array_equal(oracle.wrap_cast(v, 8), v.astype(np.uint8))
    assert oracle.wrap_cast(v, 16)[:4].tolist() == [0, 4464, 65533, 0]


def _no_launch(monkeypatch):
    def load(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(data._lib, "load", load)


class _CudaLike(torch.Tensor):
    @property
    def is_cuda(self):
        return True


def _args(**over):
    a = {"rgb": torch.zeros(2, 4, 5, 3, dtype=torch.float16), "dist": torch.zeros(2, 4, 5, dtype=torch.float32),
         "entity_id": torch.ones(2, 4, 5, dtype=torch.int32)}
    a.update(over)
    return a


@pytest.mark.parametrize("bad", ["rgb_dtype", "dist_dtype", "eid_dtype", "rank", "shape", "cpu", "list", "focal"])
def test_hypersim_frames_rejects_bad_inputs_before_launch(bad, monkeypatch):
    _no_launch(monkeypatch)
    a = _args(**{"rgb_dtype": {"rgb": torch.zeros(2, 4, 5, 3, dtype=torch.float64)},
                 "dist_dtype": {"dist": torch.zeros(2, 4, 5, dtype=torch.bfloat16)},
                 "eid_dtype": {"entity_id": torch.ones(2, 4, 5, dtype=torch.int64)},
                 "rank": {"dist": torch.zeros(4, 5)}, "shape": {"entity_id": torch.ones(2, 4, 6, dtype=torch.int32)},
                 "list": {"rgb": [[0.0]]}}.get(bad, {}))
    if bad != "cpu":
        a = {k: v.as_subclass(_CudaLike) if isinstance(v, torch.Tensor) else v for k, v in a.items()}
    kw = {"focal": float("nan")} if bad == "focal" else {}
    with pytest.raises(ValueError):
        data.hypersim_frames(a["rgb"], a["dist"], a["entity_id"], **kw)


class _Entered(Exception):
    pass


def test_hypersim_frames_enters_the_tensor_device_before_any_copy(monkeypatch):
    entered = []

    class FakeDevice:
        def __init__(self, d):
            self.d = d

        def __enter__(self):
            entered.append(self.d)
            raise _Entered

        def __exit__(self, *a):
            return False
    monkeypatch.setattr(torch.cuda, "device", FakeDevice)
    _no_launch(monkeypatch)
    a = {k: v.as_subclass(_CudaLike) for k, v in _args().items()}
    with pytest.raises(_Entered):
        data.hypersim_frames(a["rgb"], a["dist"], a["entity_id"])
    assert entered == [a["rgb"].device]


@pytest.fixture
def raw_tree(tmp_path, monkeypatch):
    raw, csv = str(tmp_path / "raw"), str(tmp_path / "split.csv")
    registry = mk.write_raw_tree(raw, csv)
    monkeypatch.setitem(sys.modules, "h5py", mk.h5py_stub(registry))
    return raw, csv, str(tmp_path / "processed")


def test_preprocess_enters_the_device_before_any_copy_or_launch(raw_tree, monkeypatch):
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
    monkeypatch.setattr(data, "_hypersim_on_host", touched)
    raw, csv, out = raw_tree
    for device, want in (("cuda:1", "cuda:1"), (None, "cuda:0")):
        with pytest.raises(_Entered):
            data.preprocess_hypersim(csv, raw, out, num_workers=0, device=device)
        assert entered[-1] == torch.device(want)
    with pytest.raises(ValueError):
        data.preprocess_hypersim(csv, raw, out, device="cpu")
    with pytest.raises(ValueError):
        data.preprocess_hypersim(csv, raw, out, batch_size=0, device="cuda:0")


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

    def on_host(rgb, dist, eid, focal, dev):
        calls.append(tuple(rgb.shape))
        return oracle.emulated_frames_on_host(rgb, dist, eid, focal, dev)
    monkeypatch.setattr(data, "_hypersim_on_host", on_host)
    monkeypatch.setattr(torch.cuda, "device", _NoDevice)
    return calls


@pytest.mark.parametrize("workers", [0, 2])
def test_preprocess_writes_the_pinned_files(raw_tree, emulated, workers):
    raw, csv, out = raw_tree
    assert data.preprocess_hypersim(csv, raw, out, batch_size=3, num_workers=workers, device="cuda:0") == len(OUT_CASES)
    assert all(b <= 3 for b, *_ in emulated) and sum(b for b, *_ in emulated) == len(OUT_CASES)
    imgs, texts = mk.read_outputs(out)
    for c in OUT_CASES:
        assert imgs[c][0].dtype == np.uint8 and imgs[c][1].dtype == np.uint16
        for k in (0, 1):
            assert mk.sha256(imgs[c][k]) == str(PINS[f"out_sha/{c}/{k}"]), (c, k)
    for name, text in texts.items():
        assert text == str(PINS[f"text/{name}"]), name


def test_preprocess_edges(raw_tree, emulated, tmp_path):
    raw, csv, out = raw_tree
    os.makedirs(os.path.join(out, "test"))
    with pytest.raises(FileExistsError):
        data.preprocess_hypersim(csv, raw, out, num_workers=0, device="cuda:0")
    assert not os.path.exists(os.path.join(out, "train"))        # nothing written before the error
    os.rmdir(os.path.join(out, "test"))
    missing = os.path.join(raw, mk.input_paths("ai_002_001", "cam_02", 5)[2])
    os.remove(missing)
    with pytest.raises(FileNotFoundError, match=re.escape(missing)):
        data.preprocess_hypersim(csv, raw, out, num_workers=0, device="cuda:0")
    assert not os.path.exists(os.path.join(out, "train"))


def test_preprocess_names_the_file_holding_entity_id_zero(tmp_path, emulated, monkeypatch):
    raw, csv = str(tmp_path / "raw"), str(tmp_path / "split.csv")
    registry = mk.write_raw_tree(raw, csv, (mk.FRAMES[0], mk.ERROR_CASE))
    monkeypatch.setitem(sys.modules, "h5py", mk.h5py_stub(registry))
    with pytest.raises(data.HypersimEntityIdError, match="ai_009_001") as e:
        data.preprocess_hypersim(csv, raw, str(tmp_path / "out"), num_workers=0, device="cuda:0")
    assert e.value.frames == [1] and isinstance(e.value, ValueError)


def test_preprocess_without_h5py_raises_a_clear_import_error(raw_tree, monkeypatch):
    raw, csv, out = raw_tree
    monkeypatch.setitem(sys.modules, "h5py", None)
    monkeypatch.setattr(torch.cuda, "device", _NoDevice)
    with pytest.raises(ImportError, match="h5py"):
        data.preprocess_hypersim(csv, raw, out, num_workers=0, device="cuda:0")


def test_abi_table_agrees_with_the_header():
    header = open(os.path.join(os.path.dirname(HERE), "include", "b200_e2eft.h")).read()
    for name in ("b200_data_hypersim_workspace_bytes", "b200_data_hypersim_frames", "b200_debug_hypersim_pow"):
        decl = re.search(r"\b" + name + r"\(([^)]*)\)", header)
        assert decl, name
        assert len(decl.group(1).split(",")) == len(_lib._SIGS[name][1]), name
    assert _lib.ABI_VERSION == 17 and "(ABI 17)" in header
    src = open(os.path.join(os.path.dirname(HERE), "diffusion_e2e_ft_b200", "csrc", "gemm_conv.cu")).read()
    assert "b200_abi_version(void) { return 17; }" in src
