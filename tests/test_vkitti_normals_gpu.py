"""GPU tests of the Virtual KITTI 2 normal generation (b200_data_vkitti_normals in csrc/data.cu): bitwise equality with
the oracle (tests/vkitti_normals_oracle.py, held to the reference run by tests/test_vkitti_normals_cpu.py) on every
case of tests/golden/vkitti_normals_pins.npz and on a full-size batch, independence of batch position and size, no
host sync, a second device, and generate_vkitti_normals end to end into the training loader."""
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

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PINS = dict(np.load(os.path.join(HERE, "golden", "vkitti_normals_pins.npz")))


def _run(depths, device=DEV):
    d = torch.from_numpy(np.stack(depths)).to(device)
    out = data.vkitti_normals(d)
    assert out.dtype == torch.uint16 and out.device == d.device and tuple(out.shape) == d.shape + (3,)
    return out.cpu().numpy()


@pytest.mark.parametrize("case", mk.SMALL)
def test_kernel_equals_the_pinned_reference_on_every_small_case(case):
    got = _run([mk.case_depth(case)])[0]
    assert np.array_equal(got, PINS[f"out/{case}"]) and np.array_equal(got, oracle.normals_frame(mk.case_depth(case)))


def test_kernel_full_size_batch_equals_oracle_and_pins():
    depths = [mk.case_depth(c) for c in mk.FULL_CASES]
    got = _run(depths)
    for c, g, d in zip(mk.FULL_CASES, got, depths):
        assert mk.sha256(g) == str(PINS[f"out_sha/{c}"]), c
        assert np.array_equal(g, oracle.normals_frame(d)), c


def test_kernel_on_distinct_seeded_frames_equals_oracle():
    """Four more full-size frames the fixture does not hold: random cm in a narrow band (many near-e ratios) and the
    full 0 .. 65535 range."""
    rng = np.random.default_rng(11)
    depths = [(1500 + rng.integers(0, 6, mk.FULL) + np.arange(mk.FULL[1]) // 3).astype(np.uint16) for _ in range(2)]
    depths += [rng.integers(0, 65536, mk.FULL).astype(np.uint16) for _ in range(2)]
    got = _run(depths)
    for g, d in zip(got, depths):
        assert np.array_equal(g, oracle.normals_frame(d))


def test_result_does_not_depend_on_batch_position_or_size():
    depths = [mk.case_depth(c) for c in mk.FULL_CASES]
    four = _run(depths)
    rev = _run(depths[::-1])[::-1]
    assert np.array_equal(four, rev)
    for i, d in enumerate(depths):
        assert np.array_equal(_run([d])[0], four[i])
    sixteen = _run(depths * 4)
    assert all(np.array_equal(sixteen[i], four[i % 4]) for i in range(16))


def test_no_host_sync():
    d = torch.from_numpy(np.stack([mk.case_depth(c) for c in mk.FULL_CASES])).to(DEV)
    data.vkitti_normals(d)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = data.vkitti_normals(d, fx=700.0, fy=710.0, u0=600.0, v0=180.0)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    want = oracle.normals_frame(mk.case_depth(mk.FULL_CASES[0]), fx=700.0, fy=710.0, u0=600.0, v0=180.0)
    assert np.array_equal(out[0].cpu().numpy(), want)


def _pow(x, force_slow):
    L = data._lib.load()
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
    out = torch.empty_like(xd)
    slow = torch.zeros(1, dtype=torch.int32, device=DEV)
    data._ck(L.b200_debug_pow_e32_neg(data._p(xd), xd.numel(), int(force_slow), data._p(out), data._p(slow),
                                      data._stream()), "b200_debug_pow_e32_neg")
    return out.cpu().numpy(), int(slow.item())


@pytest.fixture(scope="module")
def near_boundary():
    x = oracle.near_boundary_args()
    assert len(x) > 10
    return x


def test_power_near_rounding_boundaries_takes_the_exact_path(near_boundary):
    """The kernel's own float32(e) ** -x on the arguments whose value lies within 2^-44 of an fp32 rounding boundary:
    some of them fall inside the fast path's 2^-46 guard and are decided by the double-double exp."""
    got, slow = _pow(near_boundary, False)
    want = np.array([oracle.pow_e32_decimal(v) for v in near_boundary], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert 1 <= slow <= len(near_boundary)


@pytest.mark.parametrize("args", ["near", "grid", "subnormal", "random"])
def test_power_double_double_path_is_correctly_rounded(args, near_boundary):
    """The double-double path forced for every argument, against `decimal`; and the default path on the same."""
    rng = np.random.default_rng(3)
    x = {"near": near_boundary, "grid": np.arange(0, 221, dtype=np.float32) / np.float32(2),
         "subnormal": np.linspace(87.0, 104.5, 3000, dtype=np.float32),
         "random": np.concatenate([rng.uniform(0, 110, 3000), rng.uniform(0, 2, 1000)]).astype(np.float32)}[args]
    want = np.array([oracle.pow_e32_decimal(v) for v in x], np.float32).view(np.uint32)
    forced, slow = _pow(x, True)
    assert slow == len(x) and np.array_equal(forced.view(np.uint32), want)
    assert np.array_equal(_pow(x, False)[0].view(np.uint32), want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_second_device():
    torch.cuda.set_device(0)
    got = _run([mk.case_depth(c) for c in mk.FULL_CASES[:2]], device="cuda:1")
    for c, g in zip(mk.FULL_CASES, got):
        assert mk.sha256(g) == str(PINS[f"out_sha/{c}"]), c


def test_generate_writes_the_pinned_pngs_and_the_training_loader_reads_them(tmp_path):
    import cv2
    root = str(tmp_path / "virtual_kitti_2")
    files = mk.write_normals_tree(root)
    assert data.generate_vkitti_normals(root, batch_size=3, num_workers=2, device=DEV) == len(files)
    for case, (_, normal) in files.items():
        img = cv2.imread(os.path.join(root, normal), cv2.IMREAD_UNCHANGED)
        assert img.dtype == np.uint16 and mk.sha256(img) == str(PINS[f"out_sha/{case}"]), case
    ds = data.VirtualKITTI2(root, transform=True)
    assert len(ds) == len(mk.FULL_CASES)
    loader = torch.utils.data.DataLoader(ds, batch_size=2, num_workers=0, pin_memory=True)
    for raw in loader:
        batch = data.prepare_batch(raw, device=DEV)
        assert tuple(batch["normals"].shape) == (2, 3, *data.KB_CROP) and batch["val_mask"].any()
        assert torch.isfinite(batch["normals"]).all() and (batch["normals"].abs().amax(1) > 0.5).any()
