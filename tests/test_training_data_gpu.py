"""GPU tests of prepare_batch (csrc/data.cu): bitwise equality with the oracle (tests/data_oracle.py, checked against
the reference by tests/test_training_data_cpu.py) at full size, on every case of the reference-run fixture, without a
host sync, and through one E2E fine-tuning step."""
import os
import random
import sys

import numpy as np
import pytest
import torch
from torch.utils.data import default_collate

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import data_oracle as oracle  # noqa: E402
import make_data_pins as mk  # noqa: E402
from diffusion_e2e_ft_b200 import data  # noqa: E402

pytestmark = pytest.mark.gpu
KEYS = ("rgb", "depth", "metric", "normals", "val_mask")
DEV = "cuda:0"


def _synthetic(domain, H, W, seed, flips, lo, hi, invalid):
    rng = np.random.default_rng(seed)
    samples = []
    for f in flips:
        d = rng.integers(lo, hi, (H, W)).astype(np.uint16)
        d[rng.random((H, W)) < 0.05] = 0
        d[: H // 6] = invalid
        samples.append(data._sample(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), d,
                                    rng.integers(0, 256, (H, W, 3), dtype=np.uint8), f, True, 1e-5,
                                    65.0 if domain == "indoor" else 80.0, domain))
    return samples


def _pinned(batch):
    return {k: v.pin_memory() if isinstance(v, torch.Tensor) else v for k, v in batch.items()}


def _assert_equal(got, want, where):
    for k in KEYS:
        g = got[k][0] if got[k].dim() == want[k].dim() + 1 else got[k]
        assert g.dtype == want[k].dtype and g.shape == want[k].shape, (where, k, g.shape, want[k].shape)
        if not torch.equal(g.cpu(), want[k]):
            bad = (g.cpu() != want[k]).sum().item()
            raise AssertionError(f"{where} {k}: {bad} elements differ")


@pytest.mark.parametrize("domain", ["indoor", "outdoor"])
def test_full_size_matches_oracle(domain):
    H, W = (768, 1024) if domain == "indoor" else (375, 1242)
    lo, hi, inv = (300, 40000, 65535) if domain == "indoor" else (150, 12000, 65535)
    samples = _synthetic(domain, H, W, 7, (True, False), lo, hi, inv)
    out = data.prepare_batch(_pinned(default_collate(samples)))
    torch.cuda.synchronize()
    assert out["domain"] == [domain] * 2
    for b, s in enumerate(samples):
        want = oracle.sample_from_raw(s)
        got = {k: out[k][b] for k in KEYS}
        _assert_equal(got, want, (domain, b))
    assert out["val_mask"].dtype == torch.bool and out["rgb"].dtype == torch.float32
    assert tuple(out["depth"].shape) == ((2, 3, 480, 640) if domain == "indoor" else (2, 3, 352, 1216))


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("trees")
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        mk.write_hypersim_tree(str(tmp / "hypersim"), str(tmp))
        hs = data.Hypersim(str(tmp / "hypersim"), transform=True)
    finally:
        os.chdir(cwd)
    mk.write_vkitti_tree(str(tmp / "vkitti"))
    vk = data.VirtualKITTI2(str(tmp / "vkitti"), transform=True)
    vk.pairs = sorted(vk.pairs, key=lambda p: os.path.basename(p[0]))
    pins = torch.load(os.path.join(HERE, "golden", "data_pins.pt"), weights_only=False)
    return hs, vk, pins


def _raw_batch(ds, flip):
    samples = []
    for i in range(len(ds)):
        s = ds[i]
        s["flip"] = flip
        samples.append(s)
    return default_collate(samples)


@pytest.mark.parametrize("flip", [False, True])
def test_hypersim_pins_bitwise(trees, flip):
    hs, _, pins = trees
    out = data._prepare(_raw_batch(hs, flip), DEV, pins["hypersim_out"])
    for b, want in enumerate(pins["hypersim"][f"flip{int(flip)}"]):
        _assert_equal({k: out[k][b] for k in KEYS}, want, ("hypersim", flip, mk.CASES[b]))


@pytest.mark.parametrize("flip", [False, True])
def test_vkitti_pins_digests(trees, flip):
    _, vk, pins = trees
    out = data.prepare_batch(_raw_batch(vk, flip))
    for b, want in enumerate(pins["vkitti"][f"flip{int(flip)}"]):
        got = oracle.digests({k: out[k][b] for k in KEYS})
        assert all(got[k] == want[k] for k in KEYS), ("vkitti", flip, mk.CASES[b], [k for k in KEYS if got[k] != want[k]])


def test_no_host_sync():
    for domain, (H, W) in (("indoor", (768, 1024)), ("outdoor", (375, 1242))):
        batch = _pinned(default_collate(_synthetic(domain, H, W, 3, (False, True), 300, 9000, 65535)))
        data.prepare_batch(batch)                    # builds and uploads the tables once
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = data.prepare_batch(batch)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        assert out["val_mask"].any()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_other_device_than_the_current_one():
    batch = default_collate(_synthetic("indoor", 768, 1024, 5, (True, False), 300, 9000, 65535))
    torch.cuda.set_device(0)
    on1 = data.prepare_batch(batch, device="cuda:1")
    assert torch.cuda.current_device() == 0 and on1["rgb"].device == torch.device("cuda:1")
    on0 = data.prepare_batch(batch, device="cuda:0")
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    for k in KEYS:
        assert torch.equal(on1[k].cpu(), on0[k].cpu()), k


def test_e2e_ft_step_on_prepared_batch_matches_oracle_batch():
    import engine_checks as EC
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from diffusion_e2e_ft_b200.training import e2e_ft_loss
    samples = _synthetic("indoor", 96, 128, 11, (True, False), 300, 9000, 65535)
    out = data._prepare(default_collate(samples), DEV, (64, 64))
    ref = [oracle.sample_from_raw(s, size=(64, 64)) for s in samples]
    want = {k: torch.stack([r[k] for r in ref]).to(DEV) for k in KEYS}
    for k in KEYS:
        assert torch.equal(out[k], want[k]), k
    unet_ref, vae_ref = EC.MG.build_tiny()
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
    ctx = torch.randn(1, 77, 128, generator=torch.Generator().manual_seed(2)).to(DEV) * 0.5
    losses = []
    for b in (out, want):
        random.seed(0)
        loss, _ = e2e_ft_loss(unet, vae, DDIMScheduler(), b["rgb"], b["metric"], b["val_mask"], ctx, "depth")
        losses.append(loss.item())
    assert losses[0] == losses[1] and np.isfinite(losses[0])
