"""CPU tests of the training inputs (diffusion_e2e_ft_b200.data): the oracle against the reference-run fixture
tests/golden/data_pins.pt, the Pillow resampling tables against PIL, file discovery, the mixer, the flip draws and
prepare_batch's argument checks."""
import ast
import os
import random
import sys

import numpy as np
import pytest
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import data_oracle as oracle  # noqa: E402
import make_data_pins as mk  # noqa: E402
from diffusion_e2e_ft_b200 import data  # noqa: E402

KEYS = ("rgb", "depth", "metric", "normals", "val_mask")


@pytest.fixture(scope="module")
def pins():
    return torch.load(os.path.join(HERE, "golden", "data_pins.pt"), weights_only=False)


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("trees")
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        mk.write_hypersim_tree(str(tmp / "hypersim"), str(tmp))
        mk.write_vkitti_tree(str(tmp / "vkitti"))
        hs = data.Hypersim(str(tmp / "hypersim"), transform=True)
    finally:
        os.chdir(cwd)
    vk = data.VirtualKITTI2(str(tmp / "vkitti"), transform=True)
    vk.pairs = sorted(vk.pairs, key=lambda p: os.path.basename(p[0]))
    return hs, vk


def _raw(ds, i, flip):
    random.seed(0)
    s = ds[i]
    s["flip"] = flip
    return s


def test_file_discovery_follows_the_reference(trees):
    hs, vk = trees
    assert [os.path.basename(p["rgb_path"]) for p in hs.pairs] == \
        ["frame.0000.tonemap.png", "frame.0001.tonemap.jpg", "frame.0002.tonemap.png", "frame.0003.tonemap.jpg"]
    assert all(p["normal_path"].endswith(".normal_cam.png") and "geometry_preview" in p["normal_path"] for p in hs.pairs)
    assert len(vk) == 4 and [os.path.basename(p[1]) for p in vk.pairs] == [f"depth_{i:05d}.png" for i in range(4)]
    s = vk[0]
    assert s["rgb"].dtype == torch.uint8 and s["depth"].dtype == torch.uint16 and s["normals"].dtype == torch.uint8
    assert tuple(s["rgb"].shape) == (375, 1242, 3) and tuple(s["depth"].shape) == (375, 1242)
    assert s["domain"] == "outdoor" and s["far_plane"] == 80.0 and hs[0]["domain"] == "indoor"


def test_oracle_matches_reference_pins_hypersim(trees, pins):
    hs, _ = trees
    for f in (0, 1):
        for i, ref in enumerate(pins["hypersim"][f"flip{f}"]):
            got = oracle.sample_from_raw(_raw(hs, i, bool(f)), size=pins["hypersim_out"])
            for k in KEYS:
                assert got[k].dtype == ref[k].dtype and torch.equal(got[k], ref[k]), (f, i, k)


def test_oracle_matches_reference_pins_vkitti(trees, pins):
    _, vk = trees
    for f in (0, 1):
        for i, ref in enumerate(pins["vkitti"][f"flip{f}"]):
            got = oracle.digests(oracle.sample_from_raw(_raw(vk, i, bool(f))))
            assert all(got[k] == ref[k] for k in KEYS), (f, i)


def test_pins_cover_the_edge_cases(pins):
    """Random depths keep a mask; equal depths and a single valid pixel (min == max) and no valid pixel give an empty
    mask and zero depth."""
    s = pins["hypersim"]["flip0"]
    assert s[0]["val_mask"].sum() > 1 and (s[0]["depth"] == 1).any() and (s[0]["normals"] != 0).any()
    for i in (1, 2, 3):
        assert s[i]["val_mask"].sum() == 0 and s[i]["metric"].abs().sum() == 0 and s[i]["normals"].abs().sum() == 0


@pytest.mark.parametrize("shape", [(768, 1024, 480, 640), (96, 128, 60, 80), (48, 64, 30, 40), (30, 40, 75, 100)])
def test_bilinear_tables_reproduce_pillow(shape):
    H, W, h, w = shape
    a = np.random.default_rng(1).integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref = np.array(Image.fromarray(a).resize((w, h), Image.BILINEAR))

    def axis_pass(x, first, kk):        # x [N, in, C] -> [N, out, C]
        acc = np.full((x.shape[0], len(first), x.shape[2]), 1 << 21, np.int64)
        for j in range(kk.shape[1]):
            idx = np.minimum(first + j, x.shape[1] - 1)
            acc += kk[None, :, j, None].astype(np.int64) * x[:, idx].astype(np.int64)
        return np.clip(acc >> 22, 0, 255).astype(np.uint8)
    t = axis_pass(a, *data.pillow_bilinear_coeffs(W, w))
    mine = axis_pass(t.transpose(1, 0, 2), *data.pillow_bilinear_coeffs(H, h)).transpose(1, 0, 2)
    assert np.array_equal(mine, ref)


@pytest.mark.parametrize("shape", [(768, 1024, 480, 640), (96, 128, 60, 80), (48, 64, 30, 40), (375, 1242, 352, 1216)])
def test_nearest_tables_reproduce_pillow(shape):
    H, W, h, w = shape
    rows, cols = mk._nearest_rows_cols((H, W), (h, w))
    assert np.array_equal(data.pillow_nearest_index(H, h), rows)
    assert np.array_equal(data.pillow_nearest_index(W, w), cols)
    if (H, W) == (768, 1024):        # the floor((i + 0.5) * s) rule of nearest-exact differs here
        assert (np.floor((np.arange(w) + 0.5) * (W / w)).astype(int) != cols).sum() > 0


def test_flip_draws_consume_random_as_the_reference(trees):
    hs, vk = trees
    random.seed(123)
    want = [random.random() > 0.5 for _ in range(6)]
    random.seed(123)
    got = [hs[i % 4]["flip"] for i in range(3)] + [vk[i]["flip"] for i in range(3)]
    assert got == want
    off = data.VirtualKITTI2(vk.root_dir, transform=None)
    random.seed(5)
    state = random.getstate()
    assert off[0]["flip"] is False and random.getstate() == state


def test_mixed_loader_length_fractions_and_order():
    a, b = list(range(90)), [f"b{i}" for i in range(40)]
    m = data.MixedDataLoader(a, b, split1=9, split2=1)
    assert m.frac1 == 1 and m.frac2 == pytest.approx(90 / 40 / 9)
    assert len(m) == 90 + int(40 * m.frac2) == 100
    np.random.seed(3)
    out = list(m)
    assert len(out) == 100 and [x for x in out if isinstance(x, int)] == a
    np.random.seed(3)
    choice = [True] * 90 + [False] * 10
    np.random.shuffle(choice)
    assert [isinstance(x, int) for x in out] == choice


def _batch(B=2, H=8, W=10, domain="indoor"):
    return {"rgb": torch.zeros(B, H, W, 3, dtype=torch.uint8), "depth": torch.zeros(B, H, W, dtype=torch.uint16),
            "normals": torch.zeros(B, H, W, 3, dtype=torch.uint8), "flip": torch.zeros(B, dtype=torch.bool),
            "transform": torch.ones(B, dtype=torch.bool), "near_plane": torch.full((B,), 1e-5, dtype=torch.float64),
            "far_plane": torch.full((B,), 65.0, dtype=torch.float64), "domain": [domain] * B}


@pytest.mark.parametrize("bad", ["rgb_dtype", "depth_dtype", "shape", "flip", "domain", "mixed", "missing", "device",
                                 "planes", "crop"])
def test_prepare_batch_rejects_bad_inputs_before_launch(bad):
    b = _batch()
    kw = {}
    if bad == "rgb_dtype":
        b["rgb"] = b["rgb"].float()
    elif bad == "depth_dtype":
        b["depth"] = b["depth"].to(torch.int32)
    elif bad == "shape":
        b["normals"] = b["normals"][:, :, :5]
    elif bad == "flip":
        b["flip"] = torch.zeros(3, dtype=torch.bool)
    elif bad == "domain":
        b["domain"] = ["garden"] * 2
    elif bad == "mixed":
        b["domain"] = ["indoor", "outdoor"]
    elif bad == "missing":
        del b["normals"]
    elif bad == "device":
        kw["device"] = "cpu"
    elif bad == "planes":
        b["far_plane"][:] = 0.0
        kw["device"] = "cuda:0"
    elif bad == "crop":                  # Virtual KITTI 2 smaller than the 352x1216 benchmark crop
        b = _batch(domain="outdoor")
        b["far_plane"][:] = 80.0
        kw["device"] = "cuda:0"
    with pytest.raises(ValueError):
        data.prepare_batch(b, **kw)


class _Entered(Exception):
    pass


def test_prepare_batch_runs_under_the_target_device(monkeypatch):
    """The copies, the launches (ctypes calls on the current device and stream) and the table uploads must target
    `device` even when another device is current: prepare_batch enters torch.cuda.device(device) before any of them."""
    entered = []

    class FakeDevice:
        def __init__(self, d):
            self.d = torch.device(d)

        def __enter__(self):
            entered.append(self.d)
            raise _Entered

        def __exit__(self, *a):
            return False

    def no_launch():
        raise AssertionError("library touched outside the device context")
    monkeypatch.setattr(torch.cuda, "device", FakeDevice)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(data._lib, "load", no_launch)
    for device, want in (("cuda:1", "cuda:1"), (None, "cuda:0"), (torch.device("cuda", 2), "cuda:2")):
        with pytest.raises(_Entered):
            data.prepare_batch(_batch(), device=device)
        assert entered[-1] == torch.device(want)


def test_product_package_never_imports_the_data_oracle():
    pkg = os.path.join(os.path.dirname(HERE), "diffusion_e2e_ft_b200")
    for name in sorted(os.listdir(pkg)):
        if name.endswith(".py"):
            for node in ast.walk(ast.parse(open(os.path.join(pkg, name)).read())):
                if isinstance(node, (ast.Import, ast.ImportFrom)):
                    mods = [a.name for a in node.names] if isinstance(node, ast.Import) else [node.module or ""]
                    assert not any(m.split(".")[0] in ("data_oracle", "oracle", "load") for m in mods), (name, mods)
