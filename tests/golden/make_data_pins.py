"""Write tests/golden/data_pins.pt: what the reference's training datasets (training/dataloaders/load.py `Hypersim`,
`VirtualKITTI2`) return for synthetic Hypersim and Virtual KITTI 2 trees, with the flip forced each way.

    python tests/golden/make_data_pins.py <reference checkout>

The trees come from `write_hypersim_tree` / `write_vkitti_tree` (seeded, so the tests write the same files again).
Hypersim is pinned at 48x64 -> 30x40 through `SynchronizedTransform_Hyper(30, 40)` (the recipe's 1.6 ratio) and its
outputs are stored; the Virtual KITTI 2 crop is fixed at 352x1216, so only SHA-256 digests of its outputs are stored.
Cases: random depths with invalid pixels (zero depth; the VKITTI sky at 655.35 m past the far plane) and normals
facing towards and away from the camera, all valid depths equal, exactly one valid pixel, and no valid pixel.
"""
import os
import random
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
HYPERSIM_IN = (48, 64)
HYPERSIM_OUT = (30, 40)
VKITTI_IN = (375, 1242)
CASES = ("random", "equal", "one_valid", "none_valid")


def _nearest_rows_cols(in_hw, out_hw):
    """Source pixels Pillow's NEAREST resize samples, read off a resized index image."""
    from PIL import Image
    H, W = in_hw
    idx = np.arange(H * W, dtype=np.float32).reshape(H, W)
    r = np.array(Image.fromarray(idx).resize(out_hw[::-1], Image.NEAREST))
    return (r[:, 0] // W).astype(int), (r[0] % W).astype(int)


def _depth(case, shape, rng, lo, hi, invalid, one_at):
    d = rng.integers(lo, hi, shape).astype(np.uint16)
    if case == "random":
        d[rng.random(shape) < 0.1] = 0
        d[: shape[0] // 5] = invalid                    # a band past the far plane (VKITTI sky)
    elif case == "equal":
        d[:] = (lo + hi) // 2
        d[rng.random(shape) < 0.2] = 0
    elif case == "one_valid":
        d[:] = invalid
        d[one_at] = (lo + hi) // 3
    else:
        d[:] = 0
        d[: shape[0] // 2] = invalid
    return d


def write_hypersim_tree(root, csv_dir):
    """Hypersim layout under root (train/<scene>/images/..., normals/<scene>/images/...) and the split CSV under
    csv_dir/data/hypersim/processed/train/.  Returns the CSV rows' (rgb, depth, normal) paths the reference keeps."""
    from PIL import Image
    import pandas as pd
    rng = np.random.default_rng(20261017)
    rows, kept = [], []
    sr, sc = _nearest_rows_cols(HYPERSIM_IN, HYPERSIM_OUT)
    for i, case in enumerate(CASES):
        scene, cam, frame = f"ai_001_{i:03d}", "cam_00", i
        rgb_rel = os.path.join(scene, "images", f"scene_{cam}_final_preview",
                               f"frame.{frame:04d}.tonemap." + ("jpg" if i % 2 else "png"))
        depth_rel = os.path.join(scene, "images", f"scene_{cam}_geometry_hdf5", f"frame.{frame:04d}.depth_meters.png")
        normal = os.path.join(root, "normals", scene, "images", f"scene_{cam}_geometry_preview",
                              f"frame.{frame:04d}.normal_cam.png")
        for p in (os.path.join(root, "train", rgb_rel), os.path.join(root, "train", depth_rel), normal):
            os.makedirs(os.path.dirname(p), exist_ok=True)
        rgb = rng.integers(0, 256, (*HYPERSIM_IN, 3), dtype=np.uint8)
        Image.fromarray(rgb).save(os.path.join(root, "train", rgb_rel), quality=90)
        one_at = (sr[HYPERSIM_OUT[0] // 2], sc[HYPERSIM_OUT[1] // 3])
        d = _depth(case, HYPERSIM_IN, rng, 400, 30000, 65535, one_at)
        Image.fromarray(d).save(os.path.join(root, "train", depth_rel))
        Image.fromarray(rng.integers(0, 256, (*HYPERSIM_IN, 3), dtype=np.uint8)).save(normal)
        rows.append(dict(scene_name=scene, camera_name=cam, frame_id=frame, included_in_public_release=True,
                         split_partition_name="train", rgb_path=rgb_rel, depth_path=depth_rel))
        kept.append((os.path.join(root, "train", rgb_rel), os.path.join(root, "train", depth_rel), normal))
    # rows the reference skips: not released, another split, a missing file
    rows.append(dict(rows[0], included_in_public_release=False))
    rows.append(dict(rows[1], split_partition_name="val"))
    rows.append(dict(rows[2], frame_id=99, rgb_path=rows[2]["rgb_path"].replace("0002", "0099")))
    csv = os.path.join(csv_dir, "data", "hypersim", "processed", "train", "filename_meta_train.csv")
    os.makedirs(os.path.dirname(csv), exist_ok=True)
    pd.DataFrame(rows).to_csv(csv, index=False)
    return kept


def write_vkitti_tree(root):
    """Virtual KITTI 2 layout under root: JPEG RGB, 16-bit depth PNG in cm, 16-bit RGB normal PNG.  Returns the
    (rgb, depth, normal) paths in case order."""
    import cv2
    rng = np.random.default_rng(20261018)
    out = []
    H, W = VKITTI_IN
    for i, case in enumerate(CASES):
        scene, weather, cam = ("Scene01", "Scene06")[i % 2], ("morning", "fog")[i // 2], "Camera_0"
        stem = f"_{i:05d}"
        paths = (os.path.join(root, "vkitti_2.0.3_rgb", scene, weather, "frames", "rgb", cam, f"rgb{stem}.jpg"),
                 os.path.join(root, "vkitti_2.0.3_depth", scene, weather, "frames", "depth", cam, f"depth{stem}.png"),
                 os.path.join(root, "vkitti_DAG_normals", scene, weather, "frames", "normal", cam, f"normal{stem}.png"))
        for p in paths:
            os.makedirs(os.path.dirname(p), exist_ok=True)
        cv2.imwrite(paths[0], rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        cv2.imwrite(paths[1], _depth(case, (H, W), rng, 150, 9000, 65535, (H - 100, W // 3)))
        cv2.imwrite(paths[2], rng.integers(0, 65536, (H, W, 3), dtype=np.uint16))
        out.append(paths)
    os.makedirs(os.path.join(root, "vkitti_2.0.3_rgb", "Scene02", "rain", "frames", "rgb", "Camera_1"), exist_ok=True)
    return out


def _run(ds, force):
    import load as ref
    real = ref.random.random
    ref.random.random = lambda: force
    try:
        return [ds[i] for i in range(len(ds))]
    finally:
        ref.random.random = real


def main(ref_root):
    sys.path.insert(0, os.path.join(ref_root, "training", "dataloaders"))
    import load as ref
    pins = {"hypersim_in": HYPERSIM_IN, "hypersim_out": HYPERSIM_OUT, "cases": CASES}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)                       # Hypersim reads its split CSV relative to the working directory
        try:
            hroot = os.path.join(tmp, "hypersim")
            kept = write_hypersim_tree(hroot, tmp)
            ds = ref.Hypersim(root_dir=hroot, transform=True)
            ds.transform = ref.SynchronizedTransform_Hyper(*HYPERSIM_OUT)
            assert [(p["rgb_path"], p["depth_path"], p["normal_path"]) for p in ds.pairs] == kept
            pins["hypersim"] = {f"flip{f}": _run(ds, 0.9 if f else 0.1) for f in (0, 1)}
            vroot = os.path.join(tmp, "vkitti")
            paths = write_vkitti_tree(vroot)
            ds = ref.VirtualKITTI2(root_dir=vroot, transform=True)
            assert sorted(ds.pairs) == sorted(paths), ds.pairs
            ds.pairs = paths                # case order (the reference lists directories in os.listdir order)
            from data_oracle import digests
            pins["vkitti"] = {f"flip{f}": [dict(digests(s), domain=s["domain"]) for s in _run(ds, 0.9 if f else 0.1)]
                              for f in (0, 1)}
        finally:
            os.chdir(cwd)
    for s in pins["hypersim"]["flip0"] + pins["hypersim"]["flip1"]:
        for k in ("rgb", "depth", "metric", "normals", "val_mask"):
            s[k] = s[k].contiguous().clone()
    path = os.path.join(HERE, "data_pins.pt")
    torch.save(pins, path)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    main(sys.argv[1])
