"""Write tests/golden/hypersim_pins.npz from the reference's own Hypersim preprocessing.

    python tests/golden/make_hypersim_pins.py <reference checkout>

A seeded synthetic Hypersim tree (write_raw_tree: a split CSV and one placeholder file per HDF5 render) is written to a
temporary directory, and the unmodified Marigold/script/dataset_preprocess/hypersim/preprocess_hypersim.py runs on it
through runpy with two stubs in sys.modules: `h5py`, whose File(path)["dataset"] serves the seeded arrays, and
`pylab`, which re-exports NumPy's count_nonzero, clip and np as pylab does.  It runs twice: once as it is, and once
with numpy.power replaced by a correctly rounded fp64 power (hypersim_oracle.pow_cr).  Every frame is 768 x 1024,
the size the script hard-codes.  The fixture stores SHA-256 digests of the inputs and of the pinned run's PNG pixels,
the pinned run's list and CSV text and 90th percentiles, the sparse differences of the unpinned run, and the script's failure on a frame
holding entity id 0 (run on its own, since the script stops there)."""
import contextlib
import hashlib
import io
import os
import runpy
import sys
import tempfile
import types
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import hypersim_oracle as oracle  # noqa: E402

OUT = os.path.join(HERE, "hypersim_pins.npz")
H, W = 768, 1024
# (case, scene, camera, frame id, split, included_in_public_release)
FRAMES = (
    ("random_hdr", "ai_001_001", "cam_00", 0, "train", True),
    ("random_hdr_f32", "ai_001_001", "cam_00", 1, "train", True),
    ("dark", "ai_001_001", "cam_01", 7, "train", True),
    ("all_invalid", "ai_001_002", "cam_00", 3, "train", True),
    ("excluded", "ai_001_002", "cam_00", 4, "train", False),
    ("constant", "ai_001_002", "cam_00", 12, "val", True),
    ("index_integral", "ai_002_001", "cam_00", 0, "val", True),
    ("nan_valid", "ai_002_001", "cam_02", 5, "val", True),
    ("nan_invalid", "ai_003_004", "cam_00", 99, "test", True),
    ("inf_negative", "ai_003_004", "cam_00", 100, "test", True),
    ("far_depth", "ai_003_004", "cam_01", 2, "test", True),
    ("nan_dist", "ai_003_005", "cam_00", 0, "train", True),
)
CASES = tuple(f[0] for f in FRAMES)
ERROR_CASE = ("entity_zero", "ai_009_001", "cam_00", 0, "train", True)


def case_arrays(name):
    """The seeded (color [H,W,3], depth_meters [H,W], render_entity_id [H,W] int32) of one case, in the dtypes the
    HDF5 files would hold (float16, or float32 where the case needs its range)."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    rgb = np.exp(rng.normal(-1.5, 1.5, (H, W, 3))).astype(np.float16)
    dist = (1.0 + 9.0 * rng.random((H, W)) + 3.0 * np.sin(x / 60.0) ** 2).astype(np.float16)
    eid = rng.integers(1, 400, (H, W)).astype(np.int32)
    eid[rng.random((H, W)) < 0.07] = -1
    if name == "random_hdr_f32":
        rgb = np.exp(rng.normal(0.0, 2.5, (H, W, 3))).astype(np.float32)
        dist = (0.3 + 40.0 * rng.random((H, W))).astype(np.float32)
    elif name == "dark":                        # p90 < 1e-4: scale 0
        rgb = (rng.random((H, W, 3)) * 5e-5).astype(np.float32)
    elif name == "all_invalid":                 # no valid pixel: scale 1
        eid[:] = -1
    elif name in ("random_hdr", "excluded"):
        pass
    elif name == "constant":                    # one brightness: the lerp of equal order statistics
        rgb[:] = np.float16(0.37)
    elif name == "index_integral":              # (n - 1) * 0.9 integral: 500001 valid pixels
        eid[:] = -1
        eid.flat[rng.choice(H * W, 500001, replace=False)] = 7
    elif name == "nan_valid":                   # a NaN brightness among the valid pixels: p90 and scale NaN
        rgb[5, 9, 1] = np.nan
        eid[5, 9] = 3
    elif name == "nan_invalid":                 # NaN only where invalid: ignored by the percentile
        rgb[eid == -1] = np.nan
    elif name == "inf_negative":                # +inf / -inf in one channel of a pixel, never both: the brightness
        rgb = rgb.astype(np.float32)            # is +-inf there, p90 and the scale stay finite
        u, ch = rng.random((H, W)), rng.integers(0, 3, (H, W))
        yy, xx = np.nonzero(u < 0.02)
        rgb[yy, xx, ch[yy, xx]] = np.inf
        yy, xx = np.nonzero((u >= 0.02) & (u < 0.04))
        rgb[yy, xx, ch[yy, xx]] = -np.inf
        rgb[(u >= 0.04) & (u < 0.12)] *= -1
    elif name == "far_depth":                   # plane depths past 65.535 m wrap; negative distances too
        dist = (rng.random((H, W)) * 150.0).astype(np.float32)
        dist[:40] = -rng.random((40, W)).astype(np.float32) * 3
        dist[40:60] = np.float32(3e6)
    elif name == "nan_dist":
        dist[100:110, 200:260] = np.nan
        dist[300, 300:320] = np.inf
        eid[100:105, 200:260] = -1
    elif name == "entity_zero":
        eid[10, 10] = 0
    else:
        raise KeyError(name)
    return rgb, dist, eid


def input_paths(scene, camera, frame_id):
    images = os.path.join(scene, "images")
    return (os.path.join(images, f"scene_{camera}_final_hdf5", f"frame.{frame_id:04d}.color.hdf5"),
            os.path.join(images, f"scene_{camera}_geometry_hdf5", f"frame.{frame_id:04d}.depth_meters.hdf5"),
            os.path.join(images, f"scene_{camera}_geometry_hdf5", f"frame.{frame_id:04d}.render_entity_id.hdf5"))


def write_raw_tree(dataset_dir, split_csv, frames=FRAMES):
    """The split CSV (Hypersim's metadata_images_split_scene_v1.csv columns) and an empty placeholder per HDF5 file
    under dataset_dir.  Returns {absolute path: case array} for the h5py stub."""
    import pandas as pd
    registry = {}
    for case, scene, cam, fid, _, _ in frames:
        for p, a in zip(input_paths(scene, cam, fid), case_arrays(case)):
            full = os.path.abspath(os.path.join(dataset_dir, p))
            os.makedirs(os.path.dirname(full), exist_ok=True)
            open(full, "wb").close()
            registry[full] = a
    pd.DataFrame({"scene_name": [f[1] for f in frames], "camera_name": [f[2] for f in frames],
                  "frame_id": [f[3] for f in frames], "included_in_public_release": [f[5] for f in frames],
                  "exclude_reason": ["" if f[5] else "bad" for f in frames],
                  "split_partition_name": [f[4] for f in frames]}).to_csv(split_csv, index=False)
    return registry


def h5py_stub(registry):
    """A module whose File(path, mode)["dataset"] is the registered array for that path."""
    class File:
        def __init__(self, path, mode="r"):
            self.a = registry[os.path.abspath(path)]

        def __getitem__(self, key):
            assert key == "dataset", key
            return self.a

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False
    return types.SimpleNamespace(File=File, __name__="h5py")


def pylab_stub():
    return types.SimpleNamespace(count_nonzero=np.count_nonzero, clip=np.clip, np=np, __name__="pylab")


@contextlib.contextmanager
def stubs(registry):
    saved = {k: sys.modules.get(k) for k in ("h5py", "pylab")}
    sys.modules["h5py"] = h5py_stub(registry)
    sys.modules["pylab"] = pylab_stub()
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def run_script(script, split_csv, dataset_dir, output_dir, registry, pinned):
    """Runs the script; returns the values its np.percentile calls returned, in call order (one per frame with a
    valid pixel)."""
    original, original_percentile = np.power, np.percentile
    p90 = []

    def percentile(*a, **k):
        p90.append(float(original_percentile(*a, **k)))
        return p90[-1]

    def power(base, expo, *a, **k):
        if a or k or np.ndim(expo) != 0 or np.asarray(base).dtype != np.float64:
            return original(base, expo, *a, **k)
        return oracle.pow_cr(base, float(expo))
    argv = sys.argv
    sys.argv = [script, "--split_csv", split_csv, "--dataset_dir", dataset_dir, "--output_dir", output_dir]
    np.power = power if pinned else original
    np.percentile = percentile
    sys.modules.pop("hypersim_util", None)
    try:
        with stubs(registry), contextlib.redirect_stderr(io.StringIO()), contextlib.redirect_stdout(io.StringIO()):
            runpy.run_path(script, run_name="__main__")
    finally:
        np.power, np.percentile = original, original_percentile
        sys.argv = argv
    return p90


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def read_outputs(output_dir, frames=FRAMES):
    """{case: (bgr, depth)} of the PNGs the script wrote, and {file name: text} of its lists and CSVs."""
    import cv2
    imgs = {}
    for case, scene, cam, fid, split, inc in frames:
        if inc:
            d = os.path.join(output_dir, split, scene)
            imgs[case] = (cv2.imread(os.path.join(d, f"rgb_{cam}_fr{fid:04d}.png"), cv2.IMREAD_UNCHANGED),
                          cv2.imread(os.path.join(d, f"depth_plane_{cam}_fr{fid:04d}.png"), cv2.IMREAD_UNCHANGED))
    texts = {}
    for split in ("train", "val", "test"):
        for name in (f"filename_list_{split}.txt", f"filename_meta_{split}.csv"):
            texts[name] = open(os.path.join(output_dir, split, name)).read()
    return imgs, texts


def main(ref):
    script = os.path.join(os.path.abspath(ref), "Marigold", "script", "dataset_preprocess", "hypersim",
                          "preprocess_hypersim.py")
    sys.path.insert(0, os.path.dirname(script))
    with tempfile.TemporaryDirectory() as tmp:
        raw, csv = os.path.join(tmp, "raw"), os.path.join(tmp, "split.csv")
        registry = write_raw_tree(raw, csv)
        outs = {}
        for pinned in (False, True):
            out = os.path.join(tmp, f"out_{int(pinned)}")
            p90 = run_script(script, csv, raw, out, registry, pinned)
            outs[pinned] = read_outputs(out)
        csv0 = os.path.join(tmp, "split_error.csv")
        reg0 = write_raw_tree(os.path.join(tmp, "raw_error"), csv0, (ERROR_CASE,))
        try:
            run_script(script, csv0, os.path.join(tmp, "raw_error"), os.path.join(tmp, "out_error"), reg0, True)
            error = "none"
        except AssertionError:
            error = "AssertionError"
    pins = {"cases": np.array(CASES), "entity_zero_error": np.array(error)}
    (imgs, texts), (imgs_u, texts_u) = outs[True], outs[False]
    for name, text in texts.items():
        pins[f"text/{name}"] = np.array(text)
    diff = []
    # the script's 90th percentiles, in its walk order (split by split, rows in order), NaN for a frame without a
    # valid pixel (the script computes none there)
    walk = [c for split in ("train", "val", "test") for c, _, _, _, sp, inc in FRAMES if sp == split and inc]
    with_valid = [c for c in walk if (case_arrays(c)[2] != -1).any()]
    assert len(p90) == len(with_valid), (len(p90), with_valid)
    for c in walk:
        pins[f"p90/{c}"] = np.array(p90[with_valid.index(c)] if c in with_valid else np.nan)
    for i, c in enumerate(CASES):
        arrays = case_arrays(c)
        pins[f"in_sha/{c}"] = np.array(sha256(np.concatenate([a.reshape(-1).view(np.uint8) for a in arrays])))
        if c not in imgs:
            continue
        for k, (a, b) in enumerate(zip(imgs[c], imgs_u[c])):
            pins[f"out_sha/{c}/{k}"] = np.array(sha256(a))
            for idx in zip(*np.nonzero(a != b)):
                diff.append((i, k, int(np.ravel_multi_index(idx, a.shape)), int(b[idx]), int(a[idx])))
        bgr, depth = oracle.frame(*arrays)
        print(f"{c:16s} oracle == pinned reference: {np.array_equal(bgr, imgs[c][0])} {np.array_equal(depth, imgs[c][1])}"
              f"  unpinned differs at {int((imgs[c][0] != imgs_u[c][0]).sum())}")
    pins["unpinned_diff"] = np.array(diff, np.int64).reshape(-1, 5)   # case, output (0 rgb, 1 depth), flat index,
    pins["unpinned_text_equal"] = np.array(texts == texts_u)          # unpinned, pinned
    np.savez_compressed(OUT, **pins)
    print(f"{OUT}: {os.path.getsize(OUT)} bytes, {len(diff)} unpinned differences, entity id 0 -> {error}")


if __name__ == "__main__":
    main(sys.argv[1])
