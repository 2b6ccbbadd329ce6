"""Write tests/golden/vkitti_normals_pins.npz from the reference's own normal generator.

    python tests/golden/make_vkitti_normals_pins.py <reference checkout>

A seeded synthetic Virtual KITTI 2 tree (write_normals_tree) is written to a temporary directory, and the unmodified
depth-to-normal-translator/python/gen_vkitti_normals.py runs there through runpy (its root is the relative
data/virtual_kitti_2), twice: once as it is, and once with numpy.power(e, lap32) replaced by the correctly rounded
fp32 power (vkitti_normals_oracle.pow_e32_neg).  The pinned run's outputs are stored in full for the small cases and
as SHA-256 for the full-size frames, together with the sparse differences of the unpinned run and the script's pair
list relative to its root."""
import hashlib
import os
import runpy
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import vkitti_normals_oracle as oracle  # noqa: E402

OUT = os.path.join(HERE, "vkitti_normals_pins.npz")
FULL = (375, 1242)
ROOT = os.path.join("data", "virtual_kitti_2")


def _piecewise_linear(n, slopes, start=1000):
    return start + np.concatenate([[0], np.cumsum(np.asarray(slopes)[np.arange(n - 1) * len(slopes) // max(n - 1, 1)])])


def case_depth(name):
    """The seeded uint16 centimetre depth of one case."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    small = {"random": (24, 40), "random_narrow": (24, 40), "smooth": (32, 48), "planes": (20, 30), "steps": (24, 32),
             "sky": (24, 32), "zeros": (16, 20), "constant": (8, 8), "tiny_3x3": (3, 3), "tiny_3x4": (3, 4),
             "tiny_4x3": (4, 3), "tiny_5x7": (5, 7)}
    H, W = small.get(name, FULL)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    kind = name[5:] if name.startswith("full_") else name
    if kind == "random":
        d = rng.integers(0, 65536, (H, W))
    elif kind in ("random_narrow",) or kind.startswith("tiny"):
        d = 1000 + rng.integers(0, 5, (H, W))
    elif kind == "smooth":
        d = np.rint(1500 + 40000 * (y / H) ** 2 + 800 * np.sin(x / 9.0 + y / 23.0) * np.cos(y / 7.0))
    elif kind == "planes":       # integer cm slopes whose changes of 0, 1 and 2 put soft_min's ratios at 1, ~e, ~e^2
        d = _piecewise_linear(W, [2, 3, 3, 5, 4, 4, 6, 7, 7, 9])[None, :] + _piecewise_linear(H, [1, 2, 2, 4], 0)[:, None]
    elif kind == "steps":
        d = 800 + 350 * (x // 5) + 1200 * (y // 6) + 40 * ((x + 2 * y) // 7 % 3)
    elif kind == "sky":
        d = np.rint(600 + 9000 * (1 - y / H) ** 3 + x)
        d[: H // 3] = 65535
    elif kind == "zeros":
        d = 2000 + rng.integers(0, 30, (H, W))
        d[rng.random((H, W)) < 0.2] = 0
    elif kind == "constant":
        d = np.full((H, W), 1234)
    elif kind == "road":         # KITTI-like: 655.35 m sky band, a road receding to the horizon, boxes, a few holes
        horizon = 140
        d = np.where(y < horizon, 65535, np.rint(150000.0 / np.maximum(y - horizon + 6, 1)))
        for (r0, r1, c0, c1, cm) in ((170, 260, 200, 420, 2300), (180, 240, 800, 950, 3400), (150, 200, 1000, 1180, 5200)):
            d[r0:r1, c0:c1] = cm + (x[r0:r1, c0:c1] - c0) // 3
        d[rng.random((H, W)) < 0.001] = 0
    elif kind == "ramp_noise":
        d = 2000 + x + y // 2 + rng.integers(0, 8, (H, W))
    else:
        raise KeyError(name)
    return np.clip(d, 0, 65535).astype(np.uint16)


SMALL = ("random", "random_narrow", "smooth", "planes", "steps", "sky", "zeros", "constant", "tiny_3x3", "tiny_3x4",
         "tiny_4x3", "tiny_5x7")
FULL_CASES = ("full_road", "full_smooth", "full_planes", "full_ramp_noise")
# (scene, variant, camera) of each case: the small maps sit in variants the training loader does not read, the
# full-size frames in ones it does
_LAYOUT = {**{c: ("Scene01", "clone", "Camera_0") for c in SMALL[:4]},
           **{c: ("Scene02", "15-deg-left", "Camera_1") for c in SMALL[4:8]},
           **{c: ("Scene20", "30-deg-right", "Camera_0") for c in SMALL[8:]},
           "full_road": ("Scene01", "morning", "Camera_0"), "full_smooth": ("Scene01", "morning", "Camera_0"),
           "full_planes": ("Scene06", "fog", "Camera_1"), "full_ramp_noise": ("Scene18", "overcast", "Camera_0")}


def write_normals_tree(root):
    """The synthetic Virtual KITTI 2 tree under `root`: one rgb JPEG and one 16-bit depth PNG per case, plus things the
    walk must skip (a non-.jpg file, an rgb directory without depths, a variant outside the ten).  Returns {case:
    (depth path, normal path)} relative to root."""
    import cv2
    files = {}
    for i, case in enumerate(SMALL + FULL_CASES):
        scene, variant, cam = _LAYOUT[case]
        d = case_depth(case)
        stem = f"_{i:05d}"
        rgb_dir = os.path.join(root, "vkitti_2.0.3_rgb", scene, variant, "frames", "rgb", cam)
        depth_dir = os.path.join(root, "vkitti_2.0.3_depth", scene, variant, "frames", "depth", cam)
        os.makedirs(rgb_dir, exist_ok=True)
        os.makedirs(depth_dir, exist_ok=True)
        rgb = np.stack([(d >> 8).astype(np.uint8), (d & 255).astype(np.uint8), np.full(d.shape, 90, np.uint8)], axis=2)
        assert cv2.imwrite(os.path.join(rgb_dir, f"rgb{stem}.jpg"), rgb)
        assert cv2.imwrite(os.path.join(depth_dir, f"depth{stem}.png"), d)
        files[case] = (os.path.join("vkitti_2.0.3_depth", scene, variant, "frames", "depth", cam, f"depth{stem}.png"),
                       os.path.join("vkitti_DAG_normals", scene, variant, "frames", "normal", cam, f"normal{stem}.png"))
    open(os.path.join(root, "vkitti_2.0.3_rgb", "Scene01", "clone", "frames", "rgb", "Camera_0", "notes.txt"), "w").close()
    os.makedirs(os.path.join(root, "vkitti_2.0.3_rgb", "Scene06", "rain", "frames", "rgb", "Camera_0"))
    open(os.path.join(root, "vkitti_2.0.3_rgb", "Scene06", "rain", "frames", "rgb", "Camera_0", "rgb_00099.jpg"),
         "wb").close()
    for sub in ("vkitti_2.0.3_rgb", "vkitti_2.0.3_depth"):
        kind = "rgb" if sub.endswith("rgb") else "depth"
        os.makedirs(os.path.join(root, sub, "Scene01", "sunny", "frames", kind, "Camera_0"))
    return files


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _run_script(script, pinned):
    original = np.power

    def power(base, expo, *a, **k):
        if isinstance(base, float) and base == np.e and isinstance(expo, np.ndarray) and expo.dtype == np.float32:
            return oracle.pow_e32_neg(-expo)
        return original(base, expo, *a, **k)
    np.power = power if pinned else original
    try:
        g = runpy.run_path(script, run_name="__main__")
    finally:
        np.power = original
    return g["dataset"].pairs


def main(ref):
    import cv2
    script = os.path.join(os.path.abspath(ref), "depth-to-normal-translator", "python", "gen_vkitti_normals.py")
    sys.path.insert(0, os.path.dirname(script))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            files = write_normals_tree(ROOT)
            outs = {}
            for pinned in (False, True):
                pairs = _run_script(script, pinned)
                outs[pinned] = {c: cv2.imread(os.path.join(ROOT, n), cv2.IMREAD_UNCHANGED) for c, (_, n) in files.items()}
        finally:
            os.chdir(cwd)
    rel = [tuple(os.path.relpath(p, ROOT) for p in t) for t in pairs]
    cases = SMALL + FULL_CASES
    pins = {"cases": np.array(cases), "pairs": np.array(rel)}
    diff = []
    for i, c in enumerate(cases):
        a, b = outs[True][c], outs[False][c]
        assert a.dtype == np.uint16 and a.shape == case_depth(c).shape + (3,), (c, a.dtype, a.shape)
        got = oracle.normals_frame(case_depth(c))
        print(f"{c:16s} {a.shape}  oracle == pinned reference: {np.array_equal(got, a)}  "
              f"unpinned differs at {int((a != b).sum())}")
        pins[f"depth_sha/{c}"] = np.array(sha256(case_depth(c)))
        pins[f"out_sha/{c}"] = np.array(sha256(a))
        if c in SMALL:
            pins[f"depth/{c}"] = case_depth(c)
            pins[f"out/{c}"] = a
        for y, x, ch in zip(*np.nonzero(a != b)):
            diff.append((i, y, x, ch, int(b[y, x, ch]), int(a[y, x, ch])))
    pins["unpinned_diff"] = np.array(diff, np.int64).reshape(-1, 6)   # case, y, x, channel, unpinned, pinned
    np.savez_compressed(OUT, **pins)
    print(f"{OUT}: {os.path.getsize(OUT)} bytes, {len(diff)} unpinned differences")


if __name__ == "__main__":
    main(sys.argv[1])
