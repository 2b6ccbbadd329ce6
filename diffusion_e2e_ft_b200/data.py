"""Training inputs: the Hypersim and Virtual KITTI 2 datasets of training/dataloaders/load.py, with the per-sample
transforms on the device (DESIGN.md §3 "Training inputs").

    Hypersim, VirtualKITTI2   <- load.py:159-376; __getitem__ only decodes the files, with the reference's own calls
    MixedDataLoader           <- load.py:18-59
    prepare_batch             <- the rest of __getitem__ (load.py:74-98, :106-152, :187-281, :343-376) plus the
                                 `.to(device)` of the training loop, on a collated batch of one dataset
    vkitti_normals            <- depth-to-normal-translator/python/gen_vkitti_normals.py:97-136 (D2NT v3) on a batch
    generate_vkitti_normals   <- the whole of gen_vkitti_normals.py: vkitti_DAG_normals/ written from the depths
    hypersim_frames           <- Marigold's hypersim_util.tone_map and dist_2_depth (preprocess_hypersim.py) on a batch
    preprocess_hypersim       <- the whole of preprocess_hypersim.py: the PNGs, lists and CSVs Hypersim reads

A training loop keeps its DataLoaders and swaps `from dataloaders.load import *` for this module, then calls
`batch = prepare_batch(batch)` on every batch.  The returned dict has the keys, shapes and dtypes the reference's
collated samples have, and the same values bit for bit; the arithmetic runs in libb200_e2eft.so (csrc/data.cu).
"""
import collections
import ctypes
import math
import os
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from . import lib as _lib
from .ops import _ck, _p, _stream

HYPERSIM_SIZE = (480, 640)                 # SynchronizedTransform_Hyper(H=480, W=640), load.py:168
HYPERSIM_FOCAL = 886.81                    # load.py:237
KB_CROP = (352, 1216)                      # KITTI benchmark crop, load.py:110-111
HYPERSIM_CSV = os.path.join("data", "hypersim", "processed", "train", "filename_meta_train.csv")
VKITTI_SCENES = ("Scene01", "Scene02", "Scene06", "Scene18", "Scene20")
VKITTI_WEATHER = ("morning", "fog", "rain", "sunset", "overcast")
VKITTI_CAMERAS = ("Camera_0", "Camera_1")
# the ten variants gen_vkitti_normals.py:31 writes normals for (the training loader reads five of them)
VKITTI_NORMAL_VARIANTS = ("15-deg-left", "15-deg-right", "30-deg-left", "30-deg-right", "clone", "morning", "fog",
                          "rain", "sunset", "overcast")
# the Virtual KITTI 2 depth camera as gen_vkitti_normals.py:68-71 gives it (vkitti_2.0.3_textgt)
VKITTI_FX, VKITTI_FY, VKITTI_U0, VKITTI_V0 = 725.0087, 725.0087, 620.5, 187.0
_PB = 22                                   # Pillow's PRECISION_BITS for 8-bit resampling


# ------------------------------------------------------------------------------------ host tables
def pillow_bilinear_coeffs(in_size, out_size):
    """Pillow's BILINEAR coefficients for one axis (precompute_coeffs + normalize_coeffs_8bpc): (first source tap
    int32 [out], 22-bit integer weights int32 [out, ks]), weights computed in double with support max(scale, 1),
    normalised, then rounded half away from zero."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = fs
    ks = int(np.ceil(support)) * 2 + 1
    first = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, ks), np.int32)
    for o in range(out_size):
        center = (o + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - lo
        w = [max(0.0, 1.0 - abs((x + lo - center + 0.5) / fs)) for x in range(n)]
        total = sum(w)
        if total != 0.0:
            w = [v / total for v in w]
        first[o] = lo
        kk[o, :n] = [int(-0.5 + v * (1 << _PB)) if v < 0 else int(0.5 + v * (1 << _PB)) for v in w]
    return first, kk


def pillow_nearest_index(in_size, out_size):
    """Source index of each output of Pillow's NEAREST resize along one axis (ImagingScaleAffine): the coordinate
    s/2, s/2 + s, ... accumulated in double and truncated.  This is not floor((i + 0.5) * s)."""
    s = in_size / out_size
    x = s * 0.5
    idx = np.empty(out_size, np.int32)
    for i in range(out_size):
        idx[i] = int(x)
        x += s
    if idx[-1] >= in_size:
        raise ValueError(f"nearest index {idx[-1]} out of range for {in_size} -> {out_size}")
    return idx


def hypersim_inv_k(H, W):
    """The inverse intrinsics of Hypersim.align_normals (np.linalg.inv of the 3x3 K, f = 886.81, c = (W/2, H/2))."""
    K = np.array([[HYPERSIM_FOCAL, 0, W / 2], [0, HYPERSIM_FOCAL, H / 2], [0, 0, 1]])
    return np.ascontiguousarray(np.linalg.inv(K), dtype=np.float64)


_TABLES = {}


def _device_table(key, build, device):
    """Host-built int32 tables, copied to the device once per (key, device) without a host sync."""
    k = (key, str(device))
    if k not in _TABLES:
        _TABLES[k] = tuple(torch.from_numpy(np.ascontiguousarray(a, np.int32)).pin_memory().to(device, non_blocking=True)
                           for a in build())
    return _TABLES[k]


# ------------------------------------------------------------------------------------ datasets (decode only)
def _flip_draw(transform):
    """The flip of SynchronizedTransform_{Hyper,VKITTI}.__call__: one random.random() > 0.5 per sample when the
    transform is on.  A flipped sample also draws torch.rand(1) three times, as the three RandomHorizontalFlip(p=1)
    calls do, so the torch generator stays in step with the reference's."""
    if not transform:
        return False
    flip = random.random() > 0.5
    if flip:
        for _ in range(3):
            torch.rand(1)
    return flip


def _sample(rgb, depth, normals, flip, transform, near_plane, far_plane, domain):
    return {"rgb": torch.from_numpy(rgb), "depth": torch.from_numpy(depth), "normals": torch.from_numpy(normals),
            "flip": bool(flip), "transform": bool(transform), "near_plane": float(near_plane),
            "far_plane": float(far_plane), "domain": domain}


class Hypersim(Dataset):
    """load.py:159-281.  Samples are decoded only: rgb uint8 [H,W,3], depth uint16 [H,W] in mm, normals uint8
    [H,W,3] (camera-space preview PNG), plus the flip flag and the settings `prepare_batch` needs.  The file list is
    read from data/hypersim/processed/train/filename_meta_train.csv relative to the working directory, as the
    reference reads it."""

    def __init__(self, root_dir, transform=True, near_plane=1e-5, far_plane=65.0):
        self.root_dir = root_dir
        self.split_path = HYPERSIM_CSV
        self.near_plane = near_plane
        self.far_plane = far_plane
        self.transform = bool(transform)
        self.pairs = self._find_pairs()

    def _find_pairs(self):
        import pandas as pd
        df = pd.read_csv(self.split_path)
        train = os.path.join(self.root_dir, "train")
        head = os.path.split(train)[0]
        pairs = []
        for _, row in df.iterrows():
            if not (row["included_in_public_release"] and row["split_partition_name"] == "train"):
                continue
            rgb = os.path.join(train, row["rgb_path"])
            depth = os.path.join(train, row["depth_path"])
            normal = os.path.join(head, "normals", row["scene_name"], "images",
                                  f"scene_{row['camera_name']}_geometry_preview",
                                  f"frame.{str(row['frame_id']).zfill(4)}.normal_cam.png")
            if os.path.exists(rgb) and os.path.exists(depth) and os.path.exists(normal):
                pairs.append({"rgb_path": rgb, "depth_path": depth, "normal_path": normal})
        return pairs

    def __len__(self):
        return len(self.pairs)

    def __getitem__(self, idx):
        from PIL import Image
        p = self.pairs[idx]
        rgb = np.array(Image.open(p["rgb_path"]).convert("RGB"))
        depth = np.array(Image.open(p["depth_path"]))
        if depth.dtype != np.uint16:
            depth = depth.astype(np.uint16)          # 16-bit PNGs open as mode I;16 (uint16) or I (int32)
        normals = np.array(Image.open(p["normal_path"]).convert("RGB"))
        return _sample(rgb, depth, normals, _flip_draw(self.transform), self.transform, self.near_plane,
                       self.far_plane, "indoor")


class VirtualKITTI2(Dataset):
    """load.py:284-376.  Samples are decoded only: rgb uint8 [H,W,3], depth uint16 [H,W] in cm, normals uint8
    [H,W,3] (the 16-bit D2NT normal PNG through PIL's convert('RGB'), which keeps the high byte), plus the flip flag
    and the settings `prepare_batch` needs."""

    def __init__(self, root_dir, transform=None, near_plane=1e-5, far_plane=80.0):
        self.root_dir = root_dir
        self.near_plane = near_plane
        self.far_plane = far_plane
        self.transform = bool(transform)
        self.pairs = self._find_pairs()

    def _find_pairs(self, variants=VKITTI_WEATHER):
        rgb_root = os.path.join(self.root_dir, "vkitti_2.0.3_rgb")
        depth_root = os.path.join(self.root_dir, "vkitti_2.0.3_depth")
        normal_root = os.path.join(self.root_dir, "vkitti_DAG_normals")
        pairs = []
        for scene in VKITTI_SCENES:
            for weather in variants:
                for camera in VKITTI_CAMERAS:
                    rgb_dir = os.path.join(rgb_root, scene, weather, "frames", "rgb", camera)
                    depth_dir = os.path.join(depth_root, scene, weather, "frames", "depth", camera)
                    normal_dir = os.path.join(normal_root, scene, weather, "frames", "normal", camera)
                    if not (os.path.exists(rgb_dir) and os.path.exists(depth_dir)):
                        continue
                    for f in os.listdir(rgb_dir):          # directory order, as the reference lists it
                        if not f.endswith(".jpg"):
                            continue
                        stem = f[3:]
                        pairs.append((os.path.join(rgb_dir, "rgb" + stem),
                                      os.path.join(depth_dir, "depth" + stem.replace(".jpg", ".png")),
                                      os.path.join(normal_dir, "normal" + stem.replace(".jpg", ".png"))))
        return pairs

    def __len__(self):
        return len(self.pairs)

    def __getitem__(self, idx):
        import cv2
        from PIL import Image
        rgb_path, depth_path, normal_path = self.pairs[idx]
        rgb = np.array(Image.open(rgb_path).convert("RGB"))
        depth = cv2.imread(depth_path, cv2.IMREAD_ANYCOLOR | cv2.IMREAD_ANYDEPTH)
        if depth is None or depth.dtype != np.uint16 or depth.ndim != 2:
            raise ValueError(f"{depth_path}: expected a single-channel 16-bit PNG")
        normals = np.array(Image.open(normal_path).convert("RGB"))
        return _sample(rgb, depth, normals, _flip_draw(self.transform), self.transform, self.near_plane,
                       self.far_plane, "outdoor")


class MixedDataLoader:
    """load.py:18-59: draws each batch from loader1 or loader2 in a shuffled order that takes split1 : split2 of
    them, capped at what each loader holds."""

    def __init__(self, loader1, loader2, split1=9, split2=1):
        self.loader1 = loader1
        self.loader2 = loader2
        self.split1 = split1
        self.split2 = split2
        self.frac1, self.frac2 = self.get_split_fractions()
        self.randchoice1 = None

    def get_split_fractions(self):
        size1, size2 = len(self.loader1), len(self.loader2)
        return (min((size2 / size1) * (self.split1 / self.split2), 1),
                min((size1 / size2) * (self.split2 / self.split1), 1))

    def create_split(self):
        choice = [True] * int(len(self.loader1) * self.frac1) + [False] * int(len(self.loader2) * self.frac2)
        np.random.shuffle(choice)
        return choice

    def __iter__(self):
        self.loader_iter1 = iter(self.loader1)
        self.loader_iter2 = iter(self.loader2)
        self.randchoice1 = self.create_split()
        self.indx = 0
        return self

    def __next__(self):
        if self.indx == len(self.randchoice1):
            raise StopIteration
        first = self.randchoice1[self.indx]
        self.indx += 1
        return next(self.loader_iter1) if first else next(self.loader_iter2)

    def __len__(self):
        return int(len(self.loader1) * self.frac1) + int(len(self.loader2) * self.frac2)


# ------------------------------------------------------------------------------------ device transforms
def _one_value(batch, key):
    v = batch[key]
    vals = v.tolist() if isinstance(v, torch.Tensor) else list(v) if isinstance(v, (list, tuple)) else [v]
    if not vals or any(x != vals[0] for x in vals):
        raise ValueError(f"batch[{key!r}] must hold one value for the whole batch, got {vals}")
    return vals[0]


def _check_batch(batch, device):
    if not isinstance(batch, dict):
        raise ValueError(f"prepare_batch takes a collated sample dict, got {type(batch).__name__}")
    missing = [k for k in ("rgb", "depth", "normals", "flip", "transform", "near_plane", "far_plane", "domain")
               if k not in batch]
    if missing:
        raise ValueError(f"batch is missing {missing}")
    rgb, depth, normals = batch["rgb"], batch["depth"], batch["normals"]
    for name, t, dt, nd in (("rgb", rgb, torch.uint8, 4), ("depth", depth, torch.uint16, 3),
                            ("normals", normals, torch.uint8, 4)):
        if not isinstance(t, torch.Tensor) or t.dtype != dt or t.dim() != nd:
            raise ValueError(f"batch[{name!r}] must be a {nd}-d {dt} tensor, got "
                             f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__} "
                             f"{tuple(t.shape) if isinstance(t, torch.Tensor) else ''}")
    B, H, W = depth.shape
    if B < 1 or H < 1 or W < 1 or rgb.shape != (B, H, W, 3) or normals.shape != (B, H, W, 3):
        raise ValueError(f"rgb / normals must be [B,H,W,3] with depth [B,H,W]: got {tuple(rgb.shape)}, "
                         f"{tuple(normals.shape)}, {tuple(depth.shape)}")
    flip = batch["flip"]
    if not isinstance(flip, torch.Tensor) or flip.dtype != torch.bool or tuple(flip.shape) != (B,):
        raise ValueError(f"batch['flip'] must be a bool tensor [{B}]")
    domain = _one_value(batch, "domain")
    if domain not in ("indoor", "outdoor") or len(batch["domain"]) != B:
        raise ValueError(f"batch['domain'] must be {B} x 'indoor' (Hypersim) or 'outdoor' (Virtual KITTI 2)")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()) \
        if torch.cuda.is_available() else None
    if dev is None or dev.type != "cuda":
        raise ValueError(f"prepare_batch runs on a CUDA device (no CPU fallback), got {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    for name in ("rgb", "depth", "normals", "flip"):
        t = batch[name]
        if t.device.type not in ("cpu", "cuda") or (t.is_cuda and t.device != dev):
            raise ValueError(f"batch[{name!r}] is on {t.device}, prepare_batch targets {dev}")
    near, far = float(_one_value(batch, "near_plane")), float(_one_value(batch, "far_plane"))
    if not (0.0 <= near < far):
        raise ValueError(f"need 0 <= near_plane < far_plane, got {near}, {far}")
    transform = bool(_one_value(batch, "transform"))
    if domain == "outdoor" and transform and (H < KB_CROP[0] or W < KB_CROP[1]):
        raise ValueError(f"Virtual KITTI 2 images of {H}x{W} are smaller than the {KB_CROP[0]}x{KB_CROP[1]} crop")
    return dev, domain, transform, near, far


def prepare_batch(batch, device=None):
    """A collated raw batch of one dataset (Hypersim or VirtualKITTI2) -> the dict the reference's collate returns, on
    the device: rgb [B,3,H,W], depth [B,3,H,W] (in [-1, 1]), metric [B,1,H,W], normals [B,3,H,W] (all fp32), val_mask
    [B,1,H,W] bool and domain (a list of "indoor" / "outdoor").  H x W is 480 x 640 for Hypersim and 352 x 1216 for
    Virtual KITTI 2 when the dataset's transform is on, else the decoded size.  The raw tensors are copied to `device`
    (default: the current CUDA device) without blocking; pin them (DataLoader(pin_memory=True)) for an asynchronous
    copy.  The copies, the kernels and the outputs are on `device` whether or not it is the current device.  The
    per-sample settings (transform, near_plane, far_plane, domain) are read on the host: leave them on the CPU, as the
    DataLoader collates them.  Shape, dtype and device errors raise ValueError before anything is launched; nothing
    syncs the host."""
    return _prepare(batch, device, HYPERSIM_SIZE)


def _prepare(batch, device, hypersim_size):
    dev, domain, transform, near, far = _check_batch(batch, device)
    with torch.cuda.device(dev):                     # the stream, the launches and the table uploads target `dev`
        return _launch(batch, dev, domain, transform, near, far, hypersim_size)


def _launch(batch, dev, domain, transform, near, far, hypersim_size):
    L = _lib.load()
    B, H, W = batch["depth"].shape
    rgb, depth, normals = (batch[k].to(dev, non_blocking=True).contiguous() for k in ("rgb", "depth", "normals"))
    flip = batch["flip"].to(dev, non_blocking=True).contiguous().view(torch.uint8) if transform else None
    st = _stream()
    if domain == "indoor":
        OH, OW = hypersim_size if transform else (H, W)
        resize = (OH, OW) != (H, W)                  # Pillow returns a copy at the same size
        # a resized sample gets its flip correction here and its mirror from the resize; otherwise the finalise
        # applies both, as for Virtual KITTI 2
        ik = hypersim_inv_k(H, W).reshape(-1)
        depth_m = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        aligned = torch.empty_like(normals)
        _ck(L.b200_data_hypersim_source(_p(depth), _p(normals), _p(flip if resize else None), B, H, W,
                                        (ctypes.c_double * 9)(*ik.tolist()), _p(depth_m), _p(aligned), st),
            "b200_data_hypersim_source")
        rows, cols = _device_table(("nearest", H, W, OH, OW), lambda: (pillow_nearest_index(H, OH),
                                                                        pillow_nearest_index(W, OW)), dev)
        src_m, src_cm, top, left, img_H, img_W, img_flip = depth_m, None, 0, 0, H, W, flip
        if resize:
            xmin, xk, ymin, yk = _device_table(("bilinear", H, W, OH, OW),
                                               lambda: (*pillow_bilinear_coeffs(W, OW), *pillow_bilinear_coeffs(H, OH)),
                                               dev)
            tmp = torch.empty((B, H, OW, 3), dtype=torch.uint8, device=dev)
            out_u8 = []
            for src in (rgb, aligned):
                dst = torch.empty((B, OH, OW, 3), dtype=torch.uint8, device=dev)
                _ck(L.b200_data_resize_u8(_p(src), B, H, W, 3, OH, OW, _p(xmin), _p(xk), xk.shape[1], _p(ymin), _p(yk),
                                          yk.shape[1], _p(flip), _p(tmp), _p(dst), st), "b200_data_resize_u8")
                out_u8.append(dst)
            rgb, aligned = out_u8
            img_H, img_W, img_flip = OH, OW, None
        norm_img = aligned
    else:
        OH, OW = KB_CROP if transform else (H, W)
        top, left = H - OH, (W - OW) // 2
        rows, cols = _device_table(("crop", H, W, OH, OW), lambda: (np.arange(top, top + OH), np.arange(left, left + OW)),
                                   dev)
        src_m, src_cm, img_flip, img_H, img_W, norm_img = None, depth, flip, H, W, normals
    d = torch.empty((B, OH, OW), dtype=torch.float32, device=dev)
    _ck(L.b200_data_depth_gather(_p(src_m), _p(src_cm), B, H, W, OH, OW, _p(rows), _p(cols), _p(flip), _p(d), st),
        "b200_data_depth_gather")
    rng = torch.empty((B, 2), dtype=torch.float32, device=dev)
    flag = torch.empty(B, dtype=torch.int32, device=dev)
    _ck(L.b200_data_depth_range(_p(d), B, OH * OW, near, far, _p(rng), _p(flag), st), "b200_data_depth_range")
    out = {k: torch.empty((B, c, OH, OW), dtype=torch.float32, device=dev)
           for k, c in (("rgb", 3), ("depth", 3), ("metric", 1), ("normals", 3))}
    mask = torch.empty((B, 1, OH, OW), dtype=torch.bool, device=dev)
    _ck(L.b200_data_finalise(_p(rgb), _p(norm_img), B, img_H, img_W, top, left, _p(img_flip), _p(d), OH, OW, near, far,
                             _p(rng), _p(flag), _p(out["rgb"]), _p(out["depth"]), _p(out["metric"]),
                             _p(out["normals"]), _p(mask), st), "b200_data_finalise")
    out["val_mask"] = mask
    out["domain"] = [domain] * B
    return out


# ------------------------------------------------------------------------------------ Virtual KITTI 2 normals
def vkitti_normals(depth_cm, fx=VKITTI_FX, fy=VKITTI_FY, u0=VKITTI_U0, v0=VKITTI_V0):
    """D2NT "v3" normals of gen_vkitti_normals.py:97-136 (DAG-filtered gradients, depth-to-normal translation, MRF
    refinement) for a uint16 [B,H,W] CUDA tensor of centimetre depths -> torch.uint16 [B,H,W,3] on the same device:
    uint16((-n + 1) * 32767.5) in the channel order the script hands cv2.imwrite (z, y, x; the file's RGB is x, y, z).
    The intrinsics are taken as float32, as the script's torch tensor holds them.  The result is bitwise the script's
    with its fp32 np.power(e, -lap) correctly rounded (DESIGN.md §3.11).  Runs under torch.cuda.device(depth.device)
    on its current stream without syncing the host; bad arguments raise ValueError before any launch."""
    if not isinstance(depth_cm, torch.Tensor) or depth_cm.dtype != torch.uint16 or depth_cm.dim() != 3:
        raise ValueError("vkitti_normals takes a uint16 [B,H,W] tensor of centimetre depths, got "
                         f"{depth_cm.dtype if isinstance(depth_cm, torch.Tensor) else type(depth_cm).__name__} "
                         f"{tuple(depth_cm.shape) if isinstance(depth_cm, torch.Tensor) else ''}")
    if not depth_cm.is_cuda:
        raise ValueError(f"vkitti_normals runs on a CUDA device (no CPU fallback), got {depth_cm.device}")
    B, H, W = depth_cm.shape
    if not (1 <= B <= 65535 and H >= 3 and W >= 3):
        raise ValueError(f"vkitti_normals needs 1 <= B <= 65535 and H, W >= 3, got {tuple(depth_cm.shape)}")
    cam = [float(v) for v in (fx, fy, u0, v0)]
    with np.errstate(over="ignore"):
        finite = all(math.isfinite(v) and np.isfinite(np.float32(v)) for v in cam)
    if not finite:
        raise ValueError(f"vkitti_normals needs finite intrinsics, got fx, fy, u0, v0 = {cam}")
    with torch.cuda.device(depth_cm.device):
        L = _lib.load()
        depth = depth_cm.contiguous()
        out = torch.empty((B, H, W, 3), dtype=torch.uint16, device=depth.device)
        _ck(L.b200_data_vkitti_normals(_p(depth), B, H, W, *cam, _p(out), _stream()), "b200_data_vkitti_normals")
    return out


class _VKITTIDepthFrames(VirtualKITTI2):
    """The frames gen_vkitti_normals.py walks (its ten variants) as (normal path, uint16 depth [H,W]); decoded with the
    script's cv2.imread flags (:62)."""

    def __init__(self, root_dir):
        self.root_dir = root_dir
        self.pairs = self._find_pairs(VKITTI_NORMAL_VARIANTS)

    def __getitem__(self, idx):
        import cv2
        _, depth_path, normal_path = self.pairs[idx]
        depth = cv2.imread(depth_path, cv2.IMREAD_ANYCOLOR | cv2.IMREAD_ANYDEPTH)
        if depth is None or depth.dtype != np.uint16 or depth.ndim != 2:
            raise ValueError(f"{depth_path}: missing, or not a single-channel 16-bit PNG")
        return normal_path, torch.from_numpy(depth)


def _equal_size_batches(frames, batch_size):
    """Consecutive frames of one size and dtype, at most batch_size at a time: (keys, stacked [B,...]).  A frame is
    (key, tensor) or (key, tuple or list of tensors, as a DataLoader hands a tuple back); those are stacked member by
    member into a tuple, and such frames are of one size when every member's shape and dtype match."""
    keys, items = [], []

    def shape(x):
        return tuple((t.shape, t.dtype) for t in x) if isinstance(x, (tuple, list)) else (x.shape, x.dtype)

    def stack():
        if isinstance(items[0], (tuple, list)):
            return tuple(torch.stack(m) for m in zip(*items))
        return torch.stack(items)
    for key, item in frames:
        if items and (len(items) == batch_size or shape(item) != shape(items[0])):
            yield keys, stack()
            keys, items = [], []
        keys.append(key)
        items.append(item)
    if items:
        yield keys, stack()


def _normals_on_host(depth, dev):
    """uint16 depth [B,H,W] on the host -> its normals, computed on `dev`, as a uint16 [B,H,W,3] numpy array in
    ordinary host memory.  The copies go through pinned staging buffers that are released on return (the caching
    host allocator hands them to the next batch), so queued PNG writes never hold page-locked memory."""
    out = vkitti_normals(depth.pin_memory().to(dev, non_blocking=True))
    host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
    host.copy_(out, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return host.numpy().copy()


def _write_png(path, image):
    import cv2
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if not cv2.imwrite(path, image):
        raise OSError(f"cv2.imwrite could not write {path}")


def _bounded_writes(pool, jobs, write, max_pending, done=None):
    """Submit write(*job) to `pool` for each job in turn, with at most max_pending submitted and not yet finished:
    beyond that the oldest is waited for first.  `jobs` is consumed lazily, so a generator that computes its frames
    only computes the next batch once the queue has room, and host memory stays bounded however much slower writing is
    than computing.  Each result goes to done(result) in submission order.  Returns the number of jobs finished."""
    pending = collections.deque()
    finished = 0

    def finish():
        nonlocal finished
        r = pending.popleft().result()
        finished += 1
        if done is not None:
            done(r)
    for job in jobs:
        while len(pending) >= max_pending:
            finish()
        pending.append(pool.submit(write, *job))
    while pending:
        finish()
    return finished


def generate_vkitti_normals(root_dir, batch_size=8, num_workers=4, device=None):
    """What `python gen_vkitti_normals.py` does, on the device: for every frame of the script's walk over root_dir
    (5 scenes x 10 variants x 2 cameras), the D2NT v3 normals of vkitti_2.0.3_depth/.../depth_*.png written as a
    16-bit PNG to vkitti_DAG_normals/.../normal_*.png, the path VirtualKITTI2 reads.  DataLoader workers decode, runs of
    equal-size frames go through vkitti_normals batch_size at a time, and a pool of num_workers threads encodes and
    writes.  At most 2 * max(batch_size, num_workers) computed frames wait for their write at any time: the loop
    blocks on the oldest write beyond that, so host memory stays bounded however much slower encoding is than
    decoding.  Returns the number of frames written.  A missing or non-16-bit depth file raises ValueError naming it."""
    if batch_size < 1 or num_workers < 0:
        raise ValueError(f"need batch_size >= 1 and num_workers >= 0, got {batch_size}, {num_workers}")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()) \
        if torch.cuda.is_available() else None
    if dev is None or dev.type != "cuda":
        raise ValueError(f"generate_vkitti_normals runs on a CUDA device (no CPU fallback), got {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    frames = DataLoader(_VKITTIDepthFrames(root_dir), batch_size=None, shuffle=False, num_workers=num_workers)
    with torch.cuda.device(dev), ThreadPoolExecutor(max(1, num_workers)) as pool:
        jobs = ((p, n) for paths, depth in _equal_size_batches(frames, batch_size)
                for p, n in zip(paths, _normals_on_host(depth, dev)))
        return _bounded_writes(pool, jobs, _write_png, 2 * max(batch_size, num_workers))


# ------------------------------------------------------------------------------------ Hypersim preprocessing
HYPERSIM_SPLITS = ("train", "val", "test")
_HYPERSIM_HALF = {torch.float16: 1, torch.float32: 0}
_TONE_MAP_NUM = None


class HypersimEntityIdError(ValueError):
    """A frame holds render_entity_id 0, which preprocess_hypersim.py asserts against.  `frames` lists the batch
    positions of the offending frames."""

    def __init__(self, message, frames):
        super().__init__(message)
        self.frames = list(frames)


def _tone_map_numerator():
    """hypersim_util.tone_map's np.power(0.8, inv_gamma), inv_gamma = 1.0 / (1.0 / 2.2), correctly rounded."""
    global _TONE_MAP_NUM
    if _TONE_MAP_NUM is None:
        from decimal import Decimal, localcontext
        with localcontext() as c:
            c.prec = 60
            _TONE_MAP_NUM = float((Decimal(1.0 / (1.0 / 2.2)) * Decimal(0.8).ln()).exp())
    return _TONE_MAP_NUM


def _check_hypersim_frames(rgb, dist, entity_id, focal):
    def desc(t):
        return f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
    for name, t, dts, nd in (("rgb", rgb, _HYPERSIM_HALF, 4), ("dist", dist, _HYPERSIM_HALF, 3),
                             ("entity_id", entity_id, (torch.int32,), 3)):
        if not isinstance(t, torch.Tensor) or t.dtype not in dts or t.dim() != nd:
            raise ValueError(f"hypersim_frames: {name} must be a {nd}-d {' or '.join(map(str, dts))} tensor, "
                             f"got {desc(t)}")
        if not t.is_cuda:
            raise ValueError(f"hypersim_frames runs on a CUDA device (no CPU fallback), got {name} on {t.device}")
    B, H, W = dist.shape
    if tuple(rgb.shape) != (B, H, W, 3) or tuple(entity_id.shape) != (B, H, W):
        raise ValueError(f"hypersim_frames needs rgb [B,H,W,3], dist and entity_id [B,H,W]: got {tuple(rgb.shape)}, "
                         f"{tuple(dist.shape)}, {tuple(entity_id.shape)}")
    if not (1 <= B <= 65535 and 1 <= H < 2 ** 23 and 1 <= W < 2 ** 23):
        raise ValueError(f"hypersim_frames needs 1 <= B <= 65535 and 1 <= H, W < 2^23, got {tuple(dist.shape)}")
    if rgb.device != dist.device or entity_id.device != dist.device:
        raise ValueError(f"hypersim_frames: rgb, dist and entity_id on different devices: {rgb.device}, "
                         f"{dist.device}, {entity_id.device}")
    focal = float(focal)
    with np.errstate(over="ignore"):
        if not (math.isfinite(focal) and np.isfinite(np.float32(focal))):
            raise ValueError(f"hypersim_frames needs a finite focal length, got {focal}")
    return focal


def hypersim_frames(rgb, dist, entity_id, focal=HYPERSIM_FOCAL):
    """Tone mapping and plane depth of preprocess_hypersim.py for B frames on the device: radiance rgb [B,H,W,3] and
    distance-from-camera-centre dist [B,H,W] (float16 or float32, taken exactly to fp64 as the script's
    astype(float)), render_entity_id [B,H,W] int32 -> (bgr, depth): bgr uint8 [B,H,W,3] is hypersim_util.tone_map
    times 255, truncated, in the order the script hands cv2.imwrite (B, G, R); depth uint16 [B,H,W] is dist_2_depth
    in millimetres, 0 where entity id == -1, through NumPy's wrapping cast (plane depths past 65.535 m wrap, as the
    script's do).  focal is the script's FOCAL_LENGTH; H and W are the tensors' (the script hard-codes 768 x 1024).
    Bitwise the script's output with its np.power correctly rounded (DESIGN.md §3.12).  Runs under
    torch.cuda.device(rgb.device) on its current stream.  An entity id of 0, which the script asserts against, raises
    HypersimEntityIdError (a ValueError) whose `frames` are the offending batch positions; reading that flag back is
    the call's one host sync.  Bad arguments raise ValueError before any launch."""
    focal = _check_hypersim_frames(rgb, dist, entity_id, focal)
    B, H, W = dist.shape
    with torch.cuda.device(rgb.device):
        L = _lib.load()
        rgb_c, dist_c, eid = rgb.contiguous(), dist.contiguous(), entity_id.contiguous()
        bgr = torch.empty((B, H, W, 3), dtype=torch.uint8, device=rgb.device)
        depth = torch.empty((B, H, W), dtype=torch.uint16, device=rgb.device)
        err = torch.empty(B, dtype=torch.int32, device=rgb.device)
        nbytes = L.b200_data_hypersim_workspace_bytes(B, H, W)
        ws = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=rgb.device)
        _ck(L.b200_data_hypersim_frames(_p(rgb_c), _HYPERSIM_HALF[rgb.dtype], _p(dist_c), _HYPERSIM_HALF[dist.dtype],
                                        _p(eid), B, H, W, focal, _tone_map_numerator(), _p(bgr), _p(depth), _p(err),
                                        None, _p(ws), ws.numel() * 8, _stream()), "b200_data_hypersim_frames")
        bad = torch.nonzero(err.cpu()).flatten().tolist()
    if bad:
        raise HypersimEntityIdError(f"hypersim_frames: render_entity_id holds 0 in frame(s) {bad} (the reference "
                                    "asserts entity_id != 0)", bad)
    return bgr, depth


def _hypersim_paths(row):
    """preprocess_hypersim.py's input files of one metadata row (color, depth_meters, render_entity_id), relative to
    the dataset directory."""
    images = os.path.join(row.scene_name, "images")
    geo = os.path.join(images, f"scene_{row.camera_name}_geometry_hdf5")
    return (os.path.join(images, f"scene_{row.camera_name}_final_hdf5", f"frame.{row.frame_id:04d}.color.hdf5"),
            os.path.join(geo, f"frame.{row.frame_id:04d}.depth_meters.hdf5"),
            os.path.join(geo, f"frame.{row.frame_id:04d}.render_entity_id.hdf5"))


def _import_h5py():
    try:
        import h5py
    except ImportError as e:
        raise ImportError("preprocess_hypersim reads Hypersim's HDF5 renders with h5py: `pip install h5py`") from e
    return h5py


class _HypersimRawFrames(Dataset):
    """One split's frames as (metadata index, (rgb, dist, entity_id)) host tensors in the files' dtypes; decoded with
    h5py in DataLoader workers."""

    def __init__(self, dataset_dir, rows):
        self.dataset_dir = dataset_dir
        self.rows = rows                           # [(index, (color, depth_meters, render_entity_id) paths)]

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, idx):
        h5py = _import_h5py()
        i, paths = self.rows[idx]
        arrays = []
        for path, dts in zip(paths, (("float16", "float32"), ("float16", "float32"), ("int32",))):
            full = os.path.join(self.dataset_dir, path)
            with h5py.File(full, "r") as f:
                a = np.array(f["dataset"])
            if a.dtype.name not in dts:
                raise ValueError(f"{full}: expected {' or '.join(dts)} data, got {a.dtype}")
            arrays.append(torch.from_numpy(np.ascontiguousarray(a)))
        return i, tuple(arrays)


def _hypersim_on_host(rgb, dist, entity_id, focal, dev):
    """One batch of host tensors -> (bgr uint8 [B,H,W,3], depth uint16 [B,H,W]) as numpy arrays in ordinary host
    memory, computed on `dev` (the staging buffers are released on return, as in _normals_on_host)."""
    bgr, depth = hypersim_frames(*(t.pin_memory().to(dev, non_blocking=True) for t in (rgb, dist, entity_id)), focal)
    host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in (bgr, depth)]
    for h, t in zip(host, (bgr, depth)):
        h.copy_(t, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return tuple(h.numpy().copy() for h in host)


def _write_hypersim_frame(split_output_dir, i, rgb_path, depth_path, bgr, depth, valid_mask):
    """The PNG writes and the metadata of one frame, computed with the script's own NumPy calls on the same uint8 RGB
    and uint16 depth arrays."""
    _write_png(os.path.join(split_output_dir, rgb_path), bgr)
    _write_png(os.path.join(split_output_dir, depth_path), depth)
    rgb_int = np.ascontiguousarray(bgr[..., ::-1])
    restored_depth = depth / 1000.0
    invalid_ratio = (np.prod(valid_mask.shape) - valid_mask.sum()) / np.prod(valid_mask.shape)
    return i, {"rgb_path": rgb_path, "rgb_mean": np.mean(rgb_int), "rgb_std": np.std(rgb_int),
               "rgb_min": np.min(rgb_int), "rgb_max": np.max(rgb_int), "depth_path": depth_path,
               "depth_mean": np.mean(restored_depth), "depth_std": np.std(restored_depth),
               "depth_min": np.min(restored_depth), "depth_max": np.max(restored_depth),
               "invalid_ratio": invalid_ratio}


def preprocess_hypersim(split_csv, dataset_dir, output_dir, batch_size=8, num_workers=4, device=None):
    """What `python preprocess_hypersim.py --split_csv .. --dataset_dir .. --output_dir ..` does, on the device: for
    every included_in_public_release row of split_csv, split by split (train, val, test), the tone-mapped
    rgb_{camera}_fr{frame}.png and the 16-bit depth_plane_{camera}_fr{frame}.png under output_dir/{split}/{scene}/,
    then filename_list_{split}.txt and filename_meta_{split}.csv, byte for byte the script's files (with its
    np.power correctly rounded).  data.Hypersim reads output_dir as its root_dir.  DataLoader workers read the HDF5
    files with h5py, batches of up to batch_size frames go through hypersim_frames, and a pool of num_workers threads
    encodes, writes and computes each frame's metadata, with at most 2 * max(batch_size, num_workers) computed frames
    waiting at any time.  Returns the number of frames written.

    At the edges: an existing output_dir/{split} raises FileExistsError, as the script's os.makedirs does, but for
    all three splits before anything is written; a missing input file raises FileNotFoundError naming it (the script
    fails an assert), also before anything is written; an entity id of 0 raises ValueError naming the file (the
    script fails an assert); a split without rows gets an empty filename_list and a header-only CSV, where the script
    stops with an AttributeError."""
    import pandas as pd
    if batch_size < 1 or num_workers < 0:
        raise ValueError(f"need batch_size >= 1 and num_workers >= 0, got {batch_size}, {num_workers}")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()) \
        if torch.cuda.is_available() else None
    if dev is None or dev.type != "cuda":
        raise ValueError(f"preprocess_hypersim runs on a CUDA device (no CPU fallback), got {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    raw_meta_df = pd.read_csv(split_csv)
    meta_df = raw_meta_df[raw_meta_df.included_in_public_release].copy()
    for split in HYPERSIM_SPLITS:
        if os.path.exists(os.path.join(output_dir, split)):
            raise FileExistsError(f"{os.path.join(output_dir, split)} exists")
    plan = []
    for split in HYPERSIM_SPLITS:
        split_meta_df = meta_df[meta_df.split_partition_name == split].copy()
        rows = [(i, _hypersim_paths(row)) for i, row in split_meta_df.iterrows()]
        for _, paths in rows:
            for p in paths:
                if not os.path.exists(os.path.join(dataset_dir, p)):
                    raise FileNotFoundError(f"{os.path.join(dataset_dir, p)}: input file missing")
        plan.append((split, split_meta_df, rows))
    if any(rows for _, _, rows in plan):
        _import_h5py()
    written = 0
    with torch.cuda.device(dev), ThreadPoolExecutor(max(1, num_workers)) as pool:
        for split, split_meta_df, rows in plan:
            split_output_dir = os.path.join(output_dir, split)
            os.makedirs(split_output_dir)
            split_meta_df["rgb_path"] = None
            for col in ("rgb_mean", "rgb_std", "rgb_min", "rgb_max"):
                split_meta_df[col] = np.nan
            split_meta_df["depth_path"] = None
            for col in ("depth_mean", "depth_std", "depth_min", "depth_max", "invalid_ratio"):
                split_meta_df[col] = np.nan
            frames = DataLoader(_HypersimRawFrames(dataset_dir, rows), batch_size=None, shuffle=False,
                                num_workers=num_workers)
            paths = dict(rows)
            names = {i: (os.path.join(row.scene_name, f"rgb_{row.camera_name}_fr{row.frame_id:04d}.png"),
                         os.path.join(row.scene_name, f"depth_plane_{row.camera_name}_fr{row.frame_id:04d}.png"))
                     for i, row in split_meta_df.iterrows()}

            def jobs():
                for idx, (rgb, dist, eid) in _equal_size_batches(frames, batch_size):
                    try:
                        bgr, depth = _hypersim_on_host(rgb, dist, eid, HYPERSIM_FOCAL, dev)
                    except HypersimEntityIdError as e:
                        bad = [os.path.join(dataset_dir, paths[idx[k]][2]) for k in e.frames]
                        raise HypersimEntityIdError(f"render_entity_id holds 0 in {bad} (the reference asserts "
                                                    "entity_id != 0)", e.frames) from e
                    for i, b, d, e in zip(idx, bgr, depth, eid.numpy()):
                        yield (split_output_dir, i, *names[i], b, d, e != -1)

            def record(result):
                i, meta = result
                for k, v in meta.items():
                    split_meta_df.at[i, k] = v
            written += _bounded_writes(pool, jobs(), _write_hypersim_frame, 2 * max(batch_size, num_workers), record)
            with open(os.path.join(split_output_dir, f"filename_list_{split}.txt"), "w+") as f:
                if len(split_meta_df):
                    lines = split_meta_df.apply(lambda r: f"{r['rgb_path']} {r['depth_path']}", axis=1).tolist()
                    f.writelines("\n".join(lines))
            with open(os.path.join(split_output_dir, f"filename_meta_{split}.csv"), "w+") as f:
                split_meta_df.to_csv(f, header=True)
    return written
