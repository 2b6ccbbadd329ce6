"""Training inputs: the Hypersim and Virtual KITTI 2 datasets of training/dataloaders/load.py, with the per-sample
transforms on the device (DESIGN.md §3 "Training inputs").

    Hypersim, VirtualKITTI2   <- load.py:159-376; __getitem__ only decodes the files, with the reference's own calls
    MixedDataLoader           <- load.py:18-59
    prepare_batch             <- the rest of __getitem__ (load.py:74-98, :106-152, :187-281, :343-376) plus the
                                 `.to(device)` of the training loop, on a collated batch of one dataset

A training loop keeps its DataLoaders and swaps `from dataloaders.load import *` for this module, then calls
`batch = prepare_batch(batch)` on every batch.  The returned dict has the keys, shapes and dtypes the reference's
collated samples have, and the same values bit for bit; the arithmetic runs in libb200_e2eft.so (csrc/data.cu).
"""
import ctypes
import os
import random

import numpy as np
import torch
from torch.utils.data import Dataset

from . import lib as _lib
from .ops import _ck, _p, _stream

HYPERSIM_SIZE = (480, 640)                 # SynchronizedTransform_Hyper(H=480, W=640), load.py:168
HYPERSIM_FOCAL = 886.81                    # load.py:237
KB_CROP = (352, 1216)                      # KITTI benchmark crop, load.py:110-111
HYPERSIM_CSV = os.path.join("data", "hypersim", "processed", "train", "filename_meta_train.csv")
VKITTI_SCENES = ("Scene01", "Scene02", "Scene06", "Scene18", "Scene20")
VKITTI_WEATHER = ("morning", "fog", "rain", "sunset", "overcast")
VKITTI_CAMERAS = ("Camera_0", "Camera_1")
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

    def _find_pairs(self):
        rgb_root = os.path.join(self.root_dir, "vkitti_2.0.3_rgb")
        depth_root = os.path.join(self.root_dir, "vkitti_2.0.3_depth")
        normal_root = os.path.join(self.root_dir, "vkitti_DAG_normals")
        pairs = []
        for scene in VKITTI_SCENES:
            for weather in VKITTI_WEATHER:
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
