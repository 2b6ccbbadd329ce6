"""Test oracle of the training-input transforms: training/dataloaders/load.py restated in numpy, PIL and torch, from
the decoded arrays a `diffusion_e2e_ft_b200.data` sample holds to the reference's per-sample dict.  Tests only: the
product package never imports it (tests/test_training_data_cpu.py checks that)."""
import hashlib

import numpy as np
import torch
from PIL import Image

HYPERSIM_FOCAL = 886.81


def _to_tensor(img):
    """torchvision ToTensor of a PIL image: uint8 -> CHW fp32 / 255, mode F -> [1,H,W] fp32 unchanged."""
    a = np.array(img)
    if a.dtype == np.uint8:
        return torch.from_numpy(a).permute(2, 0, 1).contiguous().to(torch.float32).div(255)
    return torch.from_numpy(a.astype(np.float32, copy=True))[None]


def _hflip(img):
    return img.transpose(Image.FLIP_LEFT_RIGHT)


def _flip_images(rgb, depth, normal):
    rgb, depth, normal = _hflip(rgb), _hflip(depth), _hflip(normal)
    n = np.array(normal)
    n[:, :, 0] = 255 - n[:, :, 0]
    return rgb, depth, Image.fromarray(n)


def align_normals(normal, depth, H, W):
    """Hypersim.align_normals (load.py:190-215) with K = (886.81, 886.81, W/2, H/2)."""
    K = np.array([[HYPERSIM_FOCAL, 0, W / 2], [0, HYPERSIM_FOCAL, H / 2], [0, 0, 1]])
    inv_K = np.linalg.inv(K)
    y, x = np.meshgrid(np.arange(0, H, dtype=np.float64), np.arange(0, W, dtype=np.float64), indexing="ij")
    xy = np.concatenate([np.stack((x, y)).reshape(2, -1), np.ones((1, H * W), dtype=np.float64)], axis=0)
    points = (depth * np.matmul(inv_K[:3, :3], xy).reshape(3, H, W)).transpose((1, 2, 0))
    orient = np.sum(normal * points, axis=2) > 0
    normal[orient] *= -1
    return normal


def _finalise(rgb_t, depth_t, normal_t, near, far, domain):
    """load.py:248-281 (= :343-376)."""
    valid = (depth_t > near) & (depth_t < far)
    rgb_t = rgb_t * 2.0 - 1.0
    if valid.any():
        flat = depth_t[valid].flatten().float()
        lo, hi = torch.quantile(flat, 0.02), torch.quantile(flat, 0.98)
        if lo == hi:
            depth_t = torch.zeros_like(depth_t)
            metric = torch.zeros_like(depth_t)
            valid = torch.zeros_like(depth_t).bool()
        else:
            depth_t = torch.clamp(depth_t, lo, hi)
            depth_t[~valid] = hi
            metric = depth_t.clone()
            depth_t = torch.clamp((((depth_t - lo) / (hi - lo)) * 2.0) - 1.0, -1, 1)
    else:
        depth_t = torch.zeros_like(depth_t)
        metric = torch.zeros_like(depth_t)
    depth_t = torch.stack([depth_t, depth_t, depth_t]).squeeze()
    normal_t = normal_t * 2.0 - 1.0
    normal_t = torch.nn.functional.normalize(normal_t, p=2, dim=0)
    for c in range(3):
        normal_t[c, ~valid.squeeze()] = 0
    return {"rgb": rgb_t, "depth": depth_t, "metric": metric, "normals": normal_t, "val_mask": valid, "domain": domain}


def hypersim_sample(rgb, depth_mm, normal, flip, size=(480, 640), transform=True, near=1e-5, far=65.0):
    """Hypersim.__getitem__ from decoded arrays: rgb uint8 [H,W,3], depth_mm uint16 [H,W], normal uint8 [H,W,3]."""
    rgb_img = Image.fromarray(rgb)
    depth_img = Image.fromarray(depth_mm / 1000)
    n = (np.array(normal) / 255.0) * 2.0 - 1.0
    H, W = n.shape[:2]
    n[:, :, 1:] *= -1
    n = align_normals(n, np.array(depth_img), H, W) * -1
    normal_img = Image.fromarray(((n + 1.0) / 2.0 * 255).astype(np.uint8))
    if transform:
        if flip:
            rgb_img, depth_img, normal_img = _flip_images(rgb_img, depth_img, normal_img)
        h, w = size
        rgb_img = rgb_img.resize((w, h), Image.BILINEAR)
        depth_img = depth_img.resize((w, h), Image.NEAREST)
        normal_img = normal_img.resize((w, h), Image.BILINEAR)
    return _finalise(_to_tensor(rgb_img), _to_tensor(depth_img), _to_tensor(normal_img), near, far, "indoor")


def kitti_benchmark_crop(t):
    h, w = t.shape[-2:]
    top, left = int(h - 352), int((w - 1216) / 2)
    return t[..., top:top + 352, left:left + 1216]


def vkitti_sample(rgb, depth_cm, normal, flip, transform=True, near=1e-5, far=80.0):
    """VirtualKITTI2.__getitem__ from decoded arrays: rgb uint8 [H,W,3], depth_cm uint16 [H,W], normal uint8 [H,W,3]."""
    rgb_img = Image.fromarray(rgb)
    depth_img = Image.fromarray(depth_cm.astype(np.float32) / 100.0)
    normal_img = Image.fromarray(normal)
    if transform and flip:
        rgb_img, depth_img, normal_img = _flip_images(rgb_img, depth_img, normal_img)
    r, d, n = _to_tensor(rgb_img), _to_tensor(depth_img), _to_tensor(normal_img)
    if transform:
        r, d, n = kitti_benchmark_crop(r), kitti_benchmark_crop(d), kitti_benchmark_crop(n)
    return _finalise(r, d, n, near, far, "outdoor")


def sample_from_raw(raw, size=(480, 640)):
    """The oracle's output for one raw sample of diffusion_e2e_ft_b200.data.Hypersim / VirtualKITTI2."""
    args = (raw["rgb"].numpy(), raw["depth"].numpy(), raw["normals"].numpy(), raw["flip"])
    kw = dict(transform=raw["transform"], near=raw["near_plane"], far=raw["far_plane"])
    if raw["domain"] == "indoor":
        return hypersim_sample(*args, size=size, **kw)
    return vkitti_sample(*args, **kw)


def digests(sample):
    """SHA-256 of each output tensor's bytes (C order, little-endian; the mask as bytes)."""
    out = {}
    for k in ("rgb", "depth", "metric", "normals", "val_mask"):
        t = sample[k].detach().cpu().contiguous()
        a = t.numpy().astype(np.uint8 if t.dtype == torch.bool else np.dtype("<f4"))
        out[k] = hashlib.sha256(a.tobytes()).hexdigest()
    return out
