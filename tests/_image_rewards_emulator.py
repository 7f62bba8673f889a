"""TEST INFRASTRUCTURE: NumPy emulation of the image-reward ops (``ops.resample_u8``, ``clip_normalize_u8``,
``pair_stats_u8``, ``feature_angles``, ``scaled_cosine``; tests/_cpu_ops_emulator.py covers the other ops) so that the
host assembly of the rewards and the drivers dry-run on the CPU.  ``install(E)`` adds them to an emulator module."""
import numpy as np
import torch

from ddpo_b200 import clip_vision as CV


def transformed(a, transform):
    """numpy [B, H, W, 3] -> the transformed batch: ImageOps.mirror or Image.rotate(90 / 180 / 270) (square only)"""
    if transform in (CV.ROT90, CV.ROT270) and a.shape[1] != a.shape[2]:
        raise ValueError("rotate(90 / 270) needs a square image")
    return {CV.IDENTITY: a, CV.MIRROR: a[:, :, ::-1], CV.ROT90: np.rot90(a, 1, axes=(1, 2)),
            CV.ROT180: a[:, ::-1, ::-1], CV.ROT270: np.rot90(a, 3, axes=(1, 2))}[transform]


def resample_axis(a, axis, table):
    """one bicubic pass of the fixed-point table along ``axis`` of a uint8 array (Pillow's ImagingResampleHorizontal /
    Vertical_8bpc)"""
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    out = np.empty((table.shape[0],) + a.shape[1:], np.uint8)
    for i, row in enumerate(table):
        xmin, n = int(row[0]), int(row[1])
        acc = np.full(a.shape[1:], 1 << 21, np.int64)
        for j in range(n):
            acc += a[xmin + j] * int(row[2 + j])
        out[i] = np.clip(acc >> 22, 0, 255)
    return np.moveaxis(out, 0, axis)


def resample_u8(src, transform, axis, table_host, table_dev, dst):
    a = transformed(src.numpy(), transform)
    dst.copy_(torch.from_numpy(np.ascontiguousarray(resample_axis(a, 2 if axis == 0 else 1, table_host))))


def clip_normalize_u8(src, top, left, out):
    size = out.shape[1]
    q = src.numpy()[:, top:top + size, left:left + size].astype(np.float32) / np.float32(255)
    out.copy_(torch.from_numpy(((q.astype(np.float64) - CV.CLIP_MEAN) / CV.CLIP_STD).astype(np.float32)))


def pair_stats_u8(src, transform, out):
    assert transform in (CV.MIRROR, CV.ROT180)
    a = src.numpy()
    t = transformed(a, transform)
    n = len(a)
    a64, t64 = a.reshape(n, -1).astype(np.int64), t.reshape(n, -1).astype(np.int64)
    wrapped = ((a - t) ** 2).reshape(n, -1).astype(np.int64)           # numpy's uint8 wrap
    out.copy_(torch.from_numpy(np.stack([wrapped.sum(1), a64.sum(1), (a64 * a64).sum(1), (a64 * t64).sum(1)], 1)))


def _cos(x, y):
    return (x * y).sum(-1) / (np.sqrt((x * x).sum(-1)) * np.sqrt((y * y).sum(-1)))


def feature_angles(feats, variants, out):
    f = feats.double().numpy().reshape(variants, out.numel(), -1)
    ang = [np.degrees(np.arccos(np.clip(_cos(f[0], f[v]), 0, 1))) for v in range(1, variants)]
    out.copy_(torch.from_numpy(np.mean(ang, 0).astype(np.float32)))


def scaled_cosine(img, txt, logit_scale, out):
    s = float(np.exp(np.float32(logit_scale)))
    out.copy_(torch.from_numpy((s * _cos(img.double().numpy(), txt.double().numpy())).astype(np.float32)))


def install(emulator):
    for f in (resample_u8, clip_normalize_u8, pair_stats_u8, feature_angles, scaled_cosine):
        setattr(emulator, f.__name__, f)
