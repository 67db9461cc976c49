"""Homography-pretraining image pairs on the GPU.  Drop-in for the item of the reference's pretraining dataset

    data.oxford_paris_dataset.OxfordParis1MDataset.__getitem__      (data/oxford_paris_dataset.py:27-66)

batched as the default ``DataLoader`` collate batches it, from images the loader has already decoded and resized.  Per image: 4
random corner offsets, the homographies ``H_warp`` (full image) and ``H_true`` (between the two crops) by
``cv2.getPerspectiveTransform``, ``cv2.warpPerspective`` (INTER_LINEAR, constant-0 border), the crop by ``offset`` and
``cv2.cvtColor(RGB2GRAY) / 255``: ONE launch of ``og_homography_pairs`` (csrc/homography.cuh) for the whole batch, which computes
only the crop of the warped image.  Every output equals cv2's bit for bit (OpenCV's fixed-point arithmetic, restated), wherever
cv2's LU solve of the homography succeeds; on a degenerate corner configuration (a pivot below 100 DBL_EPSILON) the homography is
OpenCV's LU failure value [[0,0,0],[0,0,0],[0,0,1]], where cv2 4.13 falls back to an SVD.

Not done here: the JPEG decode and the INTER_AREA resize (host, before this), and the colour augmentation (random, between the
crop and the gray conversion in the reference; a caller that needs it keeps the reference loader).

CUDA tensors only, and no autograd.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _cabi
from ._cabi import ptr, stream

__all__ = ['synthesize_homography_pairs']


def synthesize_homography_pairs(images_u8: torch.Tensor, offset: int, warp_offset: Optional[torch.Tensor] = None,
                                generator: Optional[torch.Generator] = None) -> dict:
    """images_u8 [B, H, W, 3] uint8 RGB (CUDA) -> {'image0' [B,1,h,w] f32, 'image1' [B,1,h,w] f32,
    'transformation': {'type': ['perspective'] * B, 'H' [B,3,3] f32}} with h = H - 2 offset, w = W - 2 offset.

    ``warp_offset`` [B, 4, 2] integers in [-offset, offset): (x, y) of the corners (off, off), (off, H-off-1), (W-off-1, off),
    (W-off-1, H-off-1), in the reference's order; None draws them uniformly, as the reference's ``np.random.randint`` does, with
    ``torch.randint`` on ``generator``'s device (the images' device when None)."""
    B, H, W, offset = _check_images(images_u8, offset)
    if warp_offset is not None:
        if not torch.is_tensor(warp_offset) or warp_offset.dtype.is_floating_point or warp_offset.dtype.is_complex \
                or warp_offset.dtype == torch.bool:
            raise TypeError('warp_offset must be an integer tensor')
        if tuple(warp_offset.shape) != (B, 4, 2):
            raise ValueError(f'warp_offset must be [B, 4, 2] = {(B, 4, 2)}, got {tuple(warp_offset.shape)}')
        lo, hi = int(warp_offset.min()), int(warp_offset.max())
        if lo < -offset or hi >= offset:
            raise ValueError(f'warp_offset must lie in [-offset, offset) = [{-offset}, {offset}), got [{lo}, {hi}]')
    if images_u8.device.type != 'cuda':
        raise RuntimeError('openglue_b200: images_u8 must be a CUDA tensor (sm_90a); there is no CPU path')
    dev = images_u8.device
    if warp_offset is None:
        gdev = generator.device if generator is not None else dev
        warp_offset = torch.randint(-offset, offset, (B, 4, 2), generator=generator, device=gdev, dtype=torch.int32)
    return _pairs(images_u8, offset, warp_offset.to(device=dev, dtype=torch.int32).contiguous())


def _check_images(images_u8: torch.Tensor, offset: int):
    """-> (B, H, W, offset) of a valid images_u8 [B, H, W, 3] uint8 and offset; raises before any launch otherwise"""
    if not torch.is_tensor(images_u8) or images_u8.dtype != torch.uint8:
        raise TypeError(f'images_u8 must be a uint8 tensor, got {getattr(images_u8, "dtype", type(images_u8))}')
    if images_u8.dim() != 4 or images_u8.shape[3] != 3:
        raise ValueError(f'images_u8 must be [B, H, W, 3] RGB, got {tuple(images_u8.shape)}')
    B, H, W, _ = images_u8.shape
    if isinstance(offset, bool) or int(offset) != offset:
        raise TypeError(f'offset must be an integer, got {offset!r}')
    offset = int(offset)
    if B < 1 or B > 65535:
        raise ValueError(f'the batch must hold 1 .. 65535 images, got {B}')
    if offset < 1 or 2 * offset >= min(H, W):
        raise ValueError(f'offset must be >= 1 with 2 * offset < min(H, W) = {min(H, W)}, got {offset}')
    return B, H, W, offset


def _pairs(images_u8: torch.Tensor, offset: int, warp_offset: torch.Tensor) -> dict:
    """The launch of synthesize_homography_pairs on checked arguments (``warp_offset``: int32 [B, 4, 2] on the images' device,
    in range): no host synchronisation, so it can be captured in a CUDA graph."""
    B, H, W, _ = images_u8.shape
    dev = images_u8.device
    images_u8 = images_u8.detach().contiguous()
    h, w = H - 2 * offset, W - 2 * offset
    image0 = torch.empty(B, 1, h, w, dtype=torch.float32, device=dev)
    image1 = torch.empty(B, 1, h, w, dtype=torch.float32, device=dev)
    H_true = torch.empty(B, 3, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().og_homography_pairs(ptr(images_u8), B, H, W, offset, ptr(warp_offset), ptr(image0), ptr(image1),
                                                    ptr(H_true), stream(dev)), 'og_homography_pairs')
    return {'image0': image0, 'image1': image1, 'transformation': {'type': ['perspective'] * B, 'H': H_true}}
