"""Drop-in for the reference's default online features, ``SIFT`` (models/features/sift.py:16-49 on models/features/base.py:8-82):
kornia's DoG detector (``ScaleSpaceDetector`` with ``BlobDoG``, ``ConvQuadInterp3d(10)``, ``ScalePyramid(3, 1.6, 32,
double_image=True)``, ``LAFOrienter(19)``), the reference's ``run_nms`` and kornia's ``LAFDescriptor(SIFTDescriptor(41))`` with
RootSIFT, restated from kornia 0.6.3 and run on the GPU.

Every stage is a kernel of ``libopenglue_b200.so`` (``csrc/kornia_sift.cuh``): the scale-space pyramid, the extrema with their
quadratic interpolation and the per-octave and global top-k, ``run_nms``, and the orientation and descriptor of the selected
keypoints only (orientation does not change which keypoints ``run_nms`` keeps, so orienting after the selection gives the
reference's result for less work).  ``forward`` / ``extract_batch`` read the kept counts back to size their outputs;
``extract_padded`` writes a fixed capacity with the counts on the device and never synchronises.  There is no CPU path.

Order: descending response.  torch leaves the order of ties unspecified; here equal responses keep the lower index at every
top-k (voxel index within an octave, then octave, then per-octave rank), and ``run_nms``'s key sort puts equal keys in
detector order.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr, stream
from .features import padded_capacity

__all__ = ['SIFT']

MAX_FEATURES = 8192                 # keypoints per image the detector and run_nms sort in one CTA's shared memory


class SIFT(nn.Module):
    """``SIFT(descriptor_dim=128, max_keypoints=8000, perform_nms=True, nms_diameter=9, patch_size=41, upright=False,
    rootsift=True, device=cpu)``, the reference's constructor.  ``forward(images [B,1,H,W] float in [0, 1], or uint8 / 255)`` returns the
    reference's batch ``(lafs [B,N,2,3], responses [B,N], descriptors [B,N,128])``, N min-stacked over the batch as ``run_nms``
    does; ``extract_batch`` gives one such tuple per image and ``extract_padded`` a fixed capacity.  ``device`` is accepted for
    the reference's signature; the module follows the images' device."""

    def __init__(self, descriptor_dim: int = 128, max_keypoints: int = 8000, perform_nms: bool = True, nms_diameter: int = 9,
                 patch_size: int = 41, upright: bool = False, rootsift: bool = True, device=None):
        super().__init__()
        if int(descriptor_dim) != 128:
            raise ValueError(f'SIFT descriptors have 128 entries, got descriptor_dim={descriptor_dim}')
        if int(patch_size) != 41:
            raise ValueError(f'only patch_size=41 (the reference default) is supported, got {patch_size}')
        if not 1 <= int(max_keypoints) <= MAX_FEATURES:
            raise ValueError(f'max_keypoints must be in [1, {MAX_FEATURES}], got {max_keypoints}')
        if perform_nms and (int(nms_diameter) < 1 or int(nms_diameter) % 2 == 0):
            raise ValueError(f'nms_diameter must be a positive odd number, got {nms_diameter}')
        self.descriptor_dim, self.max_keypoints = 128, int(max_keypoints)
        self.perform_nms, self.nms_diameter = bool(perform_nms), int(nms_diameter)
        self.patch_size, self.upright, self.rootsift = 41, bool(upright), bool(rootsift)
        self._ws = {}

    def extra_repr(self) -> str:
        return (f'max_keypoints={self.max_keypoints}, perform_nms={self.perform_nms}, nms_diameter={self.nms_diameter}, '
                f'upright={self.upright}, rootsift={self.rootsift}')

    def _workspace(self, dev, B, H, W):
        lib = _cabi.lib()
        key = (dev, B, H, W)
        if key not in self._ws:
            while len(self._ws) >= 2:                                   # the two image sizes of a pair batch stay cached
                del self._ws[next(iter(self._ws))]
            n = _cabi.check_size(lib.og_ksift_workspace_bytes(B, H, W, self.max_keypoints), 'og_ksift_workspace_bytes')
            m = _cabi.check_size(lib.og_ksift_select_workspace_bytes(B, self.max_keypoints), 'og_ksift_select_workspace_bytes')
            self._ws[key] = (torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(m, dtype=torch.uint8, device=dev))
        return self._ws[key]

    @staticmethod
    def _image(images: torch.Tensor) -> torch.Tensor:
        if not torch.is_tensor(images) or images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f'images must be [B, 1, H, W], got {tuple(images.shape) if torch.is_tensor(images) else type(images)}')
        if images.device.type != 'cuda':
            raise RuntimeError('openglue_b200.SIFT needs CUDA tensors (sm_90a); there is no CPU path')
        if images.dtype == torch.uint8:
            return (images.float() / 255.).contiguous()
        if not images.is_floating_point():
            raise ValueError(f'images must be float in [0, 1] or uint8, got {images.dtype}')
        return images.detach().float().contiguous()

    def _detect_select(self, img: torch.Tensor, min_stack: bool):
        """The detector and run_nms of B images: (ws, det_lafs, det_resp, sel, n_sel)."""
        B, _, H, W = img.shape
        dev, k = img.device, self.max_keypoints
        lib = _cabi.lib()
        st = stream(dev)
        ws, work = self._workspace(dev, B, H, W)
        det_lafs = torch.empty(B, k, 2, 3, dtype=torch.float32, device=dev)
        det_resp = torch.empty(B, k, dtype=torch.float32, device=dev)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        _cabi.check(lib.og_ksift_pyramid(ptr(img), B, H, W, k, ptr(ws), ws.numel(), st), 'og_ksift_pyramid')
        _cabi.check(lib.og_ksift_detect(B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp), ptr(count), st), 'og_ksift_detect')
        sel = torch.empty(B, k, dtype=torch.int32, device=dev)
        n_sel = torch.empty(B, dtype=torch.int32, device=dev)
        _cabi.check(lib.og_ksift_select(ptr(det_lafs), ptr(det_resp), ptr(count), B, H, W, k, int(self.perform_nms), self.nms_diameter,
                                        self.max_keypoints, int(min_stack), ptr(work), work.numel(), ptr(sel), ptr(n_sel), st),
                    'og_ksift_select')
        return ws, det_lafs, det_resp, sel, n_sel

    def _describe(self, img, ws, det_lafs, det_resp, sel, n, out_cap):
        B, _, H, W = img.shape
        dev = img.device
        f32 = dict(dtype=torch.float32, device=dev)
        lafs, scores, desc = torch.empty(B, out_cap, 2, 3, **f32), torch.empty(B, out_cap, **f32), torch.empty(B, out_cap, 128, **f32)
        _cabi.check(_cabi.lib().og_ksift_describe(ptr(img), B, H, W, self.max_keypoints, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp),
                                                  self.max_keypoints, ptr(sel), ptr(n), out_cap, int(self.upright), int(self.rootsift),
                                                  ptr(lafs), ptr(scores), ptr(desc), None, stream(dev)), 'og_ksift_describe')
        return lafs, scores, desc

    @torch.no_grad()
    def _run(self, images: torch.Tensor, min_stack: bool):
        img = self._image(images)
        with torch.cuda.device(img.device):
            ws, det_lafs, det_resp, sel, n_sel = self._detect_select(img, min_stack)
            counts = n_sel.tolist()                                     # the one host synchronisation: the output sizes
            lafs, scores, desc = self._describe(img, ws, det_lafs, det_resp, sel, n_sel, max(max(counts), 1))
        return lafs, scores, desc, counts

    def forward(self, image: torch.Tensor, mask=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """The reference's ``Features.forward``: every image keeps the batch's smallest kept count (min-stack).  ``mask`` is ignored,
        as in the reference."""
        lafs, scores, desc, counts = self._run(image, min_stack=True)
        n = counts[0] if counts else 0
        return lafs[:, :n], scores[:, :n], desc[:, :n]

    def extract_batch(self, images: torch.Tensor) -> List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        """B same-size images through one launch per stage: a list of B ``(lafs [1,N_b,2,3], responses [1,N_b], descriptors
        [1,N_b,128])``, each equal to ``forward`` of that image alone."""
        lafs, scores, desc, counts = self._run(images, min_stack=False)
        return [(lafs[b:b + 1, :k], scores[b:b + 1, :k], desc[b:b + 1, :k]) for b, k in enumerate(counts)]

    @torch.no_grad()
    def extract_padded(self, images: torch.Tensor, capacity: Optional[int] = None):
        """``extract_batch`` at a fixed capacity, without a host synchronisation.

        images [B,1,H,W] -> (lafs [B,K,2,3], responses [B,K], descriptors [B,K,128], num_keypoints [B] int32, overflow [B] int32),
        all on the images' device, K = ``capacity`` (default ``max_keypoints``).  Rows [0, num_keypoints[b]) of image b are
        ``extract_batch``'s rows for it, the rows past them are 0.  ``overflow[b] = 1`` where K cuts the image (the first K rows in
        response order are kept)."""
        K = padded_capacity(self.max_keypoints, capacity)
        img = self._image(images)
        B = img.shape[0]
        dev = img.device
        i32 = dict(dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            ws, det_lafs, det_resp, sel, n_sel = self._detect_select(img, min_stack=False)
            num, overflow = torch.empty(B, **i32), torch.zeros(B, **i32)
            _cabi.check(_cabi.lib().og_keypoint_counts(ptr(n_sel), B, self.max_keypoints, -1, K, ptr(num), None, ptr(overflow), stream(dev)),
                        'og_keypoint_counts')
            lafs, scores, desc = self._describe(img, ws, det_lafs, det_resp, sel, num, K)
        return lafs, scores, desc, num, overflow
