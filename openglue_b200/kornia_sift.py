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

from typing import NamedTuple

import torch

from . import _cabi
from ._cabi import ptr, stream
from ._frontend import FrontEnd

__all__ = ['SIFT']

MAX_FEATURES = 8192                 # keypoints per image the detector and run_nms sort in one CTA's shared memory


class Detection(NamedTuple):
    """The scale-space detector's workspace, its rows (lafs [B, max_keypoints, 2, 3], responses [B, max_keypoints]), and
    ``run_nms``'s selection with its length per image"""
    ws: torch.Tensor
    lafs: torch.Tensor
    resp: torch.Tensor
    sel: torch.Tensor
    n_sel: torch.Tensor


def scale_space_select(fe: FrontEnd, img: torch.Tensor, min_stack: bool, pyramid: str, detect: str):
    """kornia's scale-space detector (the C entry points ``pyramid`` and ``detect``: og_ksift_* or og_kgftt_*) and the reference's
    run_nms on B images for ``SIFT`` and ``GFTTAffNetHardNet``"""
    B, _, H, W = img.shape
    dev, k = img.device, fe.max_keypoints
    lib = _cabi.lib()
    st = stream(dev)
    ws, work = fe._workspace(dev, B, H, W)
    lafs = torch.empty(B, k, 2, 3, dtype=torch.float32, device=dev)
    resp = torch.empty(B, k, dtype=torch.float32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    _cabi.check(getattr(lib, pyramid)(ptr(img), B, H, W, k, ptr(ws), ws.numel(), st), pyramid)
    _cabi.check(getattr(lib, detect)(B, H, W, k, ptr(ws), ws.numel(), ptr(lafs), ptr(resp), ptr(count), st), detect)
    sel = torch.empty(B, k, dtype=torch.int32, device=dev)
    n_sel = torch.empty(B, dtype=torch.int32, device=dev)
    _cabi.check(lib.og_ksift_select(ptr(lafs), ptr(resp), ptr(count), B, H, W, k, int(fe.perform_nms), fe.nms_diameter, k,
                                    int(min_stack), ptr(work), work.numel(), ptr(sel), ptr(n_sel), st), 'og_ksift_select')
    return Detection(ws, lafs, resp, sel, n_sel)


class SIFT(FrontEnd):
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

    def extra_repr(self) -> str:
        return (f'max_keypoints={self.max_keypoints}, perform_nms={self.perform_nms}, nms_diameter={self.nms_diameter}, '
                f'upright={self.upright}, rootsift={self.rootsift}')

    def _workspace_bytes(self, lib, B, H, W):
        return {'og_ksift_workspace_bytes': lib.og_ksift_workspace_bytes(B, H, W, self.max_keypoints),
                'og_ksift_select_workspace_bytes': lib.og_ksift_select_workspace_bytes(B, self.max_keypoints)}

    def _detect_select(self, img: torch.Tensor, min_stack: bool, overflow=None):
        return scale_space_select(self, img, min_stack, 'og_ksift_pyramid', 'og_ksift_detect')

    def _describe(self, img, ws, det_lafs, det_resp, sel, n, out_cap):
        """The orientation, descriptor and LAF of the selected detector rows det_lafs[b, sel[b, j]], j < n[b]"""
        B, _, H, W = img.shape
        lafs, scores, desc = out = self._outputs(B, out_cap, img.device)
        k = self.max_keypoints
        _cabi.check(_cabi.lib().og_ksift_describe(ptr(img), B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp), k, ptr(sel),
                                                  ptr(n), out_cap, int(self.upright), int(self.rootsift), ptr(lafs), ptr(scores), ptr(desc),
                                                  None, stream(img.device)), 'og_ksift_describe')
        return out
