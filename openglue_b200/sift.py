"""Drop-in for the reference's ``OPENCV_SIFT`` local features (``models/features/opencv/__init__.py:5``:
``sift_create_torch(max_keypoints, nms_diameter, rootsift)``, i.e. ``OpenCVFeaturesTorchWrapper(sift_create(...))``,
torch_wrapper.py:19-49, _features.py:10-18, base.py:14-182), run on the GPU.

The reference converts the image to uint8 (``(255. * image).astype(np.uint8)``), runs
``cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000).detectAndCompute`` on the host, keeps the keypoints a greedy
radius NMS (``nms_diameter / 2``) leaves, then the ``max_keypoints`` largest responses, RootSIFT-normalises their descriptors and
turns them into LAFs (``scale = 6 size``, ``theta = -angle``).  Here every step is a kernel of ``libopenglue_b200.so``
(``csrc/sift.cuh``): scale-space pyramid, extrema and their interpolation, orientations, cv2's keypoint order and duplicate
removal, NMS + top-k, and descriptors for the selected keypoints only, with RootSIFT and the LAFs in the same pass.  The only host
step of ``forward`` / ``extract_batch`` is reading the per-image keypoint counts to size the outputs; ``extract_padded`` writes
outputs of a fixed capacity with the counts on the device and never synchronises.  There is no CPU path.

Outputs are ordered by descending response, equal responses in cv2's keypoint order (the reference's order is argpartition's,
which is unspecified).  An image without keypoints gives N = 0 (the reference fails there: cv2 returns no descriptors).
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

from . import _cabi
from ._cabi import ptr, stream
from ._frontend import FrontEnd

__all__ = ['OpenCVSIFT', 'sift_create_torch']

DEFAULT_CAPACITY = 1 << 16          # keypoints per image before NMS (cv2 finds about 7,000 on a 960 x 720 texture)


class Detection(NamedTuple):
    """``OpenCVSIFT._detect_select``'s result: the workspace with the scale space, the keypoints [B, capacity, 5] (x, y, size,
    angle, response) with their packed octaves, the keypoints found per image, the selection and its length per image"""
    ws: torch.Tensor
    kp: torch.Tensor
    octave: torch.Tensor
    count: torch.Tensor
    sel: torch.Tensor
    n_sel: torch.Tensor


class OpenCVSIFT(FrontEnd):
    """``OpenCVSIFT(max_keypoints=-1, nms_diameter=9., rootsift=True)``: ``forward(image [1,1,H,W]) -> (lafs [1,N,2,3],
    scores [1,N], descriptors [1,N,128])`` on the image's device; ``extract_batch(images [B,1,H,W])`` runs B same-size images
    through one launch per stage and returns one such tuple per image.  Images are float in [0, 1] (quantised as the reference
    does) or uint8.  ``capacity`` bounds the keypoints per image before NMS; more raise."""

    _cv2_detector = _uint8_input = True

    def __init__(self, max_keypoints: int = -1, nms_diameter: float = 9., rootsift: bool = True, capacity: int = DEFAULT_CAPACITY):
        super().__init__()
        self.max_keypoints, self.nms_diameter, self.rootsift = int(max_keypoints), float(nms_diameter), bool(rootsift)
        self.capacity = int(capacity)

    def extra_repr(self) -> str:
        return f'max_keypoints={self.max_keypoints}, nms_diameter={self.nms_diameter}, rootsift={self.rootsift}'

    def _workspace_bytes(self, lib, B, H, W):
        return {'og_sift_workspace_bytes': lib.og_sift_workspace_bytes(B, H, W, self.capacity),
                'og_sift_select_workspace_bytes': lib.og_sift_select_workspace_bytes(B, self.capacity)}

    def _detect_select(self, img: torch.Tensor, min_stack: bool = False, overflow: Optional[torch.Tensor] = None):
        """Detection and NMS + top-k of B images (``forward`` takes one, so there is no min-stack).  With ``overflow`` (int32 [B])
        the padded detection runs: count[b] is the number of keypoints written and overflow[b] flags a capacity exceeded."""
        B, _, H, W = img.shape
        dev = img.device
        lib = _cabi.lib()
        cap = self.capacity
        dtype = 0 if img.dtype == torch.uint8 else 1
        i32 = dict(dtype=torch.int32, device=dev)
        st = stream(dev)
        ws, work = self._workspace(dev, B, H, W)
        kp = torch.empty(B, cap, 5, dtype=torch.float32, device=dev)
        octave, count = torch.empty(B, cap, **i32), torch.empty(B, **i32)
        if overflow is None:
            _cabi.check(lib.og_sift_detect(ptr(img), dtype, B, H, W, cap, ptr(ws), ws.numel(), ptr(kp), ptr(octave), ptr(count), st),
                        'og_sift_detect')
        else:
            _cabi.check(lib.og_sift_detect_padded(ptr(img), dtype, B, H, W, cap, ptr(ws), ws.numel(), ptr(kp), ptr(octave), ptr(count),
                                                  ptr(overflow), st), 'og_sift_detect_padded')
        sel, n_sel = torch.empty(B, cap, **i32), torch.empty(B, **i32)
        _cabi.check(lib.og_sift_select(ptr(kp), ptr(count), B, cap, self.nms_diameter / 2, self.max_keypoints, ptr(work), work.numel(),
                                       ptr(sel), ptr(n_sel), st), 'og_sift_select')
        return Detection(ws, kp, octave, count, sel, n_sel)

    def _describe_selected(self, img, det, n, K, n_max, padded):
        """The descriptors, RootSIFT and LAFs of the selected keypoints kp[b, sel[b, j]], j < n[b].  The kernel writes those rows
        only, so extract_padded's outputs start at 0."""
        B, _, H, W = img.shape
        lafs, scores, desc = out = self._outputs(B, K, img.device, zeros=padded)
        _cabi.check(_cabi.lib().og_sift_describe(ptr(det.ws), B, H, W, self.capacity, ptr(det.kp), ptr(det.octave), ptr(det.sel), ptr(n),
                                                 K, n_max, int(self.rootsift), ptr(lafs), ptr(scores), ptr(desc), None,
                                                 stream(img.device)), 'og_sift_describe')
        return out


def sift_create_torch(max_keypoints: int = -1, nms_diameter: float = 9., rootsift: bool = True) -> OpenCVSIFT:
    """The registry constructor of ``OPENCV_SIFT`` (reference models/features/opencv/_features_torch.py)."""
    return OpenCVSIFT(max_keypoints=max_keypoints, nms_diameter=nms_diameter, rootsift=rootsift)
