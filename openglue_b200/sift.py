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

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr, stream
from .features import padded_capacity

__all__ = ['OpenCVSIFT', 'sift_create_torch']

DEFAULT_CAPACITY = 1 << 16          # keypoints per image before NMS (cv2 finds about 7,000 on a 960 x 720 texture)


class OpenCVSIFT(nn.Module):
    """``OpenCVSIFT(max_keypoints=-1, nms_diameter=9., rootsift=True)``: ``forward(image [1,1,H,W]) -> (lafs [1,N,2,3],
    scores [1,N], descriptors [1,N,128])`` on the image's device; ``extract_batch(images [B,1,H,W])`` runs B same-size images
    through one launch per stage and returns one such tuple per image.  Images are float in [0, 1] (quantised as the reference
    does) or uint8.  ``capacity`` bounds the keypoints per image before NMS; more raise."""

    def __init__(self, max_keypoints: int = -1, nms_diameter: float = 9., rootsift: bool = True, capacity: int = DEFAULT_CAPACITY):
        super().__init__()
        self.max_keypoints, self.nms_diameter, self.rootsift = int(max_keypoints), float(nms_diameter), bool(rootsift)
        self.capacity = int(capacity)
        self._ws = {}

    def extra_repr(self) -> str:
        return f'max_keypoints={self.max_keypoints}, nms_diameter={self.nms_diameter}, rootsift={self.rootsift}'

    def _workspace(self, dev, B, H, W):
        lib = _cabi.lib()
        key = (dev, B, H, W)
        if key not in self._ws:
            while len(self._ws) >= 2:                                   # the two image sizes of a pair batch stay cached
                del self._ws[next(iter(self._ws))]
            n = _cabi.check_size(lib.og_sift_workspace_bytes(B, H, W, self.capacity), 'og_sift_workspace_bytes')
            m = _cabi.check_size(lib.og_sift_select_workspace_bytes(B, self.capacity), 'og_sift_select_workspace_bytes')
            self._ws[key] = (torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(m, dtype=torch.uint8, device=dev))
        return self._ws[key]

    @staticmethod
    def _image(images: torch.Tensor):
        if images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f'images must be [B, 1, H, W], got {tuple(images.shape)}')
        if images.dtype == torch.uint8:
            return images.contiguous(), 0
        return images.detach().float().contiguous(), 1

    def _detect_select(self, img: torch.Tensor, dtype: int, overflow: Optional[torch.Tensor] = None):
        """detection and NMS + top-k of B images: (ws, kp, octave, count, sel, n_sel).  With ``overflow`` (int32 [B]) the padded
        detection runs: count[b] is the number of keypoints written and overflow[b] flags a capacity exceeded."""
        B, _, H, W = img.shape
        dev = img.device
        lib = _cabi.lib()
        cap = self.capacity
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
        return ws, kp, octave, count, sel, n_sel

    @torch.no_grad()
    def _run(self, images: torch.Tensor, want_raw: bool = False):
        dev = images.device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200.OpenCVSIFT needs CUDA tensors (sm_90a); there is no CPU path')
        img, dtype = self._image(images)
        B, _, H, W = images.shape
        lib = _cabi.lib()
        cap = self.capacity
        with torch.cuda.device(dev):
            st = stream(dev)
            ws, kp, octave, count, sel, n_sel = self._detect_select(img, dtype)
            counts = torch.cat([count, n_sel]).tolist()                # the one host synchronisation
            if max(counts[:B]) > cap:
                raise RuntimeError(f'{max(counts[:B])} SIFT keypoints in one image exceed the capacity {cap}: raise OpenCVSIFT(capacity=...)')
            n_sel_h = counts[B:]
            n = max(n_sel_h)
            out_cap = max(n, 1)
            lafs = torch.empty(B, out_cap, 2, 3, dtype=torch.float32, device=dev)
            scores = torch.empty(B, out_cap, dtype=torch.float32, device=dev)
            desc = torch.empty(B, out_cap, 128, dtype=torch.float32, device=dev)
            raw = torch.empty(B, out_cap, 128, dtype=torch.float32, device=dev) if want_raw else None
            _cabi.check(lib.og_sift_describe(ptr(ws), B, H, W, cap, ptr(kp), ptr(octave), ptr(sel), ptr(n_sel), out_cap, n, int(self.rootsift),
                                             ptr(lafs), ptr(scores), ptr(desc), ptr(raw), st), 'og_sift_describe')
        self.last_raw = dict(kp=kp, octave=octave, count=count, sel=sel, raw_desc=raw) if want_raw else None
        return [(lafs[b:b + 1, :k], scores[b:b + 1, :k], desc[b:b + 1, :k]) for b, k in enumerate(n_sel_h)]

    def forward(self, image: torch.Tensor, mask=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        B = image.shape[0]
        assert B == 1                                                   # as the reference's wrapper (torch_wrapper.py:42)
        return self._run(image)[0]

    def extract_batch(self, images: torch.Tensor) -> List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        """B same-size images through one launch per stage: a list of B ``(lafs [1,N_b,2,3], scores [1,N_b], descriptors [1,N_b,128])``,
        each equal to ``forward`` of that image."""
        return self._run(images)

    @torch.no_grad()
    def extract_padded(self, images: torch.Tensor, capacity: Optional[int] = None):
        """``extract_batch`` at a fixed capacity, without a host synchronisation.

        images [B,1,H,W] -> (lafs [B,K,2,3], scores [B,K], descriptors [B,K,128], num_keypoints [B] int32, overflow [B] int32), all
        on the images' device, K = ``capacity`` (default ``max_keypoints``).  Rows [0, num_keypoints[b]) of image b are
        ``extract_batch``'s N_b rows for it; the rows past them are 0, as ``pad_features`` writes them.

        ``overflow[b] = 1`` where ``extract_batch`` would raise or K cuts the image: more keypoints before NMS than
        ``OpenCVSIFT.capacity`` (the selection then runs on the keypoints that fitted), or more selected keypoints than K (the
        first K in response order are kept and num_keypoints[b] = K).  Check it whenever the results are next read on the host."""
        K = padded_capacity(self.max_keypoints, capacity)
        img, dtype = self._image(images)
        dev = images.device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200.OpenCVSIFT needs CUDA tensors (sm_90a); there is no CPU path')
        B, _, H, W = images.shape
        lib = _cabi.lib()
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = stream(dev)
            overflow = torch.empty(B, **i32)
            ws, kp, octave, count, sel, n_sel = self._detect_select(img, dtype, overflow)
            num = torch.empty(B, **i32)
            _cabi.check(lib.og_keypoint_counts(ptr(n_sel), B, K, -1, K, ptr(num), None, ptr(overflow), st), 'og_keypoint_counts')
            # the outputs start at 0: the descriptor kernel writes rows [0, num[b]) only
            lafs, scores, desc = torch.zeros(B, K, 2, 3, **f32), torch.zeros(B, K, **f32), torch.zeros(B, K, 128, **f32)
            _cabi.check(lib.og_sift_describe(ptr(ws), B, H, W, self.capacity, ptr(kp), ptr(octave), ptr(sel), ptr(num), K, K, int(self.rootsift),
                                             ptr(lafs), ptr(scores), ptr(desc), None, st), 'og_sift_describe')
        return lafs, scores, desc, num, overflow


def sift_create_torch(max_keypoints: int = -1, nms_diameter: float = 9., rootsift: bool = True) -> OpenCVSIFT:
    """The registry constructor of ``OPENCV_SIFT`` (reference models/features/opencv/_features_torch.py)."""
    return OpenCVSIFT(max_keypoints=max_keypoints, nms_diameter=nms_diameter, rootsift=rootsift)
