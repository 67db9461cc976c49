"""What the keypoint front-ends (``OpenCVSIFT``, ``SIFT``, ``GFTTAffNetHardNet``, ``DoGOpenCVAffNetHardNet``) share around their
kernels: the input checks, the workspace cache, the one host synchronisation of ``forward`` / ``extract_batch`` and the fixed
capacity of ``extract_padded``.  A front-end supplies its workspace sizes and two hooks: ``_detect_select`` (detection, NMS and
top-k) and ``_describe`` (the outputs of the selected keypoints)."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr, stream
from .features import padded_capacity


class FrontEnd(nn.Module):
    """The shell of a front-end.  A subclass defines

    - ``_workspace_bytes(lib, B, H, W)``: {size query name: its result} of the workspaces of one image size;
    - ``_detect_select(img, min_stack, overflow=None)``: a named tuple of what the describe stage reads, ending with ``n_sel``
      (int32 [B], the kept keypoints); OpenCV's detector also gives ``count`` (the keypoints before NMS) and, with ``overflow``,
      flags there the images over ``capacity``;
    - ``_describe(img, *det[:-1], n, K)``: ``(lafs [B,K,2,3], scores [B,K], descriptors [B,K,128])``, rows [0, n[b]) of image b
      from its selected keypoints; or ``_describe_selected`` where that is not the module's form."""

    # OpenCV's detector (OpenCVSIFT, DoGOpenCVAffNetHardNet): ``forward`` takes one image, as the reference's wrappers assert, and
    # at most ``capacity`` keypoints per image before NMS (``extract_batch`` raises past it, the padded detector flags it).
    # kornia's (SIFT, GFTTAffNetHardNet): ``forward`` min-stacks the batch, and the selection holds at most max_keypoints rows.
    _cv2_detector = False
    _uint8_input = False        # the detector reads uint8 images as they are and quantises float ones itself (OpenCVSIFT)

    def __init__(self):
        super().__init__()
        self._ws, self._packed = {}, None

    def _workspace(self, dev, B, H, W):
        """The workspaces of one image size (a tuple, or the tensor where there is one).  The two image sizes of a pair batch stay
        cached; entries not keyed by an image size (the patch CNNs' chunk buffers) stay for good."""
        key = (dev, B, H, W)
        if key not in self._ws:
            sizes = [k for k in self._ws if isinstance(k[0], torch.device)]
            while len(sizes) >= 2:
                del self._ws[sizes.pop(0)]
            ws = tuple(torch.empty(_cabi.check_size(n, what), dtype=torch.uint8, device=dev)
                       for what, n in self._workspace_bytes(_cabi.lib(), B, H, W).items())
            self._ws[key] = ws if len(ws) > 1 else ws[0]
        return self._ws[key]

    def _image(self, images, forward: bool = False) -> torch.Tensor:
        name = type(self).__name__
        if not torch.is_tensor(images):
            raise TypeError(f'openglue_b200.{name} takes a CUDA tensor [B, 1, H, W] (not numpy, the reference\'s CPU path), '
                            f'got {type(images)}')
        if images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f'images must be [B, 1, H, W], got {tuple(images.shape)}')
        if forward and self._cv2_detector:
            assert images.shape[0] == 1                                 # as the reference's wrappers (torch_wrapper.py:42)
        if images.device.type != 'cuda':
            raise RuntimeError(f'openglue_b200.{name} needs CUDA tensors (sm_90a); there is no CPU path')
        if images.dtype == torch.uint8:
            return images.contiguous() if self._uint8_input else (images.float() / 255.).contiguous()
        if not images.is_floating_point() and not self._uint8_input:
            raise ValueError(f'images must be float in [0, 1] or uint8, got {images.dtype}')
        return images.detach().float().contiguous()

    @staticmethod
    def _outputs(B: int, K: int, dev, zeros: bool = False):
        new = torch.zeros if zeros else torch.empty
        f32 = dict(dtype=torch.float32, device=dev)
        return new(B, K, 2, 3, **f32), new(B, K, **f32), new(B, K, 128, **f32)

    def _describe_selected(self, img, det, n, K: int, n_max: int, padded: bool):
        """The outputs of the keypoints ``det`` selected, K rows per image; n_max is a host bound on n"""
        return self._describe(img, *det[:-1], n, K)

    @torch.no_grad()
    def _run(self, img: torch.Tensor, min_stack: bool):
        B = img.shape[0]
        with torch.cuda.device(img.device):
            det = self._detect_select(img, min_stack)
            if self._cv2_detector:
                counts = torch.cat([det.count, det.n_sel]).tolist()     # the one host synchronisation: the output sizes
                if max(counts[:B]) > self.capacity:
                    raise RuntimeError(f'{max(counts[:B])} SIFT keypoints in one image exceed the capacity {self.capacity}: raise '
                                       f'{type(self).__name__}(capacity=...)')
                counts = counts[B:]
            else:
                counts = det.n_sel.tolist()                             # the one host synchronisation: the output sizes
            n_max = max(counts)
            out = self._describe_selected(img, det, det.n_sel, max(n_max, 1), n_max, False)
        return (*out, counts)

    def forward(self, image: torch.Tensor, mask=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """The reference's ``forward``: ``(lafs [B,N,2,3], scores [B,N], descriptors [B,N,128])``, every image keeping the batch's
        smallest kept count (min-stack; OpenCV's detector takes B = 1).  ``mask`` is ignored, as in the reference."""
        lafs, scores, desc, counts = self._run(self._image(image, forward=True), min_stack=True)
        n = counts[0] if counts else 0
        return lafs[:, :n], scores[:, :n], desc[:, :n]

    def extract_batch(self, images: torch.Tensor) -> List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        """B same-size images through one launch per stage: a list of B ``(lafs [1,N_b,2,3], scores [1,N_b], descriptors
        [1,N_b,128])``, each equal to ``forward`` of that image alone."""
        lafs, scores, desc, counts = self._run(self._image(images), min_stack=False)
        return [(lafs[b:b + 1, :k], scores[b:b + 1, :k], desc[b:b + 1, :k]) for b, k in enumerate(counts)]

    @torch.no_grad()
    def extract_padded(self, images: torch.Tensor, capacity: Optional[int] = None):
        """``extract_batch`` at a fixed capacity, without a host synchronisation.

        images [B,1,H,W] -> (lafs [B,K,2,3], scores [B,K], descriptors [B,K,128], num_keypoints [B] int32, overflow [B] int32), all
        on the images' device, K = ``capacity`` (default ``max_keypoints``).  Rows [0, num_keypoints[b]) of image b are
        ``extract_batch``'s rows for it; the rows past them are 0, as ``pad_features`` writes them.

        ``overflow[b] = 1`` where K cuts the image (the first K rows in response order are kept and num_keypoints[b] = K) or, for
        OpenCV's detector, where ``extract_batch`` would raise: more keypoints before NMS than ``capacity`` (the selection then
        runs on those that fitted).  Check it whenever the results are next read on the host."""
        K = padded_capacity(self.max_keypoints, capacity)
        img = self._image(images)
        B, dev = img.shape[0], img.device
        i32 = dict(dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            if self._cv2_detector:
                overflow = torch.empty(B, **i32)                        # written by the detector
                det = self._detect_select(img, False, overflow)
                stored = K
            else:
                det = self._detect_select(img, False)
                overflow, stored = torch.zeros(B, **i32), self.max_keypoints
            num = torch.empty(B, **i32)
            _cabi.check(_cabi.lib().og_keypoint_counts(ptr(det.n_sel), B, stored, -1, K, ptr(num), None, ptr(overflow), stream(dev)),
                        'og_keypoint_counts')
            out = self._describe_selected(img, det, num, K, K, True)
        return (*out, num, overflow)
