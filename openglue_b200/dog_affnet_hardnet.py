"""Drop-in for the reference's ``OPENCVDoGAffNetHardNet`` features (models/features/opencv/dog_affnet_harnet.py on
models/features/opencv/base.py): OpenCV's SIFT detector with the reference's radius NMS and top-k, kornia_moons' LAFs, kornia's
``LAFAffNetShapeEstimator``, ``LAFOrienter(32, angle_detector=OriNet)`` and ``HardNet``, restated from kornia 0.6.3 and run on
the GPU.

Detection and selection are ``OpenCVSIFT``'s kernels unchanged (``csrc/sift.cuh``: the image quantised as the reference does,
``uint8(255 x)``, cv2's scale space, the greedy radius NMS and the top-k).  The selected keypoints are then described from the
float image by ``csrc/dog_affnet.cuh``: kornia_moons' LAF and AffNet's patch, the affine frame and OriNet's patch, OriNet's head
with the orienter and HardNet's patch.  The three patch CNNs are NHWC convolutions as im2col + the Hopper GEMM (3xTF32 wgmma by
default, ``precision='fp32'`` for the exact CUDA-core kernel) with their eval-mode BatchNorm folded in float64 on the host, over
chunks of ``CHUNK`` patches so the scratch stays bounded.

Outputs are ordered by descending response, equal responses in cv2's keypoint order (the reference's order is argpartition's,
which is unspecified).  An image without keypoints gives N = 0 (the reference fails there).  ``forward`` / ``extract_batch`` read
the counts back to size their outputs; ``extract_padded`` writes a fixed capacity with the counts on the device and never
synchronises.  There is no CPU path, and nothing here downloads: the pretrained weights come from ``weights=`` or from the files
kornia caches under ``torch.hub.get_dir()/checkpoints``.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr, stream
from ._ops import _Ops
from ._patch_cnn import AFFNET_CONVS, CHUNK, HARDNET_CONVS, HEAD, AffNet, HardNet
from ._patch_cnn import cnn_buffers, conv_stack, fold, load_networks, nhwc_head, run_cnn, weights_key
from .features import padded_capacity
from .sift import DEFAULT_CAPACITY, OpenCVSIFT

__all__ = ['DoGOpenCVAffNetHardNet']

ORINET_CONVS = AFFNET_CONVS             # OriNet's 3x3 stack has AffNet's shapes
# the files kornia 0.6.3 caches in torch.hub.get_dir()/checkpoints, and where it fetches them from
CHECKPOINTS = {
    'affnet': ('AffNet.pth', 'https://github.com/ducha-aiki/affnet/raw/master/pretrained/AffNet.pth'),
    'orinet': ('OriNet.pth', 'https://github.com/ducha-aiki/affnet/raw/master/pretrained/OriNet.pth'),
    'hardnet': ('checkpoint_liberty_with_aug.pth',
                'https://github.com/DagnyT/hardnet/raw/master/pretrained/train_liberty_with_aug/checkpoint_liberty_with_aug.pth'),
}


class _OriNet(nn.Module):
    """OriNet's parameters (``features.<i>``): the head is Conv2d(64, 2, 8, padding=1), 3x3 outputs on the 8x8 map"""

    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(*conv_stack(ORINET_CONVS), nn.Dropout(0.25), nn.Conv2d(64, 2, kernel_size=8, padding=1, bias=True),
                                      nn.Tanh(), nn.AdaptiveAvgPool2d(1))


class _Orienter(nn.Module):
    def __init__(self):
        super().__init__()
        self.angle_detector = _OriNet()


class DoGOpenCVAffNetHardNet(nn.Module):
    """``DoGOpenCVAffNetHardNet(max_keypoints=-1, nms_diameter=9., *, weights=None, precision='tf32x3', capacity=65536)``: the
    reference's constructor, plus where the pretrained networks come from, the GEMM precision and ``OpenCVSIFT``'s bound on the
    keypoints per image before NMS.  ``forward(image [1,1,H,W] float in [0, 1], or uint8 / 255)`` returns ``(lafs [1,N,2,3],
    scores [1,N], descriptors [1,N,128])``; ``extract_batch`` gives one such tuple per image of a batch and ``extract_padded`` a
    fixed capacity.

    ``weights``: ``{'affnet': ..., 'orinet': ..., 'hardnet': ...}``, each a path to kornia's checkpoint file (a dict holding
    ``'state_dict'``) or a state dict with kornia's ``features.<i>.*`` keys; ``None`` reads the files kornia caches in
    ``torch.hub.get_dir()/checkpoints`` (``AffNet.pth``, ``OriNet.pth``, ``checkpoint_liberty_with_aug.pth``) and raises
    ``FileNotFoundError`` when one is absent.  The networks are registered under the reference module's names
    (``affnet.features.<i>.*``, ``orinet.angle_detector.features.<i>.*``, ``hardnet.features.<i>.*``), so a reference module's
    ``state_dict()`` loads."""

    def __init__(self, max_keypoints: int = -1, nms_diameter: float = 9., *, weights=None, precision: str = 'tf32x3',
                 capacity: int = DEFAULT_CAPACITY):
        super().__init__()
        if int(max_keypoints) == 0 or int(max_keypoints) < -1:
            raise ValueError(f'max_keypoints must be positive or -1 (keep all), got {max_keypoints}')
        if precision not in ('tf32x3', 'fp32'):
            raise ValueError(f"precision must be 'tf32x3' or 'fp32', got {precision!r}")
        self.max_keypoints, self.nms_diameter, self.precision = int(max_keypoints), float(nms_diameter), precision
        self._sift = OpenCVSIFT(self.max_keypoints, self.nms_diameter, capacity=capacity)
        self.affnet = AffNet()
        self.orinet = _Orienter()
        self.hardnet = HardNet()
        self.eval()
        self._ws, self._packed = {}, None
        self.load_weights(weights)

    @property
    def capacity(self) -> int:
        return self._sift.capacity

    def extra_repr(self) -> str:
        return f'max_keypoints={self.max_keypoints}, nms_diameter={self.nms_diameter}, precision={self.precision!r}'

    # ------------------------------------------------------------------ weights
    def load_weights(self, weights=None) -> None:
        """Loads AffNet, OriNet and HardNet from ``weights`` (see the class) or from kornia's cache; never downloads."""
        load_networks('DoGOpenCVAffNetHardNet', weights, CHECKPOINTS,
                      {'affnet': self.affnet, 'orinet': self.orinet.angle_detector, 'hardnet': self.hardnet})

    def _weights_on(self, dev):
        """The networks' weights on dev, packed once per parameter / buffer version: {name: [(W [Cout, K], bias [Cout])]}; OriNet's
        head as [2, (ky, kx, c)] for og_dogaff_orinet_head"""
        key = (weights_key(self), dev)
        if self._packed is None or self._packed[0] != key:
            packed = {}
            for name, net, convs in (('affnet', self.affnet.features, AFFNET_CONVS), ('orinet', self.orinet.angle_detector.features, ORINET_CONVS),
                                     ('hardnet', self.hardnet.features, HARDNET_CONVS)):
                layers = [fold(net[i].weight, net[i + 1]) for i, *_ in convs]
                layers.append(fold(net[HEAD].weight, net[HEAD + 1]) if name == 'hardnet' else nhwc_head(net[HEAD]))
                packed[name] = [(w.to(dev), b.to(dev)) for w, b in layers]
            self._packed = (key, packed)
        return self._packed[1]

    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError('openglue_b200.DoGOpenCVAffNetHardNet is the inference front-end (its networks run on their running '
                               'BatchNorm statistics); fine-tuning them is not built')
        return super().train(mode)

    # ------------------------------------------------------------------ device work
    def _workspace(self, dev, B, H, W):
        key = (dev, B, H, W)
        if key not in self._ws:
            sizes = [k for k in self._ws if k[0] != 'cnn']
            while len(sizes) >= 2:                                      # the two image sizes of a pair batch stay cached
                del self._ws[sizes.pop(0)]
            n = _cabi.check_size(_cabi.lib().og_dogaff_workspace_bytes(B, H, W), 'og_dogaff_workspace_bytes')
            self._ws[key] = torch.empty(n, dtype=torch.uint8, device=dev)
        return self._ws[key]

    @staticmethod
    def _image(images) -> torch.Tensor:
        if not torch.is_tensor(images):
            raise TypeError(f'images must be a CUDA tensor [B, 1, H, W]; numpy input (the reference\'s CPU path) is not supported, '
                            f'got {type(images)}')
        if images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f'images must be [B, 1, H, W], got {tuple(images.shape)}')
        if images.device.type != 'cuda':
            raise RuntimeError('openglue_b200.DoGOpenCVAffNetHardNet needs CUDA tensors (sm_90a); there is no CPU path')
        if images.dtype == torch.uint8:
            return (images.float() / 255.).contiguous()
        if not images.is_floating_point():
            raise ValueError(f'images must be float in [0, 1] or uint8, got {images.dtype}')
        return images.detach().float().contiguous()

    def _describe(self, img, kp, sel, n, out_cap):
        """Rows [0, n[b]) of the [B, out_cap] outputs from the selected keypoints kp[b, sel[b, j]]: (lafs, scores, desc, angles)"""
        B, _, H, W = img.shape
        dev = img.device
        f32 = dict(dtype=torch.float32, device=dev)
        lafs, scores, desc = torch.empty(B, out_cap, 2, 3, **f32), torch.empty(B, out_cap, **f32), torch.empty(B, out_cap, 128, **f32)
        angles = torch.empty(B, out_cap, **f32)
        lib = _cabi.lib()
        ops = _Ops(dev, _cabi.OG_PREC_FP32 if self.precision == 'fp32' else _cabi.OG_PREC_TF32X3)
        st = ops.st()
        wts = self._weights_on(dev)
        ws = self._workspace(dev, B, H, W)
        patches, col, act0, act1, xy = cnn_buffers(self._ws, dev)
        cap = self.capacity
        args = (ptr(img), B, H, W, ptr(ws), ws.numel())
        _cabi.check(lib.og_dogaff_pyramid(*args, st), 'og_dogaff_pyramid')
        ori_w, ori_b = wts['orinet'][-1]
        rows_all = B * out_cap
        d2 = desc.view(rows_all, 128)
        for r0 in range(0, rows_all, CHUNK):
            rows = min(CHUNK, rows_all - r0)
            _cabi.check(lib.og_dogaff_affnet_patches(*args, ptr(kp), cap, ptr(sel), ptr(n), out_cap, r0, rows, ptr(lafs), ptr(scores),
                                                     ptr(patches), st), 'og_dogaff_affnet_patches')
            run_cnn(ops, wts['affnet'], patches, rows, AFFNET_CONVS, col, (act0, act1), xy[:rows * 3].view(rows, 3))
            _cabi.check(lib.og_dogaff_frames(*args, ptr(n), out_cap, r0, rows, ptr(xy), ptr(lafs), ptr(patches), st), 'og_dogaff_frames')
            act = run_cnn(ops, wts['orinet'], patches, rows, ORINET_CONVS, col, (act0, act1), None)
            _cabi.check(lib.og_dogaff_orinet_head(*args, ptr(n), out_cap, r0, rows, ptr(act), ptr(ori_w), ptr(ori_b), ptr(lafs), ptr(angles),
                                                  ptr(patches), st), 'og_dogaff_orinet_head')
            run_cnn(ops, wts['hardnet'], patches, rows, HARDNET_CONVS, col, (act0, act1), d2[r0:r0 + rows])
        _cabi.check(lib.og_kgftt_desc_finish(ptr(desc), B, out_cap, ptr(n), st), 'og_kgftt_desc_finish')
        return lafs, scores, desc, angles

    @torch.no_grad()
    def _run(self, images):
        img = self._image(images)
        B = img.shape[0]
        with torch.cuda.device(img.device):
            _, kp, _, count, sel, n_sel = self._sift._detect_select(img, 1)
            counts = torch.cat([count, n_sel]).tolist()                 # the one host synchronisation: the output sizes
            if max(counts[:B]) > self.capacity:
                raise RuntimeError(f'{max(counts[:B])} SIFT keypoints in one image exceed the capacity {self.capacity}: raise '
                                   f'DoGOpenCVAffNetHardNet(capacity=...)')
            n = counts[B:]
            lafs, scores, desc, _ = self._describe(img, kp, sel, n_sel, max(max(n), 1))
        return [(lafs[b:b + 1, :k], scores[b:b + 1, :k], desc[b:b + 1, :k]) for b, k in enumerate(n)]

    def forward(self, image: torch.Tensor, mask=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """The reference's ``detect_and_compute`` of one image; ``mask`` is ignored, as in the reference."""
        image = self._image(image)
        assert image.size(0) == 1                                       # as the reference (dog_affnet_harnet.py)
        return self._run(image)[0]

    def extract_batch(self, images: torch.Tensor) -> List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        """B same-size images through one launch per stage: a list of B ``(lafs [1,N_b,2,3], scores [1,N_b], descriptors
        [1,N_b,128])``, each equal to ``forward`` of that image."""
        return self._run(images)

    @torch.no_grad()
    def extract_padded(self, images: torch.Tensor, capacity: Optional[int] = None):
        """``extract_batch`` at a fixed capacity, without a host synchronisation.

        images [B,1,H,W] -> (lafs [B,K,2,3], scores [B,K], descriptors [B,K,128], num_keypoints [B] int32, overflow [B] int32), all
        on the images' device, K = ``capacity`` (default ``max_keypoints``).  Rows [0, num_keypoints[b]) of image b are
        ``extract_batch``'s rows for it, the rows past them are 0.  ``overflow[b] = 1`` where ``extract_batch`` would raise (more
        keypoints before NMS than ``self.capacity``; the selection then runs on those that fitted) or K cuts the image (the first K
        rows in response order are kept)."""
        K = padded_capacity(self.max_keypoints, capacity)
        img = self._image(images)
        B = img.shape[0]
        dev = img.device
        i32 = dict(dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            overflow = torch.empty(B, **i32)
            _, kp, _, _, sel, n_sel = self._sift._detect_select(img, 1, overflow)
            num = torch.empty(B, **i32)
            _cabi.check(_cabi.lib().og_keypoint_counts(ptr(n_sel), B, K, -1, K, ptr(num), None, ptr(overflow), stream(dev)),
                        'og_keypoint_counts')
            lafs, scores, desc, _ = self._describe(img, kp, sel, num, K)
        return lafs, scores, desc, num, overflow
