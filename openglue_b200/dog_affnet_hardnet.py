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

import torch
import torch.nn as nn

from . import _cabi, _patch_cnn
from ._cabi import ptr
from ._patch_cnn import AFFNET_CONVS, CHUNK, HARDNET_CONVS, HEAD, AffNet, CNNFrontEnd, HardNet
from ._patch_cnn import cnn_buffers, conv_stack, fold, load_networks, nhwc_head
from .sift import DEFAULT_CAPACITY, OpenCVSIFT

__all__ = ['DoGOpenCVAffNetHardNet']

ORINET_CONVS = AFFNET_CONVS             # OriNet's 3x3 stack has AffNet's shapes
CHECKPOINTS = {k: _patch_cnn.CHECKPOINTS[k] for k in ('affnet', 'orinet', 'hardnet')}


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


class DoGOpenCVAffNetHardNet(CNNFrontEnd):
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

    _cv2_detector = True

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

    def _pack(self):
        """OriNet's head as [2, (ky, kx, c)] for og_dogaff_orinet_head"""
        packed = {}
        for name, net, convs in (('affnet', self.affnet.features, AFFNET_CONVS),
                                 ('orinet', self.orinet.angle_detector.features, ORINET_CONVS),
                                 ('hardnet', self.hardnet.features, HARDNET_CONVS)):
            layers = [fold(net[i].weight, net[i + 1]) for i, *_ in convs]
            layers.append(fold(net[HEAD].weight, net[HEAD + 1]) if name == 'hardnet' else nhwc_head(net[HEAD]))
            packed[name] = layers
        return packed

    # ------------------------------------------------------------------ device work
    def _workspace_bytes(self, lib, B, H, W):
        return {'og_dogaff_workspace_bytes': lib.og_dogaff_workspace_bytes(B, H, W)}

    def _detect_select(self, img: torch.Tensor, min_stack: bool, overflow=None):
        """``OpenCVSIFT``'s detection and selection, on the float image it quantises as the reference does"""
        return self._sift._detect_select(img, min_stack, overflow)

    def _describe_selected(self, img, det, n, K, n_max, padded):
        return self._describe(img, det.kp, det.sel, n, K)[:3]

    def _describe(self, img, kp, sel, n, out_cap, tap=None):
        """The selected keypoints kp[b, sel[b, j]], j < n[b], in chunks of CHUNK: kornia_moons' LAF and AffNet's patch, AffNet,
        the affine frame and OriNet's patch, OriNet and its head with HardNet's patch, HardNet; then the descriptors'
        normalisation.  ``tap(stage, r0, rows, t)``, when given, sees each chunk's patches after the stage that cuts them
        ('affnet', 'orinet', 'hardnet'): (lafs, scores, desc, angles)"""
        B, _, H, W = img.shape
        dev = img.device
        lafs, scores, desc = self._outputs(B, out_cap, dev)
        angles = torch.empty(B, out_cap, dtype=torch.float32, device=dev)
        lib = _cabi.lib()
        ops = self._ops(dev)
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
            _cabi.check(lib.og_dogaff_affnet_patches(*args, ptr(kp), cap, ptr(sel), ptr(n), out_cap, r0, rows, ptr(lafs),
                                                     ptr(scores), ptr(patches), st), 'og_dogaff_affnet_patches')
            if tap is not None:
                tap('affnet', r0, rows, patches)
            _patch_cnn.run_cnn(ops, wts['affnet'], patches, rows, AFFNET_CONVS, col, (act0, act1), xy[:rows * 3].view(rows, 3))
            _cabi.check(lib.og_dogaff_frames(*args, ptr(n), out_cap, r0, rows, ptr(xy), ptr(lafs), ptr(patches), st), 'og_dogaff_frames')
            if tap is not None:
                tap('orinet', r0, rows, patches)
            act = _patch_cnn.run_cnn(ops, wts['orinet'], patches, rows, ORINET_CONVS, col, (act0, act1), None)
            _cabi.check(lib.og_dogaff_orinet_head(*args, ptr(n), out_cap, r0, rows, ptr(act), ptr(ori_w), ptr(ori_b), ptr(lafs),
                                                  ptr(angles), ptr(patches), st), 'og_dogaff_orinet_head')
            if tap is not None:
                tap('hardnet', r0, rows, patches)
            _patch_cnn.run_cnn(ops, wts['hardnet'], patches, rows, HARDNET_CONVS, col, (act0, act1), d2[r0:r0 + rows])
        _cabi.check(lib.og_kgftt_desc_finish(ptr(desc), B, out_cap, ptr(n), st), 'og_kgftt_desc_finish')
        return lafs, scores, desc, angles
