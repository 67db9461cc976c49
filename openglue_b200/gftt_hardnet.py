"""Drop-in for the reference's ``GFTTAffNetHardNet`` features (models/features/hardnet.py on models/features/base.py:8-82):
kornia's GFTT scale-space detector (``ScaleSpaceDetector`` with ``CornerGFTT``, ``ConvQuadInterp3d(10, 1e-5)``, ``ScalePyramid(3,
1.6, 32, double_image=False)``), ``LAFAffNetShapeEstimator`` and ``LAFOrienter(19)``, the reference's ``run_nms`` and kornia's
``LAFDescriptor`` with ``HardNet``, restated from kornia 0.6.3 and run on the GPU.

Every stage is a kernel of ``libopenglue_b200.so``: the pyramid with its GFTT responses, the detector, ``run_nms``
(``csrc/kornia_gftt.cuh`` on ``csrc/kornia_sift.cuh``), and for the selected keypoints only the AffNet and HardNet patches, the
affine frames and the orientation.  The two patch CNNs are NHWC convolutions as im2col + the Hopper GEMM (3xTF32 wgmma by
default, ``precision='fp32'`` for the exact CUDA-core kernel), with their eval-mode BatchNorm folded into the weights in float64
on the host, over chunks of ``CHUNK`` patches so the scratch stays bounded.  AffNet and the orienter do not move a LAF's centre and
``run_nms`` reads only centres and responses, so running them after the selection gives the reference's result for less work.

``forward`` / ``extract_batch`` read the kept counts back to size their outputs; ``extract_padded`` writes a fixed capacity with
the counts on the device and never synchronises.  There is no CPU path, and nothing here downloads: the pretrained weights come
from ``weights=`` or from the files kornia caches under ``torch.hub.get_dir()/checkpoints``.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _cabi, _patch_cnn
from ._cabi import ptr
from ._patch_cnn import AFFNET_CONVS, CHUNK, HARDNET_CONVS, HEAD, PS, CNNFrontEnd, cnn_buffers, load_networks, nhwc_head
from ._patch_cnn import AffNet as _AffNet, HardNet as _HardNet, fold as _fold
from .kornia_sift import MAX_FEATURES, scale_space_select

__all__ = ['GFTTAffNetHardNet']

CHECKPOINTS = {k: _patch_cnn.CHECKPOINTS[k] for k in ('affnet', 'hardnet')}
ORIENT_SMOOTH = (0.33, 0.34, 0.33)  # PatchDominantGradientOrientation's fixed angular smoothing


class _AngleDetector(nn.Module):
    def __init__(self):
        super().__init__()
        self.angular_smooth = nn.Conv1d(1, 1, kernel_size=3, padding=1, bias=False, padding_mode='circular')
        with torch.no_grad():
            self.angular_smooth.weight[:] = torch.tensor([[list(ORIENT_SMOOTH)]])
        self.angular_smooth.weight.requires_grad_(False)


class _Orienter(nn.Module):
    def __init__(self):
        super().__init__()
        self.angle_detector = _AngleDetector()


class GFTTAffNetHardNet(CNNFrontEnd):
    """``GFTTAffNetHardNet(descriptor_dim=128, max_keypoints=8000, perform_nms=True, nms_diameter=9, patch_size=32, upright=False,
    device=None, *, weights=None, precision='tf32x3')``: the reference's constructor, plus where the pretrained networks come from
    and the GEMM precision.  ``forward(images [B,1,H,W] float in [0, 1], or uint8 / 255)`` returns the reference's batch ``(lafs
    [B,N,2,3], responses [B,N], descriptors [B,N,128])``, N min-stacked over the batch as ``run_nms`` does; ``extract_batch`` gives
    one such tuple per image and ``extract_padded`` a fixed capacity.

    ``weights``: ``{'affnet': ..., 'hardnet': ...}``, each a path to kornia's checkpoint file (a dict holding ``'state_dict'``) or
    a state dict with kornia's ``features.<i>.*`` keys; ``None`` reads the files kornia caches in
    ``torch.hub.get_dir()/checkpoints`` (``AffNet.pth``, ``checkpoint_liberty_with_aug.pth``) and raises ``FileNotFoundError`` when
    one is absent.  The networks are registered under the reference module's names (``detector.aff.features.<i>.*``,
    ``descriptor.descriptor.features.<i>.*``), so a reference module's ``state_dict()`` loads.  ``device`` is accepted for the
    reference's signature; the module follows the images' device."""

    def __init__(self, descriptor_dim: int = 128, max_keypoints: int = 8000, perform_nms: bool = True, nms_diameter: int = 9,
                 patch_size: int = 32, upright: bool = False, device=None, *, weights=None, precision: str = 'tf32x3'):
        super().__init__()
        if int(descriptor_dim) != 128:
            raise ValueError(f'HardNet descriptors have 128 entries, got descriptor_dim={descriptor_dim}')
        if int(patch_size) != PS:
            raise ValueError(f'only patch_size=32 (the reference default, AffNet and HardNet input size) is supported, got {patch_size}')
        if not 1 <= int(max_keypoints) <= MAX_FEATURES:
            raise ValueError(f'max_keypoints must be in [1, {MAX_FEATURES}], got {max_keypoints}')
        if perform_nms and (int(nms_diameter) < 1 or int(nms_diameter) % 2 == 0):
            raise ValueError(f'nms_diameter must be a positive odd number, got {nms_diameter}')
        if precision not in ('tf32x3', 'fp32'):
            raise ValueError(f"precision must be 'tf32x3' or 'fp32', got {precision!r}")
        self.descriptor_dim, self.max_keypoints = 128, int(max_keypoints)
        self.perform_nms, self.nms_diameter = bool(perform_nms), int(nms_diameter)
        self.patch_size, self.upright, self.precision = PS, bool(upright), precision
        self.detector = nn.Module()
        self.detector.aff = _AffNet()
        if not self.upright:
            self.detector.ori = _Orienter()
        self.descriptor = nn.Module()
        self.descriptor.descriptor = _HardNet()
        self.eval()
        self.load_weights(weights)

    def extra_repr(self) -> str:
        return (f'max_keypoints={self.max_keypoints}, perform_nms={self.perform_nms}, nms_diameter={self.nms_diameter}, '
                f'upright={self.upright}, precision={self.precision!r}')

    # ------------------------------------------------------------------ weights
    def load_weights(self, weights=None) -> None:
        """Loads AffNet and HardNet from ``weights`` (see the class) or from kornia's cache; never downloads."""
        load_networks('GFTTAffNetHardNet', weights, CHECKPOINTS, {'affnet': self.detector.aff, 'hardnet': self.descriptor.descriptor})

    def _pack(self):
        if not self.upright:
            w = self.detector.ori.angle_detector.angular_smooth.weight.detach().flatten().tolist()
            if any(abs(a - b) > 0 for a, b in zip(w, torch.tensor(ORIENT_SMOOTH).tolist())):
                raise ValueError(f'the orienter smooths its histogram with kornia\'s fixed {ORIENT_SMOOTH}, got {w}')
        aff, hard = self.detector.aff.features, self.descriptor.descriptor.features
        return {'affnet': [_fold(aff[i].weight, aff[i + 1]) for i, *_ in AFFNET_CONVS] + [nhwc_head(aff[HEAD])],
                'hardnet': [_fold(hard[i].weight, hard[i + 1]) for i, *_ in HARDNET_CONVS] + [_fold(hard[HEAD].weight, hard[HEAD + 1])]}

    # ------------------------------------------------------------------ device work
    def _workspace_bytes(self, lib, B, H, W):
        return {'og_kgftt_workspace_bytes': lib.og_kgftt_workspace_bytes(B, H, W, self.max_keypoints),
                'og_ksift_select_workspace_bytes': lib.og_ksift_select_workspace_bytes(B, self.max_keypoints)}

    def _detect_select(self, img: torch.Tensor, min_stack: bool, overflow=None):
        return scale_space_select(self, img, min_stack, 'og_kgftt_pyramid', 'og_kgftt_detect')

    def _describe(self, img, ws, det_lafs, det_resp, sel, n, out_cap, tap=None):
        """The selected detector rows det_lafs[b, sel[b, j]], j < n[b], in chunks of CHUNK: AffNet's patch, AffNet, the frame with
        the orientation and HardNet's patch, HardNet; then the descriptors' normalisation.  ``tap(stage, r0, rows, t)``, when
        given, sees each chunk's patches after the stage that cuts them ('affnet', 'hardnet') and the angles [B, K] at the end."""
        B, _, H, W = img.shape
        dev = img.device
        lafs, scores, desc = out = self._outputs(B, out_cap, dev)
        angles = None if tap is None else torch.empty(B, out_cap, dtype=torch.float32, device=dev)
        lib = _cabi.lib()
        ops = self._ops(dev)
        st = ops.st()
        wts = self._weights_on(dev)
        patches, col, act0, act1, xy = cnn_buffers(self._ws, dev)
        k = self.max_keypoints
        rows_all = B * out_cap
        d2 = desc.view(rows_all, 128)
        for r0 in range(0, rows_all, CHUNK):
            rows = min(CHUNK, rows_all - r0)
            _cabi.check(lib.og_kgftt_affnet_patches(ptr(img), B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), k, ptr(sel), ptr(n),
                                                    out_cap, r0, rows, ptr(patches), st), 'og_kgftt_affnet_patches')
            if tap is not None:
                tap('affnet', r0, rows, patches)
            _patch_cnn.run_cnn(ops, wts['affnet'], patches, rows, AFFNET_CONVS, col, (act0, act1), xy[:rows * 3].view(rows, 3))
            _cabi.check(lib.og_kgftt_frames(ptr(img), B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp), k, ptr(sel),
                                            ptr(n), out_cap, r0, rows, ptr(xy), int(self.upright), ptr(lafs), ptr(scores), ptr(angles),
                                            ptr(patches), st), 'og_kgftt_frames')
            if tap is not None:
                tap('hardnet', r0, rows, patches)
            _patch_cnn.run_cnn(ops, wts['hardnet'], patches, rows, HARDNET_CONVS, col, (act0, act1), d2[r0:r0 + rows])
        _cabi.check(lib.og_kgftt_desc_finish(ptr(desc), B, out_cap, ptr(n), st), 'og_kgftt_desc_finish')
        if tap is not None:
            tap('angles', 0, rows_all, angles)
        return out
