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

import os
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr, stream
from ._ops import _Ops
from .features import padded_capacity

__all__ = ['GFTTAffNetHardNet']

MAX_FEATURES = 8192                 # keypoints per image the detector and run_nms sort in one CTA's shared memory
PS = 32
CHUNK = 128                         # patches per CNN pass: the scratch is CHUNK * 1.34 MB (im2col of HardNet's 32x32x32 layer)
# (features index, in channels, out channels, stride) of the 3x3 convolutions; each is followed by BatchNorm2d(affine=False), ReLU
AFFNET_CONVS = [(0, 1, 16, 1), (3, 16, 16, 1), (6, 16, 32, 2), (9, 32, 32, 1), (12, 32, 64, 2), (15, 64, 64, 1)]
HARDNET_CONVS = [(0, 1, 32, 1), (3, 32, 32, 1), (6, 32, 64, 2), (9, 64, 64, 1), (12, 64, 128, 2), (15, 128, 128, 1)]
HEAD = 19                           # the 8x8 convolution of both networks (index 18 is Dropout)
BN_EPS = 1e-5
# the files kornia 0.6.3 caches in torch.hub.get_dir()/checkpoints, and where it fetches them from
CHECKPOINTS = {
    'affnet': ('AffNet.pth', 'https://github.com/ducha-aiki/affnet/raw/master/pretrained/AffNet.pth'),
    'hardnet': ('checkpoint_liberty_with_aug.pth',
                'https://github.com/DagnyT/hardnet/raw/master/pretrained/train_liberty_with_aug/checkpoint_liberty_with_aug.pth'),
}
ORIENT_SMOOTH = (0.33, 0.34, 0.33)  # PatchDominantGradientOrientation's fixed angular smoothing


def _conv_stack(convs):
    layers = []
    for _, ci, co, s in convs:
        layers += [nn.Conv2d(ci, co, kernel_size=3, stride=s, padding=1, bias=False), nn.BatchNorm2d(co, affine=False), nn.ReLU()]
    return layers


class _AffNet(nn.Module):
    """LAFAffNetShapeEstimator's parameters (``features.<i>``)"""

    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(*_conv_stack(AFFNET_CONVS), nn.Dropout(0.25), nn.Conv2d(64, 3, kernel_size=8, bias=True), nn.Tanh(),
                                      nn.AdaptiveAvgPool2d(1))


class _HardNet(nn.Module):
    """HardNet's parameters (``features.<i>``)"""

    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(*_conv_stack(HARDNET_CONVS), nn.Dropout(0.3), nn.Conv2d(128, 128, kernel_size=8, bias=False),
                                      nn.BatchNorm2d(128, affine=False))


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


def _fold(conv_w: torch.Tensor, bn: nn.BatchNorm2d, bias: Optional[torch.Tensor] = None):
    """eval-mode BatchNorm2d(affine=False) after a convolution, folded in float64: (W / s, (b - mean) / s), s = sqrt(var + eps);
    the weight as [Cout, (ky, kx, Cin)] for NHWC im2col"""
    s = torch.sqrt(bn.running_var.detach().double() + bn.eps)
    w = conv_w.detach().double() / s.view(-1, 1, 1, 1)
    b = ((bias.detach().double() if bias is not None else 0.0) - bn.running_mean.detach().double()) / s
    co = w.shape[0]
    return w.permute(0, 2, 3, 1).reshape(co, -1).float().contiguous(), b.float().contiguous()


def _state_dict_of(src, name: str) -> dict:
    if isinstance(src, (str, os.PathLike)):
        # kornia's checkpoints hold training state beside the tensors, so they need the full unpickler, as kornia loads them
        src = torch.load(os.fspath(src), map_location='cpu', weights_only=False)
    if not isinstance(src, dict):
        raise TypeError(f'weights[{name!r}] must be a checkpoint path or a state dict, got {type(src)}')
    sd = src.get('state_dict', src)
    return {k: v for k, v in sd.items() if k.startswith('features.')}


class GFTTAffNetHardNet(nn.Module):
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
        self._ws, self._packed = {}, None
        self.load_weights(weights)

    def extra_repr(self) -> str:
        return (f'max_keypoints={self.max_keypoints}, perform_nms={self.perform_nms}, nms_diameter={self.nms_diameter}, '
                f'upright={self.upright}, precision={self.precision!r}')

    # ------------------------------------------------------------------ weights
    def load_weights(self, weights=None) -> None:
        """Loads AffNet and HardNet from ``weights`` (see the class) or from kornia's cache; never downloads."""
        if weights is None:
            root = os.path.join(torch.hub.get_dir(), 'checkpoints')
            weights = {}
            for name, (fname, url) in CHECKPOINTS.items():
                path = os.path.join(root, fname)
                if not os.path.isfile(path):
                    raise FileNotFoundError(f'{path} not found: GFTTAffNetHardNet reads the {name} weights kornia caches there and never '
                                            f'downloads; fetch {url} into {root}, or pass weights={{"affnet": ..., "hardnet": ...}}')
                weights[name] = path
        if set(weights) != {'affnet', 'hardnet'}:
            raise ValueError(f"weights must have the keys 'affnet' and 'hardnet', got {sorted(weights)}")
        for name, net in (('affnet', self.detector.aff), ('hardnet', self.descriptor.descriptor)):
            res = net.load_state_dict(_state_dict_of(weights[name], name), strict=False)
            missing = [k for k in res.missing_keys if not k.endswith('num_batches_tracked')]   # older checkpoints lack the counter
            if missing or res.unexpected_keys:
                raise KeyError(f'{name} weights: missing {missing}, unexpected {res.unexpected_keys}')

    def _weights(self):
        """The networks' GEMM weights, packed once per parameter / buffer version: {name: [(W [Cout, K], bias [Cout])]}"""
        key = tuple((t._version, t.data_ptr()) for t in list(self.parameters()) + list(self.buffers()))
        if self._packed is None or self._packed[0] != key:
            if not self.upright:
                w = self.detector.ori.angle_detector.angular_smooth.weight.detach().flatten().tolist()
                if any(abs(a - b) > 0 for a, b in zip(w, torch.tensor(ORIENT_SMOOTH).tolist())):
                    raise ValueError(f'the orienter smooths its histogram with kornia\'s fixed {ORIENT_SMOOTH}, got {w}')
            packed = {}
            for name, net, convs in (('affnet', self.detector.aff.features, AFFNET_CONVS), ('hardnet', self.descriptor.descriptor.features,
                                                                                            HARDNET_CONVS)):
                layers = [_fold(net[i].weight, net[i + 1]) for i, *_ in convs]
                head = net[HEAD]
                if name == 'affnet':
                    layers.append((head.weight.detach().permute(0, 2, 3, 1).reshape(3, -1).float().contiguous(),
                                   head.bias.detach().float().contiguous()))
                else:
                    layers.append(_fold(head.weight, net[HEAD + 1]))
                packed[name] = layers
            dev = next(self.parameters()).device
            self._packed = (key, packed, dev)
        return self._packed[1]

    def _weights_on(self, dev):
        w = self._weights()
        if self._packed[2] != dev:
            self._packed = (self._packed[0], {k: [(a.to(dev), b.to(dev)) for a, b in v] for k, v in w.items()}, dev)
        return self._packed[1]

    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError('openglue_b200.GFTTAffNetHardNet is the inference front-end (AffNet and HardNet run on their running '
                               'BatchNorm statistics); fine-tuning them is not built')
        return super().train(mode)

    # ------------------------------------------------------------------ device work
    def _workspace(self, dev, B, H, W):
        lib = _cabi.lib()
        key = (dev, B, H, W)
        if key not in self._ws:
            sizes = [k for k in self._ws if k[0] != 'cnn']
            while len(sizes) >= 2:                                      # the two image sizes of a pair batch stay cached
                del self._ws[sizes.pop(0)]
            n = _cabi.check_size(lib.og_kgftt_workspace_bytes(B, H, W, self.max_keypoints), 'og_kgftt_workspace_bytes')
            m = _cabi.check_size(lib.og_ksift_select_workspace_bytes(B, self.max_keypoints), 'og_ksift_select_workspace_bytes')
            self._ws[key] = (torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(m, dtype=torch.uint8, device=dev))
        return self._ws[key]

    def _cnn_buffers(self, dev):
        """patches [CHUNK, 32, 32], im2col [CHUNK * 32 * 32 * 9 * 32], two activations [CHUNK * 32 * 32 * 32], xy [CHUNK, 3]"""
        key = ('cnn', dev)
        if key not in self._ws:
            f = lambda n: torch.empty(n, dtype=torch.float32, device=dev)
            self._ws[key] = (f(CHUNK * PS * PS), f(CHUNK * PS * PS * 9 * 32), f(CHUNK * PS * PS * 32), f(CHUNK * PS * PS * 32), f(CHUNK * 3))
        return self._ws[key]

    @staticmethod
    def _image(images: torch.Tensor) -> torch.Tensor:
        if not torch.is_tensor(images) or images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f'images must be [B, 1, H, W], got {tuple(images.shape) if torch.is_tensor(images) else type(images)}')
        if images.device.type != 'cuda':
            raise RuntimeError('openglue_b200.GFTTAffNetHardNet needs CUDA tensors (sm_90a); there is no CPU path')
        if images.dtype == torch.uint8:
            return (images.float() / 255.).contiguous()
        if not images.is_floating_point():
            raise ValueError(f'images must be float in [0, 1] or uint8, got {images.dtype}')
        return images.detach().float().contiguous()

    def _detect_select(self, img: torch.Tensor, min_stack: bool):
        """The pyramid, detector and run_nms of B images: (ws, det_lafs, det_resp, sel, n_sel)"""
        B, _, H, W = img.shape
        dev, k = img.device, self.max_keypoints
        lib = _cabi.lib()
        st = stream(dev)
        ws, work = self._workspace(dev, B, H, W)
        det_lafs = torch.empty(B, k, 2, 3, dtype=torch.float32, device=dev)
        det_resp = torch.empty(B, k, dtype=torch.float32, device=dev)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        _cabi.check(lib.og_kgftt_pyramid(ptr(img), B, H, W, k, ptr(ws), ws.numel(), st), 'og_kgftt_pyramid')
        _cabi.check(lib.og_kgftt_detect(B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp), ptr(count), st), 'og_kgftt_detect')
        sel = torch.empty(B, k, dtype=torch.int32, device=dev)
        n_sel = torch.empty(B, dtype=torch.int32, device=dev)
        _cabi.check(lib.og_ksift_select(ptr(det_lafs), ptr(det_resp), ptr(count), B, H, W, k, int(self.perform_nms), self.nms_diameter,
                                        self.max_keypoints, int(min_stack), ptr(work), work.numel(), ptr(sel), ptr(n_sel), st),
                    'og_ksift_select')
        return ws, det_lafs, det_resp, sel, n_sel

    def _cnn(self, ops: _Ops, layers, x: torch.Tensor, rows: int, convs, col, acts, out: torch.Tensor):
        """One patch CNN on rows NHWC patches x [rows, 32, 32, 1]: 3x3 convolutions with folded BatchNorm and ReLU, then the 8x8
        convolution as one GEMM over the flattened 8x8xC activations into out [rows, Cout]"""
        lib, st = ops.lib, ops.st()
        h = w = PS
        for li, (_, ci, co, s) in enumerate(convs):
            wt, b = layers[li]
            if s == 1:
                _cabi.check(lib.og_sp_im2col3x3(ptr(x), rows, h, w, ci, ptr(col), st), 'og_sp_im2col3x3')
            else:
                _cabi.check(lib.og_kgftt_im2col3x3_s2(ptr(x), rows, h, w, ci, ptr(col), st), 'og_kgftt_im2col3x3_s2')
                h, w = (h + 1) // 2, (w + 1) // 2
            a = col[:rows * h * w * 9 * ci].view(rows * h * w, 9 * ci)
            y = acts[li % 2][:rows * h * w * co].view(rows * h * w, co)
            x = ops.linear(a, wt, b, relu=True, out=y)
        wt, b = layers[-1]
        ops.linear(x.view(rows, -1), wt, b, out=out)

    def _describe(self, img, ws, det_lafs, det_resp, sel, n, out_cap):
        B, _, H, W = img.shape
        dev = img.device
        f32 = dict(dtype=torch.float32, device=dev)
        lafs, scores, desc = torch.empty(B, out_cap, 2, 3, **f32), torch.empty(B, out_cap, **f32), torch.empty(B, out_cap, 128, **f32)
        lib = _cabi.lib()
        ops = _Ops(dev, _cabi.OG_PREC_FP32 if self.precision == 'fp32' else _cabi.OG_PREC_TF32X3)
        st = ops.st()
        wts = self._weights_on(dev)
        patches, col, act0, act1, xy = self._cnn_buffers(dev)
        k = self.max_keypoints
        rows_all = B * out_cap
        d2 = desc.view(rows_all, 128)
        for r0 in range(0, rows_all, CHUNK):
            rows = min(CHUNK, rows_all - r0)
            _cabi.check(lib.og_kgftt_affnet_patches(ptr(img), B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), k, ptr(sel), ptr(n), out_cap, r0,
                                                    rows, ptr(patches), st), 'og_kgftt_affnet_patches')
            self._cnn(ops, wts['affnet'], patches, rows, AFFNET_CONVS, col, (act0, act1), xy[:rows * 3].view(rows, 3))
            _cabi.check(lib.og_kgftt_frames(ptr(img), B, H, W, k, ptr(ws), ws.numel(), ptr(det_lafs), ptr(det_resp), k, ptr(sel), ptr(n),
                                            out_cap, r0, rows, ptr(xy), int(self.upright), ptr(lafs), ptr(scores), None, ptr(patches), st),
                        'og_kgftt_frames')
            self._cnn(ops, wts['hardnet'], patches, rows, HARDNET_CONVS, col, (act0, act1), d2[r0:r0 + rows])
        _cabi.check(lib.og_kgftt_desc_finish(ptr(desc), B, out_cap, ptr(n), st), 'og_kgftt_desc_finish')
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
