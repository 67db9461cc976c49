"""Drop-in for the reference's ``models.features.superpoint.model.SuperPointNet`` (SURVEY.md section 8, row f4): the detector /
descriptor front-end that feeds the matching core when features are not cached (reference models/matching_module.py:77-79,
inference.py).  Same constructor arguments, same ``state_dict`` keys (``conv1a.weight`` ... ``convDb.bias``: existing SuperPoint
checkpoints load), same ``forward(image [B,1,H,W]) -> (lafs [B,N,2,3], scores [B,N], descriptors [B,N,D])``.

All arithmetic runs in ``libopenglue_b200.so`` (``csrc/superpoint.cuh`` + the tensor-core GEMM): activations are NHWC, a 3x3
convolution is an im2col gather + one GEMM with bias / ReLU fused (3xTF32 wgmma; the 1-channel input layer and ``precision='fp32'``
run the exact fp32 kernel), then max-pool, channel norm, cell softmax, pixel heat map + non-maximum suppression + threshold + border
removal, ordered compaction, top-k and bilinear descriptor sampling as one kernel each.  The only host step of ``forward`` is
reading the per-image keypoint counts (the reference's ``torch.nonzero`` synchronises in the same place) to size the output;
``extract_padded`` sizes its outputs by a fixed capacity instead and keeps the counts on the device, so it never synchronises
and can be captured into a CUDA graph.
``SuperPointNetBn`` (BatchNorm variant, model.py:132-199: conv -> BatchNorm2d -> ReLU, also behind the two 1x1 heads) is the
same kernel schedule on folded weights: in eval mode ``BN(W x + b) = (g / sqrt(var + eps)) W x + (b - mean) g / sqrt(var + eps) + beta``,
folded once in float64 on the host.  There is no CPU path.
"""
from __future__ import annotations

import pathlib
from typing import Optional, Union

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr
from ._ops import _Ops
from .features import padded_capacity, weights_key

__all__ = ['SuperPointNet', 'SuperPointNetBn']

_MAX_CAND = 16384


class SuperPointNet(nn.Module):
    def __init__(self, max_keypoints: int = -1, descriptor_dim: int = 256, nms_kernel: int = 9, remove_borders_size: int = 4,
                 keypoint_threshold: float = 0.0, weights: Optional[Union[str, pathlib.Path]] = None, precision: str = 'tf32x3'):
        super().__init__()
        self.max_keypoints, self.descriptor_dim, self.nms_kernel = max_keypoints, descriptor_dim, nms_kernel
        self.remove_borders_size, self.keypoint_threshold = remove_borders_size, keypoint_threshold
        self.precision = precision
        conv = lambda i, o: nn.Conv2d(i, o, kernel_size=(3, 3), stride=(1, 1), padding=1)
        self.layers_channels = [[1, 64, 64, 64], [64, 64, 64, 64], [64, 128, 128, 128], [128, 128, 128, 128]]    # model.py:35-40
        for i, ch in enumerate(self.layers_channels):
            setattr(self, f'conv{i + 1}a', conv(ch[0], ch[1]))
            setattr(self, f'conv{i + 1}b', conv(ch[2], ch[3]))
        self.convPa = conv(128, 256)
        self.convPb = nn.Conv2d(256, 65, kernel_size=1, stride=1, padding=0)
        self.convDa = conv(128, 256)
        self.convDb = nn.Conv2d(256, descriptor_dim, kernel_size=1, stride=1, padding=0)
        self._packed = None
        if weights is not None:
            print(self.load_state_dict(torch.load(str(weights), map_location='cpu'), strict=True))

    # ------------------------------------------------------------------ weights: [Cout, Cin, 3, 3] -> [Cout, (3 ky + kx) Cin + ci]
    def _conv_params(self, name, m):
        """(weight [Cout, Cin, kh, kw], bias [Cout]) the kernels run for convolution `name` (hook: SuperPointNetBn folds its BatchNorm in)"""
        return m.weight.detach(), m.bias.detach()

    def _weights(self):
        key = weights_key(self)
        if self._packed is None or self._packed[0] != key:
            w = {}
            for name, m in self.named_children():
                if isinstance(m, nn.Conv2d):
                    wt, bias = self._conv_params(name, m)
                    co, ci, kh, kw = wt.shape
                    w[name] = (wt.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous(), bias.contiguous())
            self._packed = (key, w)
        return self._packed[1]

    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError('openglue_b200.SuperPointNet is the inference front-end (the reference keeps its feature extractor '
                               'in eval mode unless it is fine-tuned, matching_module.py:77-79); fine-tuning it is not built')
        return super().train(mode)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, image: torch.Tensor, mask=None):
        dev = image.device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200.SuperPointNet needs CUDA tensors (sm_90a); there is no CPU path')
        if image.dim() != 4 or image.shape[1] != 1 or image.shape[2] % 8 or image.shape[3] % 8:
            raise ValueError('image must be [B, 1, H, W] with H, W multiples of 8')
        H, W = image.shape[2], image.shape[3]
        probs, coarse = self._network(image)
        return self._keypoints(probs, coarse, H, W)

    def _ops(self, dev):
        return _Ops(dev, _cabi.OG_PREC_FP32 if self.precision == 'fp32' else _cabi.OG_PREC_TF32X3)

    def _network(self, image: torch.Tensor):
        """The layers (model.py:61-78): image [B, 1, H, W] -> (probs [B hc wc, 65] after the cell softmax, coarse [B hc wc, D] with
        unit rows), NHWC, hc = H / 8, wc = W / 8."""
        dev = image.device
        B, _, H, W = image.shape
        x = image.detach().float().contiguous()                       # [B, 1, H, W] == NHWC with one channel
        ops = self._ops(dev)
        lib = ops.lib
        wts = self._weights()
        with torch.cuda.device(dev):
            st = ops.st()
            col = ops.empty(B * H * W * 9 * 64)                          # im2col scratch, sized for the largest layer (full resolution, 64 channels)

            def conv3(t, h, w, cin, name, relu=True):
                wp, bias = wts[name]
                a = col[:B * h * w * 9 * cin].view(B * h * w, 9 * cin)
                _cabi.check(lib.og_sp_im2col3x3(ptr(t), B, h, w, cin, ptr(a), st), 'og_sp_im2col3x3')
                return ops.linear(a, wp, bias, relu=relu)               # [B h w, cout] = NHWC

            h, w, cin = H, W, 1
            for i, ch in enumerate(self.layers_channels):
                x = conv3(x, h, w, cin, f'conv{i + 1}a'); cin = ch[1]
                x = conv3(x, h, w, cin, f'conv{i + 1}b'); cin = ch[3]
                if i != 3:
                    y = ops.empty(B * (h // 2) * (w // 2), cin)
                    _cabi.check(lib.og_sp_maxpool2x2(ptr(x), B, h, w, cin, ptr(y), st), 'og_sp_maxpool2x2')
                    x, h, w = y, h // 2, w // 2
            hc, wc = h, w
            # descriptor head (model.py:68-71)
            da = conv3(x, hc, wc, 128, 'convDa')
            coarse = ops.linear(da, *wts['convDb'])
            _cabi.check(lib.og_row_normalize(ptr(coarse), coarse.shape[0], self.descriptor_dim, 0, 0.0, st), 'og_row_normalize')
            # detector head (model.py:73-75) + heat map, NMS, threshold, borders (model.py:82-99)
            pa = conv3(x, hc, wc, 128, 'convPa')
            probs = ops.linear(pa, *wts['convPb'])                       # [B hc wc, 65]
            _cabi.check(lib.og_softmax_rows(ptr(probs), 65, probs.shape[0], 65, st), 'og_softmax_rows')
            self.last_probs = probs.view(B, hc, wc, 65)                  # kept for inspection / tests
        return probs, coarse

    @torch.no_grad()
    def extract_padded(self, image: torch.Tensor, capacity: Optional[int] = None):
        """``forward`` for a batch whose images keep their own keypoint counts, without a host synchronisation.

        image [B,1,H,W] -> (lafs [B,K,2,3], scores [B,K], descriptors [B,K,D], num_keypoints [B] int32, overflow [B] int32), all
        on the image's device, K = ``capacity`` (default ``max_keypoints``).  Rows [0, num_keypoints[b]) of image b are what
        ``forward(image[b:b+1])`` returns (its own top-k, raster order when it keeps every keypoint; no ``min_stack``); the rows
        past them are 0, as ``pad_features`` writes them.

        ``overflow[b] = 1`` where ``forward`` would raise or K cuts the image: more non-maximum-suppression survivors than the
        16384 candidates an image holds (the first 16384 in raster order are used), or more kept keypoints than K (the first K
        in output order are kept and num_keypoints[b] = K).  Check it whenever the results are next read on the host."""
        K = padded_capacity(self.max_keypoints, capacity)
        if image.dim() != 4 or image.shape[1] != 1 or image.shape[2] % 8 or image.shape[3] % 8:
            raise ValueError('image must be [B, 1, H, W] with H, W multiples of 8')
        if image.device.type != 'cuda':
            raise RuntimeError('openglue_b200.SuperPointNet needs CUDA tensors (sm_90a); there is no CPU path')
        H, W = image.shape[2], image.shape[3]
        probs, coarse = self._network(image)
        return self._keypoints_padded(probs, coarse, H, W, K)

    def _candidates(self, probs: torch.Tensor, H: int, W: int, ops: _Ops):
        """heat map, NMS, threshold and borders, then the ordered compaction: (cand_idx, cand_score [B, cap], count [B], cap)"""
        dev = probs.device
        hc, wc = H // 8, W // 8
        B = probs.shape[0] // (hc * wc)
        lib, st = ops.lib, ops.st()
        heat = ops.empty(B, H, W)
        _cabi.check(lib.og_sp_heat_nms(ptr(probs), B, hc, wc, int(self.nms_kernel), float(self.keypoint_threshold), int(self.remove_borders_size),
                                       ptr(heat), st), 'og_sp_heat_nms')
        cap = min(H * W, _MAX_CAND)
        cand_idx = torch.empty(B, cap, dtype=torch.int32, device=dev)
        cand_score = ops.empty(B, cap)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        _cabi.check(lib.og_sp_compact(ptr(heat), B, H * W, cap, ptr(cand_idx), ptr(cand_score), ptr(count), st),
                    'og_sp_compact')
        return cand_idx, cand_score, count, cap

    def _keypoints_padded(self, probs: torch.Tensor, coarse: torch.Tensor, H: int, W: int, K: int):
        """The post-processing of extract_padded from the layers' outputs (as _keypoints), at K rows per image"""
        dev = probs.device
        hc, wc = H // 8, W // 8
        B = probs.shape[0] // (hc * wc)
        d = self.descriptor_dim
        ops = self._ops(dev)
        lib = ops.lib
        i32 = dict(dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            st = ops.st()
            cand_idx, cand_score, count, cap = self._candidates(probs, H, W, ops)
            n_out, mode, overflow = torch.empty(B, **i32), torch.empty(B, **i32), torch.zeros(B, **i32)
            _cabi.check(lib.og_keypoint_counts(ptr(count), B, cap, int(self.max_keypoints), K, ptr(n_out), ptr(mode), ptr(overflow), st),
                        'og_keypoint_counts')
            # the outputs start at 0: select and sampling write rows [0, n_out[b]) only
            kpts, scores, desc = ops.zeros(B, K, 2), ops.zeros(B, K), ops.zeros(B, K, d)
            # max_count = cap: the sort's shared memory covers any count the device holds
            _cabi.check(lib.og_sp_select(ptr(cand_idx), ptr(cand_score), ptr(count), ptr(n_out), ptr(mode), B, cap, W, K, cap, ptr(kpts), ptr(scores), st),
                        'og_sp_select')
            _cabi.check(lib.og_sp_sample_desc(ptr(coarse), B, hc, wc, d, ptr(kpts), ptr(n_out), K, K, 8, ptr(desc), st), 'og_sp_sample_desc')
            real = (torch.arange(K, device=dev) < n_out[:, None]).float()
            lafs = ops.zeros(B, K, 2, 3)                                 # identity frame + position on the real rows (model.py:119-127)
            lafs[:, :, 0, 0] = real
            lafs[:, :, 1, 1] = real
            lafs[:, :, :, 2] = kpts
        return lafs, scores, desc, n_out, overflow

    def _keypoints(self, probs: torch.Tensor, coarse: torch.Tensor, H: int, W: int):
        """The post-processing of forward (model.py:84-129) from the layers' outputs: probs [B hc wc, 65] and coarse [B hc wc, D]
        (NHWC, hc = H / 8, wc = W / 8, CUDA float32) -> (lafs [B,N,2,3], scores [B,N], descriptors [B,N,D])."""
        dev = probs.device
        hc, wc = H // 8, W // 8
        B = probs.shape[0] // (hc * wc)
        ops = self._ops(dev)
        lib = ops.lib
        with torch.cuda.device(dev):
            st = ops.st()
            cand_idx, cand_score, count, cap = self._candidates(probs, H, W, ops)
            counts = count.tolist()                                      # the one host synchronisation (the reference's nonzero)
            if max(counts) > cap:
                raise RuntimeError(f'{max(counts)} keypoints survive non-maximum suppression in one image (capacity {cap}): raise keypoint_threshold')
            k = self.max_keypoints
            keep = [c if (k == -1 or k >= c) else k for c in counts]    # top_k_keypoints (utils.py:34-39)
            mode = [0 if (k == -1 or k >= c) else 1 for c in counts]
            n = min(keep)
            if any(v != n for v in keep):                                # min_stack (models/features/utils.py:28-56): top-k of every image
                keep, mode = [n] * B, [1] * B
            d = self.descriptor_dim
            if n == 0:
                z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
                return z(B, 0, 2, 3), z(B, 0), z(B, 0, d)
            n_out = torch.tensor(keep, dtype=torch.int32, device=dev)
            modes = torch.tensor(mode, dtype=torch.int32, device=dev)
            kpts, scores = ops.empty(B, n, 2), ops.empty(B, n)
            _cabi.check(lib.og_sp_select(ptr(cand_idx), ptr(cand_score), ptr(count), ptr(n_out), ptr(modes), B, cap, W, n, max(counts), ptr(kpts), ptr(scores), st),
                        'og_sp_select')
            desc = ops.empty(B, n, d)
            _cabi.check(lib.og_sp_sample_desc(ptr(coarse), B, hc, wc, d, ptr(kpts), ptr(n_out), n, n, 8, ptr(desc), st), 'og_sp_sample_desc')
            lafs = torch.zeros(B, n, 2, 3, dtype=torch.float32, device=dev)  # identity frame + position (model.py:119-127)
            lafs[:, :, 0, 0] = 1.0
            lafs[:, :, 1, 1] = 1.0
            lafs[:, :, :, 2] = kpts
        return lafs, scores, desc


class SuperPointNetBn(SuperPointNet):
    """Drop-in for the reference's ``SuperPointNetBn`` (models/features/superpoint/model.py:132-199): every convolution is followed by
    a BatchNorm2d (``bn1a`` ... ``bn4b``, ``bnPa``, ``bnPb``, ``bnDa``, ``bnDb``; same ``state_dict`` keys, same checkpoint format
    ``{'model_state_dict': ...}`` with the U-Net style key names renamed by ``rename_weights_keys``).  Inference only: the
    normalisation uses the running statistics and is folded into the convolution it follows, so the forward pass is
    ``SuperPointNet``'s kernel schedule, unchanged."""

    def __init__(self, max_keypoints: int = -1, descriptor_dim: int = 256, nms_kernel: int = 9, remove_borders_size: int = 4,
                 keypoint_threshold: float = 0.0, weights: Optional[Union[str, pathlib.Path]] = None, precision: str = 'tf32x3'):
        super().__init__(max_keypoints, descriptor_dim, nms_kernel, remove_borders_size, keypoint_threshold, weights=None, precision=precision)
        for i, ch in enumerate(self.layers_channels):                       # model.py:141-148
            setattr(self, f'bn{i + 1}a', nn.BatchNorm2d(ch[1]))
            setattr(self, f'bn{i + 1}b', nn.BatchNorm2d(ch[3]))
        self.bnPa, self.bnPb = nn.BatchNorm2d(256), nn.BatchNorm2d(65)
        self.bnDa, self.bnDb = nn.BatchNorm2d(256), nn.BatchNorm2d(256)
        if weights is not None:                                             # model.py:173-178
            sd = self.rename_weights_keys(torch.load(str(weights), map_location='cpu')['model_state_dict'])
            print(self.load_state_dict(sd, strict=True))

    _RENAMES = [('inc.conv.conv.0', 'conv1a'), ('inc.conv.conv.1', 'bn1a'), ('inc.conv.conv.3', 'conv1b'), ('inc.conv.conv.4', 'bn1b')] + [
        (f'down{i}.mpconv.1.conv.{j}', f'{kind}{i + 1}{ab}') for i in (1, 2, 3)
        for j, kind, ab in ((0, 'conv', 'a'), (1, 'bn', 'a'), (3, 'conv', 'b'), (4, 'bn', 'b'))]

    @staticmethod
    def rename_weights_keys(state_dict):
        """checkpoint key names of the BatchNorm SuperPoint release -> this module's (model.py:151-171)"""
        for key in list(state_dict.keys()):
            new = key
            for old, repl in SuperPointNetBn._RENAMES:
                new = new.replace(old, repl)
            state_dict[new] = state_dict.pop(key)
        return state_dict

    def _conv_params(self, name, m):
        bn = getattr(self, 'bn' + name[4:])                                 # conv1a -> bn1a, convPb -> bnPb
        g = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        wt = m.weight.detach().double() * g.view(-1, 1, 1, 1)
        bias = (m.bias.detach().double() - bn.running_mean.detach().double()) * g + bn.bias.detach().double()
        return wt.float(), bias.float()
