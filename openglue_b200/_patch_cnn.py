"""What the kornia patch-CNN front-ends (``GFTTAffNetHardNet``, ``DoGOpenCVAffNetHardNet``) share: kornia's AffNet / OriNet /
HardNet layer tables and checkpoint files, the eval-mode BatchNorm fold, checkpoint reading, the packed-weight cache, and the CNNs
as NHWC im2col + the Hopper GEMM over chunks of ``CHUNK`` patches."""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn

from . import _cabi
from ._cabi import ptr
from ._frontend import FrontEnd
from ._ops import _Ops
from .features import weights_key

PS = 32
CHUNK = 128                         # patches per CNN pass: the scratch is CHUNK * 1.34 MB (im2col of HardNet's 32x32x32 layer)
# (features index, in channels, out channels, stride) of the 3x3 convolutions; each is followed by BatchNorm2d(affine=False), ReLU.
# OriNet's stack has AffNet's shapes.
AFFNET_CONVS = [(0, 1, 16, 1), (3, 16, 16, 1), (6, 16, 32, 2), (9, 32, 32, 1), (12, 32, 64, 2), (15, 64, 64, 1)]
HARDNET_CONVS = [(0, 1, 32, 1), (3, 32, 32, 1), (6, 32, 64, 2), (9, 64, 64, 1), (12, 64, 128, 2), (15, 128, 128, 1)]
HEAD = 19                           # the 8x8 convolution of the networks (index 18 is Dropout)
BN_EPS = 1e-5
# the files kornia 0.6.3 caches in torch.hub.get_dir()/checkpoints, and where it fetches them from
CHECKPOINTS = {
    'affnet': ('AffNet.pth', 'https://github.com/ducha-aiki/affnet/raw/master/pretrained/AffNet.pth'),
    'orinet': ('OriNet.pth', 'https://github.com/ducha-aiki/affnet/raw/master/pretrained/OriNet.pth'),
    'hardnet': ('checkpoint_liberty_with_aug.pth',
                'https://github.com/DagnyT/hardnet/raw/master/pretrained/train_liberty_with_aug/checkpoint_liberty_with_aug.pth'),
}


def conv_stack(convs):
    layers = []
    for _, ci, co, s in convs:
        layers += [nn.Conv2d(ci, co, kernel_size=3, stride=s, padding=1, bias=False), nn.BatchNorm2d(co, affine=False), nn.ReLU()]
    return layers


class AffNet(nn.Module):
    """LAFAffNetShapeEstimator's parameters (``features.<i>``)"""

    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(*conv_stack(AFFNET_CONVS), nn.Dropout(0.25), nn.Conv2d(64, 3, kernel_size=8, bias=True), nn.Tanh(),
                                      nn.AdaptiveAvgPool2d(1))


class HardNet(nn.Module):
    """HardNet's parameters (``features.<i>``)"""

    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(*conv_stack(HARDNET_CONVS), nn.Dropout(0.3), nn.Conv2d(128, 128, kernel_size=8, bias=False),
                                      nn.BatchNorm2d(128, affine=False))


def fold(conv_w: torch.Tensor, bn: nn.BatchNorm2d, bias: Optional[torch.Tensor] = None):
    """eval-mode BatchNorm2d(affine=False) after a convolution, folded in float64: (W / s, (b - mean) / s), s = sqrt(var + eps);
    the weight as [Cout, (ky, kx, Cin)] for NHWC im2col"""
    s = torch.sqrt(bn.running_var.detach().double() + bn.eps)
    w = conv_w.detach().double() / s.view(-1, 1, 1, 1)
    b = ((bias.detach().double() if bias is not None else 0.0) - bn.running_mean.detach().double()) / s
    co = w.shape[0]
    return w.permute(0, 2, 3, 1).reshape(co, -1).float().contiguous(), b.float().contiguous()


def nhwc_head(conv: nn.Conv2d):
    """A convolution without BatchNorm after it, as (weight [Cout, (ky, kx, Cin)], bias [Cout])"""
    co = conv.weight.shape[0]
    return conv.weight.detach().permute(0, 2, 3, 1).reshape(co, -1).float().contiguous(), conv.bias.detach().float().contiguous()


def state_dict_of(src, name: str) -> dict:
    if isinstance(src, (str, os.PathLike)):
        # kornia's checkpoints hold training state beside the tensors, so they need the full unpickler, as kornia loads them
        src = torch.load(os.fspath(src), map_location='cpu', weights_only=False)
    if not isinstance(src, dict):
        raise TypeError(f'weights[{name!r}] must be a checkpoint path or a state dict, got {type(src)}')
    sd = src.get('state_dict', src)
    return {k: v for k, v in sd.items() if k.startswith('features.')}


def load_networks(owner: str, weights, checkpoints: dict, nets: dict) -> None:
    """Loads each of ``nets`` ({name: module with ``features``}) from ``weights[name]`` (a path or a state dict), or, with
    ``weights=None``, from kornia's cache ``torch.hub.get_dir()/checkpoints/<checkpoints[name][0]>``; never downloads."""
    if weights is None:
        root = os.path.join(torch.hub.get_dir(), 'checkpoints')
        weights = {}
        for name, (fname, url) in checkpoints.items():
            path = os.path.join(root, fname)
            if not os.path.isfile(path):
                keys = ', '.join(f'"{k}": ...' for k in checkpoints)
                raise FileNotFoundError(f'{path} not found: {owner} reads the {name} weights kornia caches there and never '
                                        f'downloads; fetch {url} into {root}, or pass weights={{{keys}}}')
            weights[name] = path
    if set(weights) != set(nets):
        raise ValueError(f'weights must have the keys {sorted(nets)}, got {sorted(weights)}')
    for name, net in nets.items():
        res = net.load_state_dict(state_dict_of(weights[name], name), strict=False)
        missing = [k for k in res.missing_keys if not k.endswith('num_batches_tracked')]   # older checkpoints lack the counter
        if missing or res.unexpected_keys:
            raise KeyError(f'{name} weights: missing {missing}, unexpected {res.unexpected_keys}')


def cnn_buffers(ws: dict, dev):
    """patches [CHUNK, 32, 32], im2col [CHUNK * 32 * 32 * 9 * 32], two activations [CHUNK * 32 * 32 * 32], xy [CHUNK, 3], cached in
    ``ws`` under ('cnn', dev)"""
    key = ('cnn', dev)
    if key not in ws:
        f = lambda n: torch.empty(n, dtype=torch.float32, device=dev)
        ws[key] = (f(CHUNK * PS * PS), f(CHUNK * PS * PS * 9 * 32), f(CHUNK * PS * PS * 32), f(CHUNK * PS * PS * 32), f(CHUNK * 3))
    return ws[key]


def run_cnn(ops: _Ops, layers, x: torch.Tensor, rows: int, convs, col, acts, out: Optional[torch.Tensor]):
    """One patch CNN on rows NHWC patches x [rows, 32, 32, 1]: 3x3 convolutions with folded BatchNorm and ReLU, then the 8x8
    convolution as one GEMM over the flattened 8x8xC activations into out [rows, Cout].  With ``out=None`` the head is skipped and
    the last activations [rows * 8 * 8, C] are returned."""
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
    if out is None:
        return x
    wt, b = layers[len(convs)]
    ops.linear(x.view(rows, -1), wt, b, out=out)
    return out


class CNNFrontEnd(FrontEnd):
    """A front-end that describes through the patch CNNs: ``precision`` picks the GEMM, ``_pack()`` gives the networks' GEMM
    layers ({name: [(W [Cout, K], bias [Cout])]}), and the networks run on their running BatchNorm statistics only"""

    def _ops(self, dev) -> _Ops:
        return _Ops(dev, _cabi.OG_PREC_FP32 if self.precision == 'fp32' else _cabi.OG_PREC_TF32X3)

    def _weights_on(self, dev):
        """``_pack()`` on dev, once per parameter / buffer version"""
        key = (weights_key(self), dev)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, {name: [(w.to(dev), b.to(dev)) for w, b in layers] for name, layers in self._pack().items()})
        return self._packed[1]

    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError(f'openglue_b200.{type(self).__name__} is an inference front-end (its networks run on their running '
                               'BatchNorm statistics); fine-tuning them is not built')
        return super().train(mode)
