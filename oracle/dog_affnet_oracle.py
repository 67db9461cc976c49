"""Pure-torch restatement of the kornia and kornia_moons pieces behind the reference's ``OPENCVDoGAffNetHardNet`` features
(models/features/opencv/dog_affnet_harnet.py on models/features/opencv/base.py): ``kornia_moons.feature.laf_from_opencv_SIFT_kpts``,
``K.tensor_to_image`` / ``K.image_to_tensor``, ``KF.OriNet(True)`` and ``KF.LAFOrienter(32, angle_detector=...)``.  AffNet,
HardNet and ``extract_patches_from_pyramid`` are oracle/kornia_gftt_oracle.py's and oracle/kornia_sift_oracle.py's.

TEST INFRASTRUCTURE (the checker, never the product path).  Neither kornia nor kornia_moons is a dependency of this project and
neither is installed where these files were written, so what follows restates kornia 0.6.3 and kornia_moons as recalled from their
published source, not as executed; parity with them is unverified where they are absent.  Everything runs in the dtype of its
input (float32 and float64) with the ATen operations in kornia's order.  The details taken from memory:
  - ``laf_from_opencv_SIFT_kpts(kpts, mrSize=6.0)``: ``laf_from_center_scale_ori(xy, 6 * size, -angle)`` on float32 tensors made
    from the keypoints' Python floats (``6 * size`` is multiplied in double, then rounded): the rotation
    ``angle_to_rotation_matrix(-angle) = [[cos, sin], [-sin, cos]]`` of ``deg2rad(t) = t * pi / 180``, then ``scale_laf``.
  - ``OriNet``: ``_normalize_input`` (Bessel std, eps 1e-6), six 3x3 convolutions with AffNet's shapes (1-16-16-32/2-32-64/2-64),
    each followed by ``BatchNorm2d(affine=False)`` and ReLU, ``Dropout(0.25)``, ``Conv2d(64, 2, kernel_size=8, padding=1,
    bias=True)`` (3x3 outputs on the 8x8 map), ``Tanh``, ``AdaptiveAvgPool2d(1)``; ``angle = atan2(y0 + 1e-8, y1 + 1e-8)``.
  - ``LAFOrienter(32, angle_detector=OriNet)``: 32-pixel patches by ``extract_patches_from_pyramid`` on the LAF as it is (not made
    upright), then ``set_laf_orientation(laf, rad2deg(angle) + get_laf_orientation(laf))``.
  - ``LAFAffNetShapeEstimator(True)`` preserves the input orientation (``preserve_orientation=True`` by default).

The pretrained checkpoints cannot be fetched here, so ``OriNet(True)`` loads seeded synthetic weights
(``synthetic_orinet_state_dict``), as the AffNet and HardNet stand-ins do; nothing touches the network.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn

from oracle import kornia_gftt_oracle as KG
from oracle import kornia_sift_oracle as KO

ORINET_SEED = 1703
PS = 32
ORINET_CONVS = KG.AFFNET_CONVS
ORINET_HEAD = 19


# ---- kornia.utils.image ----
def tensor_to_image(tensor: torch.Tensor, keepdim: bool = False) -> np.ndarray:
    """K.tensor_to_image: [1, C, H, W] -> [H, W] for one gray channel (numpy, the tensor's dtype)"""
    image = tensor.cpu().detach().numpy()
    if image.ndim == 4:
        image = image.transpose(0, 2, 3, 1)
        if image.shape[0] == 1 and not keepdim:
            image = image.squeeze(0)
    elif image.ndim == 3:
        image = image.transpose(1, 2, 0)
    if image.shape[-1] == 1 and not keepdim:
        image = image.squeeze(-1)
    return image


def image_to_tensor(image: np.ndarray, keepdim: bool = True) -> torch.Tensor:
    """K.image_to_tensor of a gray [H, W] image: [1, H, W] (keepdim) or [1, 1, H, W]"""
    t = torch.from_numpy(image)
    if t.dim() == 2:
        t = t.unsqueeze(0)
    else:
        t = t.permute(2, 0, 1)
    return t if keepdim else t.unsqueeze(0)


# ---- kornia_moons.feature ----
def laf_from_center_scale_ori(xy: torch.Tensor, scale: torch.Tensor, ori: torch.Tensor) -> torch.Tensor:
    """kornia.feature.laf.laf_from_center_scale_ori: xy [B, N, 2], scale [B, N, 1, 1], ori [B, N, 1] (degrees)"""
    B, N = xy.shape[:2]
    a = KO.deg2rad(ori.squeeze(-1))
    c, s = torch.cos(a), torch.sin(a)
    rot = torch.stack([c, s, -s, c], dim=-1).view(B, N, 2, 2)
    laf = torch.cat([rot, xy.unsqueeze(-1)], dim=-1)
    return KG.scale_laf(laf, scale)


def laf_from_opencv_SIFT_kpts(kpts, mrSize: float = 6.0, device=torch.device('cpu'), with_resp: bool = False):
    """kornia_moons.feature.laf_from_opencv_SIFT_kpts: cv2 keypoints -> LAFs [1, N, 2, 3] float32 (and responses [1, N])"""
    N = len(kpts)
    xy = torch.tensor([(k.pt[0], k.pt[1]) for k in kpts], device=device, dtype=torch.float).view(1, N, 2)
    scales = torch.tensor([(mrSize * k.size) for k in kpts], device=device, dtype=torch.float).view(1, N, 1, 1)
    angles = torch.tensor([(-k.angle) for k in kpts], device=device, dtype=torch.float).view(1, N, 1)
    laf = laf_from_center_scale_ori(xy, scales, angles).reshape(1, -1, 2, 3)
    if not with_resp:
        return laf
    resp = torch.tensor([k.response for k in kpts], device=device, dtype=torch.float).view(1, N, 1)
    return laf, resp


def lafs_from_kp(kp: torch.Tensor, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """laf_from_opencv_SIFT_kpts of keypoints stored as kp [B, N, 5] = (x, y, size, angle, response) float32, in ``dtype``: the
    scale is 6 size rounded to float32 (kornia_moons multiplies in double, then stores float32); float64 keeps it exact"""
    B, N = kp.shape[:2]
    k = kp.double()
    scale = (6.0 * k[..., 2]).to(torch.float32 if dtype == torch.float32 else torch.float64).to(dtype)
    return laf_from_center_scale_ori(k[..., :2].to(dtype), scale.view(B, N, 1, 1), (-k[..., 3]).to(dtype).view(B, N, 1))


# ---- kornia/feature/orientation.py: OriNet ----
def orinet_features() -> nn.Sequential:
    """OriNet.features"""
    return nn.Sequential(*KG._conv_stack(ORINET_CONVS), nn.Dropout(0.25), nn.Conv2d(64, 2, kernel_size=8, stride=1, padding=1, bias=True),
                         nn.Tanh(), nn.AdaptiveAvgPool2d(1))


def synthetic_orinet_state_dict(seed: int = ORINET_SEED) -> dict:
    """OriNet weights in kornia's key layout.  The head's pre-activation is its bias (0.8, -0.6) plus a term of std about 0.3, so
    the pooled (y0, y1) stays near (0.66, -0.54), far from atan2's singularity at 0, while the angle still varies from patch to patch"""
    sd, g = KG._synthetic(ORINET_CONVS, seed)
    sd[f'features.{ORINET_HEAD}.weight'] = torch.randn(2, 64, 8, 8, generator=g) * (0.3 / math.sqrt(0.5 * 64 * 64))
    sd[f'features.{ORINET_HEAD}.bias'] = torch.tensor([0.8, -0.6]) + 0.02 * torch.randn(2, generator=g)
    return sd


def orinet_in(dtype: torch.dtype, sd: dict = None) -> nn.Sequential:
    f = orinet_features()
    f.load_state_dict({k[len('features.'):]: v for k, v in (sd or synthetic_orinet_state_dict()).items()})
    return f.eval().to(dtype)


def orinet_xy(patches: torch.Tensor, features: nn.Module) -> torch.Tensor:
    """OriNet's pooled head output [n, 2] of patches [n, 1, 32, 32]"""
    return features(KG.normalize_input(patches)).view(-1, 2)


def orinet_angle(patches: torch.Tensor, features: nn.Module) -> torch.Tensor:
    """OriNet.forward: angles (radians) [n]"""
    xy = orinet_xy(patches, features)
    return torch.atan2(xy[:, 0] + 1e-8, xy[:, 1] + 1e-8)


def orinet_patches(img: torch.Tensor, laf: torch.Tensor) -> torch.Tensor:
    """OriNet's standardised input [B N, 1, 32, 32]: the patches of the LAFs as they are"""
    return KG.normalize_input(KO.extract_patches_from_pyramid(img, laf, PS).view(-1, 1, PS, PS))


def laf_orienter(laf: torch.Tensor, img: torch.Tensor, features: nn.Module, want_angles: bool = False):
    """LAFOrienter(32, angle_detector=OriNet).forward"""
    B, N = laf.shape[:2]
    if N == 0:
        return (laf, laf.new_zeros(B, 0)) if want_angles else laf
    patches = KO.extract_patches_from_pyramid(img, laf, PS).view(-1, 1, PS, PS)
    ang = orinet_angle(patches, features).view(B, N)
    prev = KO.get_laf_orientation(laf).view_as(ang)
    out = KO.set_laf_orientation(laf, KO.rad2deg(ang) + prev)
    return (out, ang) if want_angles else out


def describe(img: torch.Tensor, kp: torch.Tensor, orinet_sd: dict = None, affnet_sd: dict = None, hardnet_sd: dict = None) -> dict:
    """DoGOpenCVAffNetHardNet.detect_and_compute after the detector, in img's dtype, for one image [1, 1, H, W] and its selected
    keypoints kp [1, N, 5]: every stage's output"""
    aff, hard = (net.to(img.device) for net in KG.features_in(img.dtype, affnet_sd, hardnet_sd))
    ori = orinet_in(img.dtype, orinet_sd).to(img.device)
    with torch.no_grad():
        moons = lafs_from_kp(kp, img.dtype)
        if moons.shape[1] == 0:
            z = img.new_zeros(1, 0)
            return dict(moons_lafs=moons, aff_lafs=moons, angles=z, lafs=moons, descriptors=img.new_zeros(1, 0, 128))
        aff_lafs = KG.affnet_shape(moons, img, aff)
        lafs, ang = laf_orienter(aff_lafs, img, ori, want_angles=True)
        desc = KG.laf_descriptors(img, lafs, hard)
    return dict(moons_lafs=moons, aff_lafs=aff_lafs, angles=ang, lafs=lafs, descriptors=desc)


# ---- stand-ins with kornia's constructor signatures (the fixture script stubs kornia and kornia_moons with these); each
# records its inputs and outputs in ``calls`` ----
class OriNet(nn.Module):
    def __init__(self, pretrained: bool = False, eps: float = 1e-8):
        super().__init__()
        self.features = orinet_features()
        self.eps = eps
        if pretrained:                              # the synthetic weights stand in for the checkpoint; no download
            self.load_state_dict(synthetic_orinet_state_dict(), strict=True)
        self.eval()

    def forward(self, patch):
        return orinet_angle(patch, self.features)


class LAFOrienter(nn.Module):
    def __init__(self, patch_size: int = 32, num_angular_bins: int = 36, angle_detector=None):
        super().__init__()
        assert patch_size == PS and isinstance(angle_detector, OriNet), 'only LAFOrienter(32, angle_detector=OriNet) is restated'
        self.patch_size = patch_size
        self.angle_detector = angle_detector
        self.calls = []

    def forward(self, laf, img):
        out, ang = laf_orienter(laf, img, self.angle_detector.features, want_angles=True)
        self.calls.append(dict(lafs_in=laf, angles=ang, lafs_out=out))
        return out


class LAFAffNetShapeEstimator(KG.LAFAffNetShapeEstimator):
    def __init__(self, pretrained: bool = False, preserve_orientation: bool = True):
        super().__init__(pretrained, preserve_orientation)
        self.calls = []

    def forward(self, laf, img):
        out = super().forward(laf, img)
        self.calls.append(dict(lafs_in=laf, lafs_out=out))
        return out


HardNet = KG.HardNet
extract_patches_from_pyramid = KO.extract_patches_from_pyramid
