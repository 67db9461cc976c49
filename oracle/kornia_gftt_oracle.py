"""Pure-torch restatement of the kornia pieces behind the reference's ``GFTTAffNetHardNet`` features (models/features/hardnet.py
on models/features/base.py): ``ScaleSpaceDetector`` with ``CornerGFTT``, ``ConvQuadInterp3d(10, 1e-5)``, ``ScalePyramid(3, 1.6, 32,
double_image=False)``, ``LAFAffNetShapeEstimator(True)`` and ``LAFOrienter(19)`` / ``PassLAF``, then ``LAFDescriptor(None, 32)``,
whose ``None`` is kornia's ``HardNet(True)``.

TEST INFRASTRUCTURE (the checker, never the product path).  kornia is not a dependency of this project.  The pieces shared with
the DoG front-end (the pyramid, ``conv_quad_interp3d``, the LAF helpers, ``extract_patches_from_pyramid``, the orienter) are
imported from oracle/kornia_sift_oracle.py; this module adds what ``GFTTAffNetHardNet`` needs on top, restating kornia 0.6.3 in
the dtype of its input (float32 and float64) with the ATen operations in kornia's order.

What this restatement takes kornia 0.6.3 to do.  kornia is not installed where these files were written, so each answer is from
that release's published source as recalled, not from an execution; ``test_gftt_hardnet_host.py::test_parity_with_kornia`` is
the only check against kornia itself and runs only where kornia is installed:
  - ``ScaleSpaceDetector.detect`` with ``scale_space_response=False`` runs the response on the ``n_levels + 3 = 6`` Gaussian levels
    of an octave as a ``[B * 6, 1, h, w]`` batch with the level sigmas, then drops the last level (``extra_levels`` is odd: "3rd
    extra level is required for DoG only"), so levels 0 .. 4 enter the 3-D NMS.  ``minima_are_also_good=False``: maxima only.
  - ``ConvQuadInterp3d(10, eps=1e-5)``: ``eps`` scales a ``torch.rand`` jitter added to every Hessian before the solve.  That is
    random, so the restatement (and the kernels) take it at zero; a strict-maximum voxel with a singular Hessian, where the jitter
    would matter, is not solved, as in ``conv_quad_interp3d`` without it.
  - ``_normalize_input`` of AffNet and HardNet: ``torch.std_mean`` over the patch with the default Bessel correction (n - 1),
    then ``(x - mean) / (std + 1e-6)``.
  - ``LAFAffNetShapeEstimator(pretrained, preserve_orientation=True)``: orientation preserved by default.
  - ``LAFOrienter``'s ``PatchDominantGradientOrientation`` holds its angular smoothing as ``nn.Conv1d(1, 1, 3, bias=False,
    padding_mode='circular')`` with the fixed weight [0.33, 0.34, 0.33], so a reference module's ``state_dict`` carries
    ``detector.ori.angle_detector.angular_smooth.weight``; its Gaussian weighting is a plain attribute.
  - ``gftt_response``: Sobel ``spatial_gradient`` (normalised, replicate border), ``gaussian_blur2d((7, 7), (1, 1))`` (reflect) of
    dx², dy² and dx dy, ``min(0.5 (tr + sqrt|tr² - 4 det|), 0.5 (tr - sqrt|tr² - 4 det|))``, times ``sigma ** 4`` of the level.
  - Dropout is the identity in eval mode; ``AdaptiveAvgPool2d(1)`` after AffNet's 8x8 convolution averages one value.

The pretrained checkpoints cannot be fetched here, so the stand-ins' ``pretrained=True`` load seeded synthetic weights
(``synthetic_affnet_state_dict`` / ``synthetic_hardnet_state_dict``) and never touch the network.
"""
from __future__ import annotations

import hashlib
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import kornia_sift_oracle as KO

AFFNET_SEED, HARDNET_SEED = 1701, 1702
PS = 32
# (features index of the conv, in channels, out channels, stride); each is followed by BatchNorm2d(affine=False) and ReLU
AFFNET_CONVS = [(0, 1, 16, 1), (3, 16, 16, 1), (6, 16, 32, 2), (9, 32, 32, 1), (12, 32, 64, 2), (15, 64, 64, 1)]
HARDNET_CONVS = [(0, 1, 32, 1), (3, 32, 32, 1), (6, 32, 64, 2), (9, 64, 64, 1), (12, 64, 128, 2), (15, 128, 128, 1)]
AFFNET_HEAD, HARDNET_HEAD = 19, 19          # the 8x8 convolutions (index 18 is Dropout)
BN_EPS = 1e-5


# ---- kornia/feature/responses.py ----
def gftt_response(x: torch.Tensor, sigmas: torch.Tensor = None) -> torch.Tensor:
    """kornia.feature.responses.gftt_response(grads_mode='sobel'): the smaller eigenvalue of the blurred structure tensor."""
    g = KO.spatial_gradient(x, 'sobel')
    dx, dy = g[:, :, 0], g[:, :, 1]
    dx2 = KO.gaussian_blur2d(dx ** 2, 7, 1.0)
    dy2 = KO.gaussian_blur2d(dy ** 2, 7, 1.0)
    dxy = KO.gaussian_blur2d(dx * dy, 7, 1.0)
    det_m = dx2 * dy2 - dxy * dxy
    trace_m = dx2 + dy2
    e1 = 0.5 * (trace_m + torch.sqrt((trace_m ** 2 - 4 * det_m).abs()))
    e2 = 0.5 * (trace_m - torch.sqrt((trace_m ** 2 - 4 * det_m).abs()))
    scores = torch.min(e1, e2)
    if sigmas is not None:
        scores = scores * sigmas.pow(4).view(-1, 1, 1, 1)
    return scores


# ---- kornia/feature/scale_space_detector.py (scale_space_response=False, maxima only) ----
def octave_response(octave: torch.Tensor, sigmas: torch.Tensor) -> torch.Tensor:
    """The GFTT response of every level of one octave [B, 1, L, h, w] as one [B L, 1, h, w] batch, the last level dropped:
    [B, 1, L - 1, h, w]."""
    B, CH, L, h, w = octave.shape
    r = gftt_response(octave.permute(0, 2, 1, 3, 4).reshape(B * L, CH, h, w), sigmas.view(-1)).view(B, L, CH, h, w)
    return r.permute(0, 2, 1, 3, 4)[:, :, :-1]


def octave_candidates(resp_vol: torch.Tensor, sigma0: float, num_feats: int, mr_size: float = 6.0):
    """One octave of detect from its response volume: conv_quad_interp3d (maxima only), the per-octave top-k (ties: lower voxel
    first), the LAFs and the border test.  -> (responses [B, n], octave-pixel LAFs [B, n, 2, 3], voxel indices [B, n])"""
    B, CH, L, h, w = resp_vol.shape
    coord_max, resp_max = KO.conv_quad_interp3d(resp_vol, 10.0)
    flat = resp_max.view(B, -1)
    coords = coord_max.view(B, 3, -1).permute(0, 2, 1)
    if flat.size(1) > num_feats:
        idx = KO._topk_low_index(flat, num_feats)
        best = torch.gather(flat, 1, idx)
        cbest = torch.gather(coords, 1, idx.unsqueeze(-1).repeat(1, 1, 3))
    else:
        idx = torch.arange(flat.size(1), device=resp_vol.device).expand(B, -1)
        best, cbest = flat, coords
    n = best.size(1)
    sig = sigma0 * torch.pow(2.0, cbest[:, :, 0].contiguous().view(-1, 1, 1, 1) / 3.0).view(B, n, 1)   # _scale_index_to_scale
    cbest = torch.cat([sig, cbest[:, :, 1:]], dim=2)
    rot = torch.eye(2, dtype=resp_vol.dtype, device=resp_vol.device).view(1, 1, 2, 2)
    lafs = torch.cat([mr_size * cbest[:, :, 0].view(B, n, 1, 1) * rot, cbest[:, :, 1:3].view(B, n, 2, 1)], dim=3)
    good = KO.laf_is_inside_image(lafs, h, w)
    return best * good.to(best.dtype), lafs, idx


def detect(img: torch.Tensor, num_feats: int, want_stages: bool = False):
    """ScaleSpaceDetector(num_feats, CornerGFTT, ConvQuadInterp3d(10), ScalePyramid(3, 1.6, 32, False), mr_size=6).detect:
    (responses [B, num_feats], lafs [B, num_feats, 2, 3] in image pixels, before the affine shape and orientation)."""
    B, _, H, W = img.shape
    pyr, sigmas = KO.scale_pyramid(img, double_image=False)
    resp, lafs, stages = [], [], []
    for o, octave in enumerate(pyr):
        h, w = octave.shape[-2:]
        vol = octave_response(octave, sigmas[o])
        r, l, idx = octave_candidates(vol, float(sigmas[o][0, 0]), num_feats)
        stages.append(dict(response=vol, resp=r, lafs=l, index=idx))
        resp.append(r)
        lafs.append(KO.normalize_laf(l, h, w))
    resp = torch.cat(resp, dim=1)
    lafs = torch.cat(lafs, dim=1)
    idx = KO._topk_low_index(resp, num_feats)
    resp = torch.gather(resp, 1, idx)
    lafs = KO.denormalize_laf(torch.gather(lafs, 1, idx.unsqueeze(-1).unsqueeze(-1).repeat(1, 1, 2, 3)), H, W)
    if want_stages:
        return resp, lafs, dict(pyramid=pyr, sigmas=sigmas, octaves=stages, index=idx)
    return resp, lafs


# ---- the two patch CNNs (kornia/feature/affine_shape.py, hardnet.py) ----
def _conv_stack(convs):
    layers = []
    for _, ci, co, s in convs:
        layers += [nn.Conv2d(ci, co, kernel_size=3, stride=s, padding=1, bias=False), nn.BatchNorm2d(co, affine=False), nn.ReLU()]
    return layers


def affnet_features() -> nn.Sequential:
    """LAFAffNetShapeEstimator.features"""
    return nn.Sequential(*_conv_stack(AFFNET_CONVS), nn.Dropout(0.25), nn.Conv2d(64, 3, kernel_size=8, stride=1, padding=0, bias=True),
                         nn.Tanh(), nn.AdaptiveAvgPool2d(1))


def hardnet_features() -> nn.Sequential:
    """HardNet.features"""
    return nn.Sequential(*_conv_stack(HARDNET_CONVS), nn.Dropout(0.3), nn.Conv2d(128, 128, kernel_size=8, bias=False),
                         nn.BatchNorm2d(128, affine=False))


def normalize_input(x: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """_normalize_input of AffNet and HardNet: per-patch standardisation, Bessel-corrected std"""
    sp, mp = torch.std_mean(x, dim=(-3, -2, -1), keepdim=True)
    return (x - mp.detach()) / (sp.detach() + eps)


def _synthetic(convs, seed: int) -> dict:
    """He-scaled convolutions; BatchNorm running statistics near those of unit-variance activations (mean 0.1 N(0, 1), var in
    [0.8, 1.25]), so every layer's output stays near unit variance on standardised patches"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, ci, co, _ in convs:
        gain = 1.0 if i == 0 else 2.0                  # post-ReLU inputs carry half their variance
        sd[f'features.{i}.weight'] = torch.randn(co, ci, 3, 3, generator=g) * math.sqrt(gain / (9 * ci))
        sd[f'features.{i + 1}.running_mean'] = 0.1 * torch.randn(co, generator=g)
        sd[f'features.{i + 1}.running_var'] = 0.8 + 0.45 * torch.rand(co, generator=g)
        sd[f'features.{i + 1}.num_batches_tracked'] = torch.tensor(0)
    return sd, g


def synthetic_affnet_state_dict(seed: int = AFFNET_SEED) -> dict:
    """AffNet weights in kornia's key layout.  The last layer is scaled so its pre-activation has std 0.1 on natural images:
    |tanh| stays below 0.5 and the frames stay well conditioned."""
    sd, g = _synthetic(AFFNET_CONVS, seed)
    sd[f'features.{AFFNET_HEAD}.weight'] = torch.randn(3, 64, 8, 8, generator=g) * (0.1 / math.sqrt(0.5 * 64 * 64))
    sd[f'features.{AFFNET_HEAD}.bias'] = 0.02 * torch.randn(3, generator=g)
    return sd


def synthetic_hardnet_state_dict(seed: int = HARDNET_SEED) -> dict:
    """HardNet weights in kornia's key layout"""
    sd, g = _synthetic(HARDNET_CONVS, seed)
    sd[f'features.{HARDNET_HEAD}.weight'] = torch.randn(128, 128, 8, 8, generator=g) * math.sqrt(2.0 / (128 * 64))
    sd[f'features.{HARDNET_HEAD + 1}.running_mean'] = 0.1 * torch.randn(128, generator=g)
    sd[f'features.{HARDNET_HEAD + 1}.running_var'] = 0.8 + 0.45 * torch.rand(128, generator=g)
    sd[f'features.{HARDNET_HEAD + 1}.num_batches_tracked'] = torch.tensor(0)
    return sd


def state_dict_checksum(sd: dict) -> str:
    """sha256 over the float32 bytes of every floating tensor, in key order"""
    h = hashlib.sha256()
    for k in sorted(sd):
        if sd[k].is_floating_point():
            h.update(k.encode())
            h.update(sd[k].detach().float().contiguous().numpy().tobytes())
    return h.hexdigest()


def scale_laf(laf: torch.Tensor, scale_coef: torch.Tensor) -> torch.Tensor:
    return torch.cat([laf[:, :, :2, :2] * scale_coef, laf[:, :, :, 2:]], dim=3)


def affnet_frames(xy: torch.Tensor, laf: torch.Tensor, preserve_orientation: bool = True) -> torch.Tensor:
    """LAFAffNetShapeEstimator.forward after the network: xy [B N, 3] (tanh, pooled) and the input LAFs [B, N, 2, 3] -> LAFs"""
    B, N = laf.shape[:2]
    a1 = torch.cat([1.0 + xy[:, 0].reshape(-1, 1, 1), 0 * xy[:, 0].reshape(-1, 1, 1)], dim=2)
    a2 = torch.cat([xy[:, 1].reshape(-1, 1, 1), 1.0 + xy[:, 2].reshape(-1, 1, 1)], dim=2)
    new_laf_no_center = torch.cat([a1, a2], dim=1).reshape(B, N, 2, 2)
    new_laf = torch.cat([new_laf_no_center, laf[:, :, :, 2:3]], dim=3)
    scale_orig = KO.get_laf_scale(laf)
    if preserve_orientation:
        ori_orig = KO.get_laf_orientation(laf)
    ellipse_scale = KO.get_laf_scale(new_laf)
    laf_out = scale_laf(KO.make_upright(new_laf), scale_orig / ellipse_scale)
    if preserve_orientation:
        laf_out = KO.set_laf_orientation(laf_out, ori_orig)
    return laf_out


def affnet_patches(img: torch.Tensor, laf: torch.Tensor) -> torch.Tensor:
    """AffNet's standardised input: [B N, 1, 32, 32] from extract_patches_from_pyramid(img, make_upright(laf), 32)"""
    return normalize_input(KO.extract_patches_from_pyramid(img, KO.make_upright(laf), PS).view(-1, 1, PS, PS))


def affnet_shape(laf: torch.Tensor, img: torch.Tensor, features: nn.Module, preserve_orientation: bool = True, want_xy: bool = False):
    """LAFAffNetShapeEstimator.forward"""
    xy = features(affnet_patches(img, laf)).view(-1, 3)
    out = affnet_frames(xy, laf, preserve_orientation)
    return (out, xy) if want_xy else out


def hardnet(patches: torch.Tensor, features: nn.Module) -> torch.Tensor:
    """HardNet.forward: patches [n, 1, 32, 32] -> unit rows [n, 128]"""
    x = features(normalize_input(patches))
    return F.normalize(x.view(x.size(0), -1), dim=1)


def laf_descriptors(img: torch.Tensor, laf: torch.Tensor, features: nn.Module) -> torch.Tensor:
    """kornia.feature.integrated.get_laf_descriptors with HardNet (grayscale input)"""
    B, N = laf.shape[:2]
    if N == 0:
        return torch.empty(B, 0, 128, dtype=img.dtype, device=img.device)
    p = KO.extract_patches_from_pyramid(img, laf, PS)
    return hardnet(p.view(B * N, 1, PS, PS), features).view(B, N, -1)


def features_in(dtype: torch.dtype, affnet_sd: dict = None, hardnet_sd: dict = None):
    """(AffNet features, HardNet features) in eval mode and ``dtype``, by default with the synthetic weights"""
    a, h = affnet_features(), hardnet_features()
    a.load_state_dict({k[len('features.'):]: v for k, v in (affnet_sd or synthetic_affnet_state_dict()).items()})
    h.load_state_dict({k[len('features.'):]: v for k, v in (hardnet_sd or synthetic_hardnet_state_dict()).items()})
    return a.eval().to(dtype), h.eval().to(dtype)


def run(img: torch.Tensor, num_feats: int = 1024, nms_diameter: int = 9, upright: bool = False, min_stack: bool = True,
        affnet_sd: dict = None, hardnet_sd: dict = None):
    """The whole front-end in img's dtype, without the reference's wiring: detect, AffNet, orienter, run_nms (oracle nms2d),
    HardNet.  -> (lafs, responses, descriptors) of each image (min_stack=False) or the min-stacked batch."""
    aff, hard = (net.to(img.device) for net in features_in(img.dtype, affnet_sd, hardnet_sd))
    with torch.no_grad():
        resp, lafs = detect(img, num_feats)
        lafs = affnet_shape(lafs, img, aff)
        if not upright:
            lafs = KO.laf_orienter(lafs, img, 19)
        out = []
        B, _, H, W = img.shape
        for b in range(B):
            keep = run_nms_one(lafs[b], resp[b], H, W, nms_diameter)
            out.append((lafs[b][keep], resp[b][keep]))
        n = min(min(o[1].numel() for o in out), num_feats) if min_stack else None
        res = []
        for b, (l, r) in enumerate(out):
            k = n if min_stack else min(r.numel(), num_feats)
            idx = KO._topk_low_index(r[None], k)[0]
            l, r = l[idx], r[idx]
            d = laf_descriptors(img[b:b + 1], l[None], hard)[0]
            res.append((l, r, d))
    if min_stack:
        return tuple(torch.stack(t) for t in zip(*res))
    return res


def run_nms_one(lafs: torch.Tensor, scores: torch.Tensor, H: int, W: int, nms_diameter: int = 9) -> torch.Tensor:
    """base.py's run_nms for one image: indices of the kept rows in detector order"""
    kpts = torch.round(lafs[:, :, -1]).long()
    smin, smax = scores.amin(), scores.amax()
    ns = (scores - smin + 1e-2) / (smax - smin + 1e-1)
    kv = H * kpts[:, 0] + kpts[:, 1]
    order = torch.sort(kv.to(scores.dtype) + (1 - ns), stable=True).indices
    kv_sorted = kv[order]
    first = torch.ones_like(kv_sorted, dtype=torch.bool)
    first[1:] = kv_sorted[1:] != kv_sorted[:-1]
    uniq = order[first]
    mask = torch.zeros(1, 1, H, W, dtype=scores.dtype, device=scores.device)
    k = kpts[uniq]
    mask[0, 0, k[:, 1], k[:, 0]] = scores[uniq]
    m = KO.nms2d(mask.cpu(), (nms_diameter, nms_diameter), mask_only=True).to(mask.device)[0, 0, k[:, 1], k[:, 0]]   # CPU-only restatement
    kept = uniq[m]
    return torch.sort(kept).values


# ---- nn.Module stand-ins with kornia's constructor signatures (the fixture script stubs kornia with these) ----
class ScalePyramid(nn.Module):
    def __init__(self, n_levels: int = 3, init_sigma: float = 1.6, min_size: int = 15, double_image: bool = False):
        super().__init__()
        assert (n_levels, init_sigma, min_size, double_image) == (3, 1.6, 32, False), 'only the reference GFTT pyramid is restated'


class CornerGFTT(nn.Module):
    def __init__(self, grads_mode: str = 'sobel'):
        super().__init__()
        assert grads_mode == 'sobel'

    def forward(self, x, sigmas=None):
        return gftt_response(x, sigmas)


class ConvQuadInterp3d(nn.Module):
    def __init__(self, strict_maxima_bonus: float = 10.0, eps: float = 1e-7):
        super().__init__()
        assert strict_maxima_bonus == 10.0


class PassLAF(nn.Module):
    def forward(self, laf, img):
        return laf


class _PatchDominantGradientOrientation(nn.Module):
    def __init__(self, patch_size: int = 32):
        super().__init__()
        self.patch_size = patch_size
        self.angular_smooth = nn.Conv1d(1, 1, kernel_size=3, padding=1, bias=False, padding_mode='circular')
        with torch.no_grad():
            self.angular_smooth.weight[:] = torch.tensor([[[0.33, 0.34, 0.33]]])


class LAFOrienter(nn.Module):
    def __init__(self, patch_size: int = 32, num_angular_bins: int = 36, angle_detector=None):
        super().__init__()
        self.patch_size = patch_size
        self.angle_detector = _PatchDominantGradientOrientation(patch_size)

    def forward(self, laf, img):
        return KO.laf_orienter(laf, img, self.patch_size)


class LAFAffNetShapeEstimator(nn.Module):
    def __init__(self, pretrained: bool = False, preserve_orientation: bool = True):
        super().__init__()
        self.features = affnet_features()
        self.patch_size = PS
        if pretrained:                              # the synthetic weights stand in for the checkpoint; no download
            self.load_state_dict(synthetic_affnet_state_dict(), strict=False)
        self.preserve_orientation = preserve_orientation
        self.eval()

    def forward(self, laf, img):
        return affnet_shape(laf, img, self.features, self.preserve_orientation)


class HardNet(nn.Module):
    patch_size = PS

    def __init__(self, pretrained: bool = False):
        super().__init__()
        self.features = hardnet_features()
        if pretrained:
            self.load_state_dict(synthetic_hardnet_state_dict(), strict=True)
        self.eval()

    def forward(self, x):
        return hardnet(x, self.features)


class ScaleSpaceDetector(nn.Module):
    def __init__(self, num_features: int = 500, mr_size: float = 6.0, scale_pyr_module=None, resp_module=None, nms_module=None,
                 ori_module=None, aff_module=None, minima_are_also_good: bool = False, scale_space_response: bool = False):
        super().__init__()
        assert mr_size == 6.0 and not minima_are_also_good and not scale_space_response
        assert isinstance(resp_module, CornerGFTT) and isinstance(nms_module, ConvQuadInterp3d) and isinstance(scale_pyr_module, ScalePyramid)
        self.num_features = num_features
        self.resp, self.nms, self.scale_pyr = resp_module, nms_module, scale_pyr_module
        self.ori, self.aff = ori_module, aff_module
        self.calls = []                       # the stages of every call, for the fixture script

    def forward(self, img, mask=None):
        resp, lafs, stages = detect(img, self.num_features, want_stages=True)
        aff = self.aff(lafs, img)
        out = self.ori(aff, img)
        self.calls.append(dict(stages, det_resp=resp, det_lafs=lafs, aff_lafs=aff))
        return out, resp


class LAFDescriptor(nn.Module):
    def __init__(self, patch_descriptor_module=None, patch_size: int = 32, grayscale_descriptor: bool = True):
        super().__init__()
        self.descriptor = HardNet(True) if patch_descriptor_module is None else patch_descriptor_module
        self.patch_size = patch_size
        assert patch_size == PS

    def forward(self, img, lafs):
        return laf_descriptors(img, lafs, self.descriptor.features)
