"""Pure-torch restatement of the kornia pieces behind the reference's default online features, ``SIFT``
(models/features/sift.py:16-49 on models/features/base.py:8-82): ``ScaleSpaceDetector`` with ``BlobDoG``, ``ConvQuadInterp3d(10)``,
``ScalePyramid(3, 1.6, 32, double_image=True)`` and ``LAFOrienter(19)`` / ``PassLAF``, then ``LAFDescriptor(SIFTDescriptor(41))``.

TEST INFRASTRUCTURE (the checker, never the product path).  kornia is not a dependency of this project; every function below
restates kornia 0.6.3 (the release the reference's ``kornia>=0.6.1`` pin resolved to when it was published), names the kornia
module it restates, and calls the ATen operations in kornia's order.  Every function runs in the dtype of its input: the GPU tests
compare the kernels against the float32 form and take their bounds from the float32 - float64 difference.  kornia's constants that
it builds in float32 (Gaussian taps, ``kornia.constants.pi``) are float32 values in both forms, as kornia's ``.to(dtype)`` makes them.

Where a detail of kornia 0.6.3 differs from what a reader might expect, the restatement keeps kornia's:
  - ``ScalePyramid.get_first_level`` doubles the image with ``F.interpolate(scale_factor=2, bilinear, align_corners=False)``
    (later releases use ``upscale_double``);
  - ``spatial_gradient3d(order=2)`` convolves with the depth-flipped kernel (``kernel.flip(-3)``), so the two scale cross
    derivatives enter the Hessian with kornia's sign;
  - ``conv_quad_interp3d`` adds ``dx.flip(1)`` (scale, y, x) to ``create_meshgrid3d``'s (scale, x, y) grid;
  - ``generate_patch_grid_from_normalized_LAF`` normalises the sampling grid by ``w`` and ``h``, not ``w - 1`` and ``h - 1``;
  - ``torch.topk`` / ``max`` leave the order of ties unspecified: here, and in the kernels, the lower index goes first.
The only pin of these functions to an execution of kornia is tests/test_kornia_sift_oracle.py, which runs where kornia is
installed.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

KORNIA_RELEASE = '0.6.3'
PI = torch.tensor(3.14159265358979323846)           # kornia.constants.pi (float32)


def _nms2d_restated():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location('_og_nms2d_src', os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                                 'gen_golden_superpoint.py'))
    # gen_golden_superpoint holds the one restatement of kornia's nms2d; it is imported by path (it edits sys.path on import)
    import sys
    saved = list(sys.path)
    mod = importlib.util.module_from_spec(spec)
    try:
        spec.loader.exec_module(mod)
    finally:
        sys.path[:] = saved
    return mod.nms2d


nms2d = _nms2d_restated()


# ---- kornia/filters (kernels.py, filter.py, gaussian.py, sobel.py) ----
def gaussian_kernel1d(ksize: int, sigma: float) -> torch.Tensor:
    """kornia.filters.kernels.gaussian (float32, as kornia builds it)."""
    x = torch.arange(ksize).float() - ksize // 2
    if ksize % 2 == 0:
        x = x + 0.5
    gauss = torch.exp((-x.pow(2.0) / float(2 * sigma ** 2)))
    return gauss / gauss.sum()


def gaussian_kernel2d(ksize: int, sigma: float) -> torch.Tensor:
    """kornia.filters.kernels.get_gaussian_kernel2d: the outer product of the 1-D kernels, [1, k, k] float32."""
    kx = gaussian_kernel1d(ksize, sigma)
    return torch.matmul(kx.unsqueeze(-1), kx.unsqueeze(-1).t())[None]


def filter2d(x: torch.Tensor, kernel: torch.Tensor, border_type: str = 'reflect') -> torch.Tensor:
    """kornia.filters.filter.filter2d: pad by (k - 1) / 2 with ``border_type``, then a grouped conv2d."""
    b, c, h, w = x.shape
    k = kernel.unsqueeze(1).to(x).expand(-1, c, -1, -1)
    kh, kw = k.shape[-2:]
    pad = [(kw - 1) // 2, kw // 2, (kh - 1) // 2, kh // 2]        # _compute_padding, for odd and even kernels
    xp = F.pad(x, pad, mode=border_type)
    k = k.reshape(-1, 1, kh, kw)
    xp = xp.view(-1, k.size(0), xp.size(-2), xp.size(-1))
    return F.conv2d(xp, k, groups=k.size(0), padding=0, stride=1).view(b, c, h, w)


def gaussian_blur2d(x: torch.Tensor, ksize: int, sigma: float) -> torch.Tensor:
    """kornia.filters.gaussian.gaussian_blur2d (GaussianBlur2d: the 2-D kernel through filter2d, reflect border)."""
    return filter2d(x, gaussian_kernel2d(ksize, sigma), 'reflect')


def spatial_gradient(x: torch.Tensor, mode: str = 'sobel') -> torch.Tensor:
    """kornia.filters.sobel.spatial_gradient(order=1, normalized=True): [B, C, 2, H, W], replicate border."""
    if mode == 'sobel':
        kx = torch.tensor([[-1.0, 0.0, 1.0], [-2.0, 0.0, 2.0], [-1.0, 0.0, 1.0]])
    else:
        kx = torch.tensor([[0.0, 0.0, 0.0], [-1.0, 0.0, 1.0], [0.0, 0.0, 0.0]])
    kernel = torch.stack([kx, kx.transpose(0, 1)])
    kernel = kernel / kernel.abs().sum(dim=-1).sum(dim=-1).unsqueeze(-1).unsqueeze(-1)      # normalize_kernel2d
    b, c, h, w = x.shape
    k = kernel.to(x).unsqueeze(1).unsqueeze(1).flip(-3)
    xp = F.pad(x.reshape(b * c, 1, h, w), [1, 1, 1, 1], 'replicate')[:, :, None]
    return F.conv3d(xp, k, padding=0).view(b, c, 2, h, w)


# ---- kornia/geometry/transform/pyramid.py ----
def sift_kernel_size(sigma: float) -> int:
    """ScalePyramid.get_kernel_size: int(8 sigma + 1), made odd."""
    k = int(2.0 * 4.0 * sigma + 1.0)
    return k + 1 if k % 2 == 0 else k


def scale_pyramid(x: torch.Tensor, n_levels: int = 3, init_sigma: float = 1.6, min_size: int = 32,
                  double_image: bool = True) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """kornia.geometry.transform.pyramid.ScalePyramid.forward: octaves [B, C, n_levels + 3, h, w] and their sigmas [B, n_levels + 3]."""
    extra = 3
    sigma_step = 2 ** (1.0 / float(n_levels))
    bs = x.shape[0]
    cur_sigma = 0.5
    if double_image:
        x = F.interpolate(x, scale_factor=2.0, mode='bilinear', align_corners=False)
        cur_sigma *= 2.0
    if init_sigma > cur_sigma:
        sigma = max(math.sqrt(init_sigma ** 2 - cur_sigma ** 2), 0.01)
        k = sift_kernel_size(sigma)
        cur_level = gaussian_blur2d(x, k, sigma)
        cur_sigma = init_sigma
    else:
        cur_level = x
    sigmas = [cur_sigma * torch.ones(bs, n_levels + extra).to(x)]
    pyr = [[cur_level]]
    while True:
        cur_level = pyr[-1][0]
        for level_idx in range(1, n_levels + extra):
            sigma = cur_sigma * math.sqrt(sigma_step ** 2 - 1.0)
            k = sift_kernel_size(sigma)
            k = min(k, min(cur_level.size(2), cur_level.size(3)))
            if k % 2 == 0:
                k += 1
            cur_level = gaussian_blur2d(cur_level, k, sigma)
            cur_sigma *= sigma_step
            pyr[-1].append(cur_level)
            sigmas[-1][:, level_idx] = cur_sigma
        nxt = pyr[-1][-extra][:, :, ::2, ::2]
        cur_sigma = init_sigma
        if min(nxt.size(2), nxt.size(3)) <= min_size:
            break
        pyr.append([nxt])
        sigmas.append(cur_sigma * torch.ones(bs, n_levels + extra).to(x))
    return [torch.stack(p, dim=2) for p in pyr], sigmas


def pyrdown(x: torch.Tensor) -> torch.Tensor:
    """kornia.geometry.transform.pyramid.pyrdown: the 5x5 binomial blur (reflect), then bilinear to (h // 2, w // 2)."""
    k = torch.tensor([[1.0, 4.0, 6.0, 4.0, 1.0], [4.0, 16.0, 24.0, 16.0, 4.0], [6.0, 24.0, 36.0, 24.0, 6.0],
                      [4.0, 16.0, 24.0, 16.0, 4.0], [1.0, 4.0, 6.0, 4.0, 1.0]])[None] / 256.0
    b, c, h, w = x.shape
    xb = filter2d(x, k, 'reflect')
    return F.interpolate(xb, size=(int(float(h) / 2.0), int(float(w) // 2.0)), mode='bilinear', align_corners=False)


# ---- kornia/feature/responses.py, kornia/geometry/subpix ----
def dog_response(x: torch.Tensor) -> torch.Tensor:
    """kornia.feature.responses.BlobDoG / dog_response: consecutive levels subtracted."""
    return x[:, :, 1:] - x[:, :, :-1]


def nms3d(x: torch.Tensor) -> torch.Tensor:
    """kornia.geometry.subpix.nms.nms3d(x, (3, 3, 3), mask_only=True): strictly greater than all 26 neighbours, replicate border."""
    B, C, D, H, W = x.shape
    xp = F.pad(x.reshape(B * C, 1, D, H, W), [1] * 6, mode='replicate')[:, 0]
    m = None
    for dd in range(3):
        for dy in range(3):
            for dx in range(3):
                if dd == dy == dx == 1:
                    continue
                v = xp[:, dd:dd + D, dy:dy + H, dx:dx + W]
                m = v if m is None else torch.maximum(m, v)
    return (x.reshape(B * C, D, H, W) > m).view(B, C, D, H, W)


_D2 = [  # kornia.filters.kernels.get_diff_kernel3d_2nd_order: dxx, dyy, dss, dxy, dys, dxs; [d][h][w]
    [[[0, 0, 0], [0, 0, 0], [0, 0, 0]], [[0, 0, 0], [1, -2, 1], [0, 0, 0]], [[0, 0, 0], [0, 0, 0], [0, 0, 0]]],
    [[[0, 0, 0], [0, 0, 0], [0, 0, 0]], [[0, 1, 0], [0, -2, 0], [0, 1, 0]], [[0, 0, 0], [0, 0, 0], [0, 0, 0]]],
    [[[0, 0, 0], [0, 1, 0], [0, 0, 0]], [[0, 0, 0], [0, -2, 0], [0, 0, 0]], [[0, 0, 0], [0, 1, 0], [0, 0, 0]]],
    [[[0, 0, 0], [0, 0, 0], [0, 0, 0]], [[1, 0, -1], [0, 0, 0], [-1, 0, 1]], [[0, 0, 0], [0, 0, 0], [0, 0, 0]]],
    [[[0, 1, 0], [0, 0, 0], [0, -1, 0]], [[0, 0, 0], [0, 0, 0], [0, 0, 0]], [[0, -1, 0], [0, 0, 0], [0, 1, 0]]],
    [[[0, 0, 0], [1, 0, -1], [0, 0, 0]], [[0, 0, 0], [0, 0, 0], [0, 0, 0]], [[0, 0, 0], [-1, 0, 1], [0, 0, 0]]],
]


def spatial_gradient3d(x: torch.Tensor, order: int) -> torch.Tensor:
    """kornia.filters.sobel.spatial_gradient3d(mode='diff'): order 1 by the central-difference special case, [B, C, 3, D, H, W]
    (x, y, s); order 2 by conv3d with the depth-flipped second-order kernel, [B, C, 6, D, H, W]."""
    b, c, d, h, w = x.shape
    if order == 1:
        xp = F.pad(x, 6 * [1], 'replicate')
        ce, le, ri = slice(1, -1), slice(0, -2), slice(2, None)
        out = torch.empty(b, c, 3, d, h, w, dtype=x.dtype, device=x.device)
        out[..., 0, :, :, :] = xp[..., ce, ce, ri] - xp[..., ce, ce, le]
        out[..., 1, :, :, :] = xp[..., ce, ri, ce] - xp[..., ce, le, ce]
        out[..., 2, :, :, :] = xp[..., ri, ce, ce] - xp[..., le, ce, ce]
        return 0.5 * out
    kernel = torch.tensor(_D2, dtype=torch.float32).unsqueeze(1).to(x)
    k = kernel.repeat(c, 1, 1, 1, 1).flip(-3)
    return F.conv3d(F.pad(x, 6 * [1], 'replicate'), k, padding=0, groups=c).view(b, c, 6, d, h, w)


def safe_solve_with_mask(B: torch.Tensor, A: torch.Tensor):
    """kornia.utils.helpers.safe_solve_with_mask: LU with partial pivoting (``torch.lu(get_infos=True)``), a solution where
    the factorisation met no exact zero pivot."""
    LU, piv, info = torch.linalg.lu_factor_ex(A)
    return torch.linalg.lu_solve(LU, piv, B), info == 0


def conv_quad_interp3d(x: torch.Tensor, strict_maxima_bonus: float = 10.0):
    """kornia.geometry.subpix.spatial_soft_argmax.conv_quad_interp3d: (coords [B, C, 3, D, H, W] as (s, x, y), y_max)."""
    B, CH, D, H, W = x.shape
    zs = torch.linspace(0, D - 1, D, dtype=x.dtype, device=x.device)
    xs = torch.linspace(0, W - 1, W, dtype=x.dtype, device=x.device)
    ys = torch.linspace(0, H - 1, H, dtype=x.dtype, device=x.device)
    grid = torch.stack(torch.meshgrid([zs, xs, ys], indexing='ij'), dim=-1).permute(0, 2, 1, 3).unsqueeze(0)   # create_meshgrid3d
    grid = grid.permute(0, 4, 1, 2, 3)
    b = spatial_gradient3d(x, 1).permute(0, 1, 3, 4, 5, 2).reshape(-1, 3, 1)
    A = spatial_gradient3d(x, 2).permute(0, 1, 3, 4, 5, 2).reshape(-1, 6)
    dxx, dyy, dss = A[..., 0], A[..., 1], A[..., 2]
    dxy, dys, dxs = 0.25 * A[..., 3], 0.25 * A[..., 4], 0.25 * A[..., 5]
    Hes = torch.stack([dxx, dxy, dxs, dxy, dyy, dys, dxs, dys, dss], dim=-1).view(-1, 3, 3)
    nms_mask = nms3d(x)
    x_solved = torch.zeros_like(b)
    sol, ok = safe_solve_with_mask(b[nms_mask.view(-1)], Hes[nms_mask.view(-1)])
    new_mask = nms_mask.masked_scatter(nms_mask, ok)
    x_solved.masked_scatter_(new_mask.view(-1, 1, 1), sol[ok])
    dx = -x_solved
    far = dx.abs().max(dim=1, keepdim=True)[0] > 0.7
    dx.masked_fill_(far.expand_as(dx), 0)
    dy = 0.5 * torch.bmm(b.permute(0, 2, 1), dx)
    y_max = x + dy.view(B, CH, D, H, W)
    y_max += strict_maxima_bonus * new_mask.to(x.dtype)
    dx_res = dx.flip(1).reshape(B, CH, D, H, W, 3).permute(0, 1, 5, 2, 3, 4)
    coords = grid.repeat(B, 1, 1, 1, 1).unsqueeze(1) + dx_res
    return coords, y_max


# ---- kornia/feature/laf.py ----
def get_laf_scale(laf: torch.Tensor) -> torch.Tensor:
    out = laf[..., 0:1, 0:1] * laf[..., 1:2, 1:2] - laf[..., 1:2, 0:1] * laf[..., 0:1, 1:2] + 1e-10
    return out.abs().sqrt()


def _laf_coef(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    wf, hf = float(w - 1), float(h - 1)
    coef = torch.ones(1, 1, 2, 3).to(laf) * min(hf, wf)
    coef[0, 0, 0, 2] = wf
    coef[0, 0, 1, 2] = hf
    return coef


def normalize_laf(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """kornia.feature.laf.normalize_laf (the image given by its size)."""
    return laf / _laf_coef(laf, h, w)


def denormalize_laf(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """kornia.feature.laf.denormalize_laf (the image given by its size)."""
    return _laf_coef(laf, h, w).expand_as(laf) * laf


def laf_is_inside_image(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """kornia.feature.laf.laf_is_inside_image(border=0) through laf_to_boundary_points(laf, 12) and
    convert_points_from_homogeneous (eps 1e-8)."""
    B, N = laf.shape[:2]
    n_pts = 12
    t = torch.linspace(0, 2 * math.pi, n_pts - 1)
    pts = torch.cat([torch.sin(t).unsqueeze(-1), torch.cos(t).unsqueeze(-1), torch.ones(n_pts - 1, 1)], dim=1)
    pts = torch.cat([torch.tensor([0.0, 0.0, 1.0]).view(1, 3), pts], dim=0).unsqueeze(0).expand(B * N, n_pts, 3).to(laf)
    aux = torch.tensor([0.0, 0.0, 1.0]).view(1, 1, 3).expand(B * N, 1, 3).to(laf)
    hlaf = torch.cat([laf.reshape(-1, 2, 3), aux], dim=1)
    ph = torch.bmm(hlaf, pts.permute(0, 2, 1)).permute(0, 2, 1).reshape(B, N, n_pts, 3)
    z = ph[..., 2:]
    scale = torch.where(torch.abs(z) > 1e-8, 1.0 / (z + 1e-8), torch.ones_like(z))
    p = scale * ph[..., :2]
    good = (p[..., 0] >= 0) * (p[..., 0] <= w) * (p[..., 1] >= 0) * (p[..., 1] <= h)
    return good.min(dim=2)[0]


def rad2deg(t: torch.Tensor) -> torch.Tensor:
    return 180.0 * t / PI.to(t)


def deg2rad(t: torch.Tensor) -> torch.Tensor:
    return t * PI.to(t) / 180.0


def get_laf_orientation(laf: torch.Tensor) -> torch.Tensor:
    return rad2deg(torch.atan2(laf[..., 0, 1], laf[..., 0, 0])).unsqueeze(-1)


def make_upright(laf: torch.Tensor, eps: float = 1e-9) -> torch.Tensor:
    det = get_laf_scale(laf)
    b2a2 = torch.sqrt(laf[..., 0:1, 1:2] ** 2 + laf[..., 0:1, 0:1] ** 2) + eps
    l1 = torch.cat([(b2a2 / det).contiguous(), torch.zeros_like(det)], dim=3)
    l2 = torch.cat([((laf[..., 1:2, 1:2] * laf[..., 0:1, 1:2] + laf[..., 1:2, 0:1] * laf[..., 0:1, 0:1]) / (b2a2 * det)),
                    (det / b2a2).contiguous()], dim=3)
    unit = torch.cat([torch.cat([l1, l2], dim=2), laf[..., :, 2:3]], dim=3)
    return torch.cat([det * unit[:, :, :2, :2], unit[:, :, :, 2:]], dim=3)          # scale_laf


def rotate_laf(laf: torch.Tensor, angles_degrees: torch.Tensor) -> torch.Tensor:
    B, N = laf.shape[:2]
    a = deg2rad(angles_degrees)
    c, s = torch.cos(a), torch.sin(a)
    rot = torch.stack([c, s, -s, c], dim=-1).view(B * N, 2, 2)                       # angle_to_rotation_matrix
    out = laf.clone()
    out[:, :, :2, :2] = torch.bmm(laf[:, :, :2, :2].reshape(B * N, 2, 2), rot).reshape(B, N, 2, 2)
    return out


def set_laf_orientation(laf: torch.Tensor, angles_degrees: torch.Tensor) -> torch.Tensor:
    ori = get_laf_orientation(laf).reshape_as(angles_degrees)
    return rotate_laf(make_upright(laf), angles_degrees - ori)


def extract_patches_from_pyramid(img: torch.Tensor, laf: torch.Tensor, PS: int) -> torch.Tensor:
    """kornia.feature.laf.extract_patches_from_pyramid: per LAF the pyrdown level of log2(2 scale / PS), sampled with
    grid_sample (bilinear, border, align_corners=False) on generate_patch_grid_from_normalized_LAF's grid."""
    _, ch, h, w = img.shape
    B, N = laf.shape[:2]
    nlaf = normalize_laf(laf, h, w)
    pyr_idx = patch_pyramid_level(laf, h, w, PS)
    cur, level = img, 0
    out = torch.zeros(B, N, ch, PS, PS).to(nlaf)
    while True:
        _, ch, ch_h, ch_w = cur.shape
        for i in range(B):
            m = (pyr_idx[i] == level).view(-1)
            if m.sum() == 0:
                continue
            l = denormalize_laf(nlaf[i:i + 1, m], ch_h, ch_w)
            grid = F.affine_grid(l.view(-1, 2, 3), [int(m.sum()), ch, PS, PS], align_corners=False)
            grid[..., :, 0] = 2.0 * grid[..., :, 0].clone() / float(ch_w) - 1.0
            grid[..., :, 1] = 2.0 * grid[..., :, 1].clone() / float(ch_h) - 1.0
            patches = F.grid_sample(cur[i:i + 1].expand(grid.size(0), ch, ch_h, ch_w), grid, padding_mode='border',
                                    align_corners=False)
            out[i].masked_scatter_(m.view(-1, 1, 1, 1), patches)
        if min(ch_h, ch_w) < PS:
            break
        cur = pyrdown(cur)
        level += 1
    return out


def patch_pyramid_level(laf: torch.Tensor, h: int, w: int, PS: int) -> torch.Tensor:
    """The pyrdown level extract_patches_from_pyramid samples each LAF [B, N, 2, 3] of an h x w image from, in the LAF's dtype:
    log2(2 scale / PS) clamped to [0, min(h, w) // PS - 1], [B, N, 1, 1] int64.  Levels at or past patch_pyramid_levels are not
    visited, and their patches stay zero."""
    scale = 2.0 * get_laf_scale(denormalize_laf(normalize_laf(laf, h, w), h, w)) / float(PS)
    max_level = min(h, w) // PS
    return scale.log2().clamp(min=0.0, max=max(0, max_level - 1)).long()


def patch_pyramid_levels(h: int, w: int, PS: int) -> int:
    """How many pyrdown levels extract_patches_from_pyramid visits for patches of PS pixels."""
    n = 1
    while min(h, w) >= PS:
        h, w = int(float(h) / 2.0), int(float(w) // 2.0)
        n += 1
    return n


# ---- kornia/feature/orientation.py ----
def dominant_orientation(patch: torch.Tensor, num_bins: int = 36, eps: float = 1e-8, want_hist: bool = False):
    """kornia.feature.orientation.PatchDominantGradientOrientation.forward: angle in radians per patch [N, 1, PS, PS]."""
    N, _, ps, _ = patch.shape
    weighting = gaussian_kernel2d(ps, float(ps) / math.sqrt(2.0))[0].to(patch)
    smooth = torch.tensor([[[0.33, 0.34, 0.33]]]).to(patch)
    pi = PI.to(patch)
    g = spatial_gradient(patch, 'sobel')
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + eps) * weighting
    ori = torch.atan2(gy, gx + eps) + 2.0 * pi
    o_big = float(num_bins) * (ori + 1.0 * pi) / (2.0 * pi)
    bo0 = torch.floor(o_big)
    wo1 = o_big - bo0
    bo0 = bo0 % num_bins
    bo1 = (bo0 + 1) % num_bins
    wo0 = (1.0 - wo1) * mag
    wo1 = wo1 * mag
    bins = [F.adaptive_avg_pool2d((bo0 == i).to(patch) * wo0 + (bo1 == i).to(patch) * wo1, (1, 1)) for i in range(num_bins)]
    hist = torch.cat(bins, 1).view(-1, 1, num_bins)
    hist = F.conv1d(F.pad(hist, [1, 1], mode='circular'), smooth)
    _, idx = hist.view(-1, num_bins).max(1)
    angle = -((2.0 * pi * idx.to(patch) / float(num_bins)) - pi)
    return (angle, hist.view(-1, num_bins)) if want_hist else angle


def laf_orienter(laf: torch.Tensor, img: torch.Tensor, patch_size: int = 19, want_angles: bool = False):
    """kornia.feature.orientation.LAFOrienter(patch_size).forward."""
    B, N = laf.shape[:2]
    if N == 0:
        return (laf, laf.new_zeros(B, 0)) if want_angles else laf
    patches = extract_patches_from_pyramid(img, laf, patch_size).view(-1, 1, patch_size, patch_size)
    ang = dominant_orientation(patches).view(B, N)
    prev = get_laf_orientation(laf).view_as(ang)
    out = set_laf_orientation(laf, rad2deg(ang) + prev)
    return (out, ang) if want_angles else out


# ---- kornia/feature/siftdesc.py, integrated.py ----
def sift_pooling_kernel(ksize: int) -> torch.Tensor:
    ks_2 = float(ksize) / 2.0
    xc2 = ks_2 - (torch.arange(ksize).float() + 0.5 - ks_2).abs()
    return torch.outer(xc2, xc2) / (ks_2 ** 2)


def sift_descriptor(patch: torch.Tensor, rootsift: bool = True, num_ang_bins: int = 8, num_spatial_bins: int = 4,
                    clipval: float = 0.2) -> torch.Tensor:
    """kornia.feature.siftdesc.SIFTDescriptor.forward on patches [N, 1, PS, PS] -> [N, 8 * 4 * 4] (channel-major)."""
    N, _, ps, _ = patch.shape
    eps = 1e-10
    ksize = 2 * int(ps / (num_spatial_bins + 1))
    stride = ps // num_spatial_bins
    pad = ksize // 4
    gk = gaussian_kernel2d(ps, float(ps) / math.sqrt(2.0))[0].to(patch)
    pk = sift_pooling_kernel(ksize).to(patch).view(1, 1, ksize, ksize)
    pi = PI.to(patch)
    g = spatial_gradient(patch, 'diff')
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + eps)
    ori = torch.atan2(gy, gx + eps) + 2.0 * pi
    mag = mag * gk.expand_as(mag)
    o_big = float(num_ang_bins) * ori / (2.0 * pi)
    bo0_ = torch.floor(o_big)
    wo1_ = o_big - bo0_
    bo0 = bo0_ % num_ang_bins
    bo1 = (bo0 + 1) % num_ang_bins
    wo0 = (1.0 - wo1_) * mag
    wo1 = wo1_ * mag
    bins = [F.conv2d((bo0 == i).to(patch) * wo0 + (bo1 == i).to(patch) * wo1, pk, stride=stride, padding=pad)
            for i in range(num_ang_bins)]
    d = torch.cat(bins, dim=1).view(N, -1)
    d = F.normalize(d, p=2)
    d = torch.clamp(d, 0.0, float(clipval))
    d = F.normalize(d, p=2)
    if rootsift:
        d = torch.sqrt(F.normalize(d, p=1) + eps)
    return d


def laf_descriptors(img: torch.Tensor, laf: torch.Tensor, patch_size: int = 41, rootsift: bool = True) -> torch.Tensor:
    """kornia.feature.integrated.get_laf_descriptors with SIFTDescriptor(patch_size, rootsift=rootsift)."""
    B, N = laf.shape[:2]
    if N == 0:
        return torch.empty(B, 0, 128, dtype=img.dtype, device=img.device)
    p = extract_patches_from_pyramid(img, laf, patch_size)
    return sift_descriptor(p.view(B * N, 1, patch_size, patch_size), rootsift).view(B, N, -1)


# ---- kornia/feature/scale_space_detector.py ----
def octave_candidates(dog: torch.Tensor, sigma0: float, num_feats: int, mr_size: float = 6.0):
    """One octave of ScaleSpaceDetector.detect from its DoG [B, 1, L, h, w]: the per-octave top-k of every voxel's response
    (ties: lower voxel index first), then the border test.  Returns (responses [B, n], octave-pixel LAFs [B, n, 2, 3],
    voxel indices [B, n]), n = min(num_feats, voxels)."""
    B, CH, L, h, w = dog.shape
    coord_max, resp_max = conv_quad_interp3d(dog, 10.0)
    coord_min, resp_min = conv_quad_interp3d(-dog, 10.0)
    take_min = (resp_min > resp_max).to(resp_max.dtype)
    resp_max = resp_min * take_min + (1 - take_min) * resp_max
    coord_max = coord_min * take_min.unsqueeze(2) + (1 - take_min.unsqueeze(2)) * coord_max
    flat = resp_max.view(B, -1)
    coords = coord_max.view(B, 3, -1).permute(0, 2, 1)
    if flat.size(1) > num_feats:
        idx = _topk_low_index(flat, num_feats)
        best = torch.gather(flat, 1, idx)
        cbest = torch.gather(coords, 1, idx.unsqueeze(-1).repeat(1, 1, 3))
    else:
        idx = torch.arange(flat.size(1), device=dog.device).expand(B, -1)
        best, cbest = flat, coords
    n = best.size(1)
    sig = sigma0 * torch.pow(2.0, cbest[:, :, 0].contiguous().view(-1, 1, 1, 1) / 3.0).view(B, n, 1)   # _scale_index_to_scale
    cbest = torch.cat([sig, cbest[:, :, 1:]], dim=2)
    rot = torch.eye(2, dtype=dog.dtype, device=dog.device).view(1, 1, 2, 2)
    lafs = torch.cat([mr_size * cbest[:, :, 0].view(B, n, 1, 1) * rot, cbest[:, :, 1:3].view(B, n, 2, 1)], dim=3)
    good = laf_is_inside_image(lafs, h, w)
    return best * good.to(best.dtype), lafs, idx


def _topk_low_index(x: torch.Tensor, k: int) -> torch.Tensor:
    """torch.topk(x, k, dim=1).indices with ties broken by the lower index: a stable descending sort."""
    return torch.sort(x, dim=1, descending=True, stable=True).indices[:, :k]


def detect(img: torch.Tensor, num_feats: int, want_stages: bool = False):
    """ScaleSpaceDetector(num_feats, BlobDoG, ConvQuadInterp3d(10), ScalePyramid(3, 1.6, 32, True), scale_space_response=True,
    minima_are_also_good=True, mr_size=6).detect: (responses [B, num_feats], lafs [B, num_feats, 2, 3] in image pixels, before
    orientation)."""
    B, _, H, W = img.shape
    pyr, sigmas = scale_pyramid(img)
    resp, lafs, stages = [], [], []
    for o, octave in enumerate(pyr):
        h, w = octave.shape[-2:]
        dog = dog_response(octave)
        r, l, idx = octave_candidates(dog, float(sigmas[o][0, 0]), num_feats)
        stages.append(dict(dog=dog, resp=r, lafs=l, index=idx))
        resp.append(r)
        lafs.append(normalize_laf(l, h, w))
    resp = torch.cat(resp, dim=1)
    lafs = torch.cat(lafs, dim=1)
    idx = _topk_low_index(resp, num_feats)
    resp = torch.gather(resp, 1, idx)
    lafs = denormalize_laf(torch.gather(lafs, 1, idx.unsqueeze(-1).unsqueeze(-1).repeat(1, 1, 2, 3)), H, W)
    if want_stages:
        return resp, lafs, dict(pyramid=pyr, octaves=stages, index=idx)
    return resp, lafs


# ---- nn.Module stand-ins with kornia's constructor signatures (the fixture script stubs kornia with these) ----
class ScalePyramid(nn.Module):
    def __init__(self, n_levels: int = 3, init_sigma: float = 1.6, min_size: int = 15, double_image: bool = False):
        super().__init__()
        assert (n_levels, init_sigma, min_size, double_image) == (3, 1.6, 32, True), 'only the reference SIFT pyramid is restated'


class BlobDoG(nn.Module):
    pass


class ConvQuadInterp3d(nn.Module):
    def __init__(self, strict_maxima_bonus: float = 10.0, eps: float = 1e-7):
        super().__init__()
        assert strict_maxima_bonus == 10.0


class PassLAF(nn.Module):
    def forward(self, laf, img):
        return laf


class LAFOrienter(nn.Module):
    def __init__(self, patch_size: int = 32, num_angular_bins: int = 36, angle_detector=None):
        super().__init__()
        self.patch_size = patch_size

    def forward(self, laf, img):
        return laf_orienter(laf, img, self.patch_size)


class ScaleSpaceDetector(nn.Module):
    def __init__(self, num_features: int = 500, mr_size: float = 6.0, scale_pyr_module=None, resp_module=None, nms_module=None,
                 ori_module=None, aff_module=None, minima_are_also_good: bool = False, scale_space_response: bool = False):
        super().__init__()
        assert mr_size == 6.0 and minima_are_also_good and scale_space_response
        assert isinstance(resp_module, BlobDoG) and isinstance(nms_module, ConvQuadInterp3d) and isinstance(scale_pyr_module, ScalePyramid)
        self.num_features = num_features
        self.ori = ori_module
        self.calls = []                       # the stages of every call, for the fixture script

    def forward(self, img, mask=None):
        resp, lafs, stages = detect(img, self.num_features, want_stages=True)
        self.calls.append(dict(stages, det_resp=resp, det_lafs=lafs))
        return self.ori(lafs, img), resp


class SIFTDescriptor(nn.Module):
    def __init__(self, patch_size: int = 41, num_ang_bins: int = 8, num_spatial_bins: int = 4, rootsift: bool = True, clipval: float = 0.2):
        super().__init__()
        self.patch_size, self.rootsift = patch_size, rootsift

    def forward(self, patch):
        return sift_descriptor(patch, self.rootsift)


class LAFDescriptor(nn.Module):
    def __init__(self, patch_descriptor_module=None, patch_size: int = 32, grayscale_descriptor: bool = True):
        super().__init__()
        self.descriptor, self.patch_size = patch_descriptor_module, patch_size

    def forward(self, img, lafs):
        return laf_descriptors(img, lafs, self.patch_size, self.descriptor.rootsift)


class CornerGFTT(nn.Module):
    pass
