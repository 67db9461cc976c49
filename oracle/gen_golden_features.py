"""Mint golden vectors for the LAF side information (prepare_features_output) and the stand-alone matcher (OpenGlueMatcher) by
running the UNMODIFIED reference: ``models/laf_converter.py`` (get_laf_to_sideinfo_converter and its conversion functions),
``models/features/utils.py::prepare_features_output`` and ``inference.OpenGlueMatcher.forward`` on pre-extracted features (no
feature extractor runs), with the reference's ``SuperGlue`` as the matcher.

TEST INFRASTRUCTURE.  Runs only where the reference is checked out; outputs are committed under tests/golden/feat_*.pt.
kornia is not installed here, so its two helpers these modules call are restated from the published kornia source and patched
in (as nms2d is for the SuperPoint fixtures): get_laf_scale and get_laf_center below.

Converter fixture (feat_convert.pt): SIFT-like frames (scales 0.5 - 64 px, every orientation, anisotropy and shear, reflections),
near-singular frames (where the 1e-10 of get_laf_scale dominates), SuperPoint's identity frames and zero responses; the reference's
keypoints and side information for every method with and without log_response, in float32 and float64.

Matcher fixtures (feat_match_*.pt): 'affine' side information, planted correspondences (openglue_b200.synthetic.synthetic_pairs
with a frame per keypoint, related between planted pairs); the reference's seven outputs in float32 and float64, plus what the
decisive-row rule of the parity tests needs from the float64 scores (gen_golden.py stores the same).  Inputs are regenerated from the
seeds by ``matcher_inputs``; the fixture records the sha256 of their bytes.

    python oracle/gen_golden_features.py [case ...]
"""
from __future__ import annotations

import copy
import hashlib
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict  # noqa: E402

METHODS = ('none', 'scale', 'rotation', 'scale_rotation', 'affine')
MATCH_CASES = {
    # name: (batch, n, m, config kwargs, log_transform_response, seed)
    'feat_match_affine': (2, 1000, 968, dict(descriptor_dim=128, num_stages=3, num_iters=50, side_info_size=6), True, 21),
    'feat_match_c5': (1, 4096, 1024, dict(descriptor_dim=128, num_stages=18, num_iters=50, side_info_size=6), False, 22),   # BASELINE configs[4]
}
MATCH_THRESHOLD = 0.2
IMAGE_HW = (720, 960)


# ---- kornia restated (kornia/feature/laf.py, published source) ----
def get_laf_scale(LAF: torch.Tensor) -> torch.Tensor:
    """kornia.feature.get_laf_scale: sqrt(|det(A) + eps|) of the 2x2 part, [B, N, 1, 1]"""
    eps = 1e-10
    out = LAF[..., 0:1, 0:1] * LAF[..., 1:2, 1:2] - LAF[..., 1:2, 0:1] * LAF[..., 0:1, 1:2] + eps
    return out.abs().sqrt()


def get_laf_center(LAF: torch.Tensor) -> torch.Tensor:
    """kornia.feature.get_laf_center: the last column, [B, N, 2]"""
    return LAF[..., 2]


def sift_frames(g: torch.Generator, count: int, width: float = 1280.0, height: float = 960.0) -> torch.Tensor:
    """[count, 2, 3] SIFT-like LAFs: scale 0.5 * 128^u (0.5 - 64 px), angle in [0, 2 pi), anisotropy 2^(2u - 1), shear in
    [-0.5, 0.5), one in six reflected (negative determinant); centres uniform over the image"""
    u = torch.rand(count, 6, generator=g, dtype=torch.float64)
    s, th = 0.5 * 128.0 ** u[:, 0], 2 * math.pi * u[:, 1]
    a, h = 2.0 ** (2 * u[:, 2] - 1), u[:, 3] - 0.5
    c, sn = torch.cos(th), torch.sin(th)
    rot = torch.stack([torch.stack([c, -sn], -1), torch.stack([sn, c], -1)], -2)
    shape = torch.zeros(count, 2, 2, dtype=torch.float64)
    shape[:, 0, 0], shape[:, 0, 1], shape[:, 1, 1] = a, h, 1 / a
    A = s[:, None, None] * rot @ shape
    A[:, :, 0] *= torch.where(u[:, 4] < 1 / 6, -1.0, 1.0)[:, None]
    xy = torch.rand(count, 2, generator=g, dtype=torch.float64) * torch.tensor([width - 1, height - 1], dtype=torch.float64)
    return torch.cat([A, xy[:, :, None]], -1).float()


def convert_inputs(seed: int = 5, batch: int = 2, n: int = 517):
    """(lafs [B, n, 2, 3], responses [B, n]): every kind of frame the converter has to get right"""
    g = torch.Generator().manual_seed(seed)
    lafs = sift_frames(g, batch * n)
    R = lafs.shape[0]
    lafs[0:64, :, :2] = torch.eye(2)                                         # SuperPoint: identity frames at integer pixels
    lafs[0:64, :, 2] = torch.floor(lafs[0:64, :, 2])
    k = torch.tensor([[1.0, 2.0], [-4.0, 0.5], [3.0, -8.0], [0.25, 16.0]])     # rank one with exact products: det = 0 exactly
    for i in range(64, 96):
        p, q = k[i % 4]
        t = [1.0, -2.0, 0.5, 4.0][(i // 4) % 4]
        lafs[i, :, :2] = torch.tensor([[p, q], [t * p, t * q]])
    lafs[96:100, :, :2] = 0.0                                                # degenerate: zero frame
    lafs[100:132, :, :2] *= 1e-6 / lafs[100:132, :, :2].abs().amax((1, 2), keepdim=True)   # |det| ~ 1e-12: the 1e-10 dominates
    u = torch.rand(R, 2, generator=g)
    responses = u[:, 0] * 10.0 ** (3 * u[:, 1] - 2)                          # 0 .. 10, spread over four decades
    responses[::9] = 0.0
    return lafs.view(batch, n, 2, 3).contiguous(), responses.view(batch, n).contiguous()


def matcher_inputs(batch: int, n: int, m: int, d: int, seed: int):
    """pre-extracted features of `batch` image pairs: lafs / responses / descriptors {0, 1}; planted pairs share their response
    and descriptor (synthetic_pairs) and have related frames (image-1 frame = 0.9 x the image-0 frame, rotated by a fixed angle)"""
    data = synthetic_pairs(batch, n, m, d, 1, family='planted', seed=seed, image_wh=(IMAGE_HW[1], IMAGE_HW[0]))
    g = torch.Generator().manual_seed(seed + 1)
    A0 = sift_frames(g, batch * n)[:, :, :2].view(batch, n, 2, 2)
    A1 = sift_frames(g, batch * m)[:, :, :2].view(batch, m, 2, 2)
    c, s = math.cos(0.3), math.sin(0.3)
    rot = torch.tensor([[c, -s], [s, c]]) * 0.9
    planted = data['planted_matches0']
    for b in range(batch):
        src = (planted[b] >= 0).nonzero()[:, 0]
        A1[b, planted[b, src]] = rot @ A0[b, src]
    lafs0 = torch.cat([A0, data['keypoints0'][..., None]], -1).contiguous()
    lafs1 = torch.cat([A1, data['keypoints1'][..., None]], -1).contiguous()
    return {'lafs0': lafs0, 'responses0': data['side_info0'][..., 0].contiguous(), 'descriptors0': data['local_descriptors0'],
            'lafs1': lafs1, 'responses1': data['side_info1'][..., 0].contiguous(), 'descriptors1': data['local_descriptors1']}


def inputs_sha256(inputs: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(inputs):
        h.update(inputs[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def match_config(log_transform_response: bool, threshold: float = MATCH_THRESHOLD) -> dict:
    return {'superglue': {'laf_to_sideinfo_method': 'affine', 'log_transform_response': log_transform_response},
            'inference': {'match_threshold': threshold}}


def _reference():
    from gen_golden import _stub_modules
    sys.path.insert(0, os.environ.get('OPENGLUE_REFERENCE', '/root/reference'))
    _stub_modules()
    import kornia.feature as KF                                              # the stub module
    KF.laf.get_laf_scale = get_laf_scale
    KF.get_laf_center = get_laf_center
    import inference                                                         # the reference, unmodified
    from models.features.utils import prepare_features_output
    from models.laf_converter import get_laf_to_sideinfo_converter
    from models.superglue.superglue import SuperGlue
    return inference, prepare_features_output, get_laf_to_sideinfo_converter, SuperGlue


def mint_convert(out_dir):
    _, prepare, get_conv, _ = _reference()
    lafs, resp = convert_inputs()
    fx = {'lafs': lafs, 'responses': resp, 'side': {}, 'side_f64': {},
          'reference': 'models/laf_converter.py + models/features/utils.py:54-65 (kornia get_laf_scale / get_laf_center restated), '
                       'torch ' + torch.__version__}
    for method in METHODS:
        for lr in (False, True):
            conv = get_conv(method)
            o32 = prepare(lafs, resp, torch.zeros(*lafs.shape[:2], 1), conv, log_response=lr)
            o64 = prepare(lafs.double(), resp.double(), torch.zeros(*lafs.shape[:2], 1), conv, log_response=lr)
            assert o32['side_info'].shape[-1] == 1 + conv.side_info_dim
            fx['keypoints'] = o32['keypoints'].contiguous()
            fx['side'][(method, lr)] = o32['side_info'].contiguous()
            fx['side_f64'][(method, lr)] = o64['side_info'].contiguous()
    torch.save(fx, os.path.join(out_dir, 'feat_convert.pt'))
    print(f'feat_convert: {tuple(lafs.shape)} frames, {len(fx["side"])} cases')


class _Recorder(torch.nn.Module):
    """the matcher, keeping the last scores it returned"""

    def __init__(self, sg):
        super().__init__()
        self.sg, self.scores = sg, None

    def forward(self, data):
        out = self.sg(data)
        self.scores = out['scores']
        return out


def mint_match(name, out_dir):
    inference, _, _, SuperGlue = _reference()
    batch, n, m, kw, log_resp, seed = MATCH_CASES[name]
    cfg = default_config(**kw)
    sd = synthetic_state_dict(cfg, seed=0)
    inputs = matcher_inputs(batch, n, m, cfg['descriptor_dim'], seed)
    fx = {'name': name, 'case': dict(batch=batch, n=n, m=m, log_transform_response=log_resp, seed=seed, image_hw=IMAGE_HW),
          'config': cfg, 'weights_seed': 0, 'sha256': inputs_sha256(inputs), 'match_threshold': MATCH_THRESHOLD,
          'reference': 'inference.py:124-211 OpenGlueMatcher.forward on pre-extracted features (kornia get_laf_scale / '
                       'get_laf_center restated), torch ' + torch.__version__}
    scores = {}
    runs = [(torch.float32, 'f32', MATCH_THRESHOLD), (torch.float64, 'f64', MATCH_THRESHOLD)]
    if batch * n <= 4096:
        runs.append((torch.float32, 'empty', 1.0))                          # nothing clears a threshold of 1: the no-match shapes
    for dtype, tag, thr in runs:
        sg = SuperGlue(copy.deepcopy(cfg)).eval()
        sg.load_state_dict(sd, strict=True)
        rec = _Recorder(sg.to(dtype))
        matcher = inference.OpenGlueMatcher(None, rec, match_config(log_resp, thr))
        data = {k: v.to(dtype) for k, v in inputs.items()}
        data['image0'] = torch.zeros(batch, 1, *IMAGE_HW, dtype=dtype)
        data['image1'] = torch.zeros(batch, 1, *IMAGE_HW, dtype=dtype)
        with torch.no_grad():
            out = matcher(data)
        if tag == 'empty':
            fx['empty_shapes'] = {k: tuple(v.shape) for k, v in out.items()}
            fx['empty_dtypes'] = {k: str(v.dtype) for k, v in out.items()}
            continue
        fx[tag] = {k: v.contiguous().clone() for k, v in out.items()}
        scores[tag] = rec.scores
    s64 = scores['f64'][:, :-1, :-1]
    fx['ref32_vs_ref64_max_abs'] = float((scores['f32'].double() - scores['f64']).abs().max())
    fx['row_argmax_f64'] = s64.argmax(2)
    top2 = s64.topk(2, dim=2).values
    fx['row_top2_gap_f64'] = (top2[..., 0] - top2[..., 1]).float()
    top2c = s64.topk(2, dim=1).values
    fx['col_top2_gap_f64'] = (top2c[:, 0] - top2c[:, 1]).float()
    fx['matching_scores0_f64'] = s64.max(2).values.exp().float()            # before the mutual mask
    torch.save(fx, os.path.join(out_dir, name + '.pt'))
    print(f'{name}: {fx["f32"]["confidence"].numel()} matches (f64: {fx["f64"]["confidence"].numel()}), '
          f'ref32-vs-ref64 {fx["ref32_vs_ref64_max_abs"]:.2e}')


def main():
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    only = sys.argv[1:]
    if not only or 'feat_convert' in only:
        mint_convert(out_dir)
    for name in MATCH_CASES:
        if not only or name in only:
            mint_match(name, out_dir)


if __name__ == '__main__':
    main()
