"""Homography-pretraining pairs (csrc/homography.cuh, openglue_b200/homography.py): the item of the reference's
OxfordParis1MDataset.__getitem__ (data/oxford_paris_dataset.py:27-66, no colour augmentation) for a batch of images.

1. CPU: a float64 / int64 restatement of OpenCV's arithmetic (getPerspectiveTransform's LU solve, warpPerspective's fixed-point
   INTER_LINEAR with a constant-0 border, cvtColor RGB2GRAY) equals cv2 on seeded images and reproduces the committed fixtures
   (oracle/gen_golden_homography.py, minted from the unmodified reference); argument errors; the C ABI's OG_EINVAL before any
   CUDA call.
2. GPU, og_homography_pairs through the C ABI into NaN-poisoned outputs followed by guard regions: every fixture case bit-equal
   (image0, image1, H_true); random offsets at B = 1 .. 16 bit-equal to the restatement run on the device; a degenerate corner
   configuration; a repeat call bit-identical.
3. GPU, end to end at 1472 x 1232 with offset 256: synthesize_homography_pairs -> SuperPointNet -> prepare_features_output ->
   generate_gt_matches(3, 3) finds many ground-truth matches under H_true and almost none under its transpose; one training step
   (SuperGlue.train() + criterion + backward) on these pairs equals, bit for bit, the step on the restatement's images.
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from gen_golden_homography import CASES, case_offsets, images_sha256, pair_images  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
DEV = 'cuda:0'
DBL_EPS = 2.220446049250313e-16
GUARD = 257


# ---- the restatement ----
def _f32(x) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def cv_fit(src, dst):
    """cv2.getPerspectiveTransform(src, dst) (4 x (x, y) float32 points) as 9 floats: the 8 x 8 system with float32 products, LU
    with partial pivoting (first largest |pivot|), alpha = a[j][i] * (-1 / a[i][i]), back substitution dividing by the pivot,
    M[8] = 1; a pivot below 100 DBL_EPSILON gives [0] * 8 + [1].  Python floats are IEEE doubles: no FMA."""
    a = [[0.0] * 8 for _ in range(8)]
    b = [0.0] * 8
    for i in range(4):
        sx, sy, dx, dy = (_f32(v) for v in (src[i][0], src[i][1], dst[i][0], dst[i][1]))
        a[i][0] = a[i + 4][3] = sx
        a[i][1] = a[i + 4][4] = sy
        a[i][2] = a[i + 4][5] = 1.0
        a[i][6], a[i][7] = _f32(-sx * dx), _f32(-sy * dx)           # exact double product, rounded once to float
        a[i + 4][6], a[i + 4][7] = _f32(-sx * dy), _f32(-sy * dy)
        b[i], b[i + 4] = dx, dy
    for i in range(8):
        k = i
        for j in range(i + 1, 8):
            if abs(a[j][i]) > abs(a[k][i]):
                k = j
        if abs(a[k][i]) < 100 * DBL_EPS:
            return [0.0] * 8 + [1.0]
        a[i], a[k] = a[k], a[i]
        b[i], b[k] = b[k], b[i]
        d = -1.0 / a[i][i]
        for j in range(i + 1, 8):
            alpha = a[j][i] * d
            for c in range(i + 1, 8):
                a[j][c] += alpha * a[i][c]
            b[j] += alpha * b[i]
    for i in range(7, -1, -1):
        s = b[i]
        for c in range(i + 1, 8):
            s -= a[i][c] * b[c]
        b[i] = s / a[i][i]
    return b + [1.0]


def cv_invert3(M):
    """cv::invert(DECOMP_LU) for 3 x 3: cofactors times 1 / det3; zeros when det3 == 0"""
    S = lambda r, c: M[3 * r + c]  # noqa: E731
    det = S(0, 0) * (S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) - S(0, 1) * (S(1, 0) * S(2, 2) - S(1, 2) * S(2, 0)) \
        + S(0, 2) * (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0))
    if det == 0.0:
        return [0.0] * 9
    r = 1.0 / det
    return [(S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) * r, (S(0, 2) * S(2, 1) - S(0, 1) * S(2, 2)) * r,
            (S(0, 1) * S(1, 2) - S(0, 2) * S(1, 1)) * r, (S(1, 2) * S(2, 0) - S(1, 0) * S(2, 2)) * r,
            (S(0, 0) * S(2, 2) - S(0, 2) * S(2, 0)) * r, (S(0, 2) * S(1, 0) - S(0, 0) * S(1, 2)) * r,
            (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0)) * r, (S(0, 1) * S(2, 0) - S(0, 0) * S(2, 1)) * r,
            (S(0, 0) * S(1, 1) - S(0, 1) * S(1, 0)) * r]


def gray_u8(rgb: torch.Tensor) -> torch.Tensor:
    """cvtColor RGB2GRAY on uint8 [..., 3] -> int64"""
    rgb = rgb.long()
    return (9798 * rgb[..., 0] + 19235 * rgb[..., 1] + 3735 * rgb[..., 2] + (1 << 14)) >> 15


def cv_warp_crop(img: torch.Tensor, Minv, off: int) -> torch.Tensor:
    """the crop [off, H-off) x [off, W-off) of cv2.warpPerspective(img, M, (W, H)) (INTER_LINEAR, constant 0), given Minv =
    the inverse warpPerspective computes; img [H, W, 3] uint8 on any device -> [h, w, 3] int64.  WarpPerspectiveInvoker's
    arithmetic (per-block origin, 32 / W, rint to 1/32 px) and remapBilinear's 15-bit weights."""
    H, W = img.shape[:2]
    dev = img.device
    bh0 = min(16, H)
    bw0 = min(1024 // bh0, W)
    y = torch.arange(off, H - off, device=dev, dtype=torch.float64)[:, None]
    x = torch.arange(off, W - off, device=dev, dtype=torch.int64)[None]
    xb, x1 = (x // bw0 * bw0).double(), (x % bw0).double()
    M = Minv
    X0 = M[0] * xb + M[1] * y + M[2]
    Y0 = M[3] * xb + M[4] * y + M[5]
    W0 = M[6] * xb + M[7] * y + M[8]
    Wd = W0 + M[6] * x1
    Wd = torch.where(Wd != 0, 32.0 / Wd, torch.zeros_like(Wd))
    fX = ((X0 + M[0] * x1) * Wd).clamp(-2.0 ** 31, 2.0 ** 31 - 1)
    fY = ((Y0 + M[3] * x1) * Wd).clamp(-2.0 ** 31, 2.0 ** 31 - 1)
    Xi, Yi = torch.round(fX).long(), torch.round(fY).long()       # round half to even, as cvRound
    sx, sy = (Xi >> 5).clamp(-32768, 32767), (Yi >> 5).clamp(-32768, 32767)
    fx, fy = Xi & 31, Yi & 31
    src = img.long()
    acc = torch.full((*sx.shape, 3), 1 << 14, dtype=torch.int64, device=dev)
    for dy, wy in ((0, 32 - fy), (1, fy)):
        for dx, wx in ((0, 32 - fx), (1, fx)):
            px, py = sx + dx, sy + dy
            inside = (px >= 0) & (px < W) & (py >= 0) & (py < H)
            v = src[py.clamp(0, H - 1), px.clamp(0, W - 1)] * inside[..., None]
            acc += v * (wy * wx * 32)[..., None]
    return acc >> 15


def corners(H: int, W: int, off: int, crop: bool):
    if crop:
        h, w = H - 2 * off, W - 2 * off
        return [[0, 0], [0, h - 1], [w - 1, 0], [w - 1, h - 1]]
    return [[off, off], [off, H - off - 1], [W - off - 1, off], [W - off - 1, H - off - 1]]


def restate(images: torch.Tensor, offsets: torch.Tensor, off: int):
    """-> (image0 u8 [B,h,w], image1 u8 [B,h,w], H_true f32 [B,3,3], H_true f64) for images [B,H,W,3] uint8 on any device"""
    B, H, W, _ = images.shape
    i0, i1, h32, h64 = [], [], [], []
    for b in range(B):
        o = offsets[b].tolist()
        dw = corners(H, W, off, False)
        dc = corners(H, W, off, True)
        Hw = cv_fit([[dw[i][0] + o[i][0], dw[i][1] + o[i][1]] for i in range(4)], dw)
        Ht = cv_fit([[dc[i][0] + o[i][0], dc[i][1] + o[i][1]] for i in range(4)], dc)
        crop = images[b, off:H - off, off:W - off]
        i0.append(gray_u8(crop).to(torch.uint8))
        i1.append(gray_u8(cv_warp_crop(images[b], cv_invert3(Hw), off)).to(torch.uint8))
        h64.append(torch.tensor(Ht, dtype=torch.float64).view(3, 3))
        h32.append(h64[-1].float())
    return torch.stack(i0), torch.stack(i1), torch.stack(h32), torch.stack(h64)


def by255(u8: torch.Tensor) -> torch.Tensor:
    """the reference's torch.FloatTensor(u8) / 255. (on the CPU: correctly rounded; torch on CUDA multiplies by a reciprocal)"""
    return (u8.cpu().float() / 255.).to(u8.device)


def _fx(name):
    return torch.load(os.path.join(GOLDEN, name + '.pt'), weights_only=False)


def _inputs(fx):
    c = fx['case']
    images = pair_images(c['batch'], c['H'], c['W'], c['seed'])
    assert images_sha256(images) == fx['sha256'], 'the regenerated images differ from the ones the fixture was minted from'
    assert torch.equal(case_offsets(c['kind'], c['batch'], c['offset'], c['seed']), fx['warp_offset'])
    return images, fx['warp_offset'], c['offset']


def _check_against_fixture(fx, i0, i1, h32):
    assert torch.equal(h32, fx['H_true']), (h32 - fx['H_true']).abs().max()
    if 'image0' in fx:
        assert torch.equal(i0, fx['image0']), int((i0 != fx['image0']).sum())
        assert torch.equal(i1, fx['image1']), int((i1 != fx['image1']).sum())
    else:
        assert [images_sha256(t) for t in i0] == fx['image0_sha256']
        assert [images_sha256(t) for t in i1] == fx['image1_sha256'], \
            [int((a[list(fx['rows'])] != r).sum()) for a, r in zip(i1, fx['image1_rows'])]


# ---- CPU ----
def test_restatement_equals_cv2():
    cv2 = pytest.importorskip('cv2')
    import numpy as np
    g = torch.Generator().manual_seed(3)
    checked = 0
    for (H, W, off, seed) in [(1232, 1472, 256, 1), (40, 37, 8, 2), (33, 50, 10, 3), (64, 98, 16, 4), (17, 300, 4, 5),
                              (300, 17, 4, 6), (36, 40, 14, 7)]:
        images = pair_images(3, H, W, seed)
        for b in range(3):
            o = torch.randint(-off, off, (4, 2), generator=g).tolist()
            dw = corners(H, W, off, False)
            src = np.array([[dw[i][0] + o[i][0], dw[i][1] + o[i][1]] for i in range(4)], np.float32)
            M = cv2.getPerspectiveTransform(src, np.array(dw, np.float32))
            if M[2, 2] != 1.0:
                continue                              # cv2 4.13 left its LU solve for an SVD: not restated
            assert M.reshape(-1).tolist() == cv_fit(src.tolist(), dw)
            full = cv2.warpPerspective(images[b].numpy(), M, (W, H))
            got = cv_warp_crop(images[b], cv_invert3(M.reshape(-1).tolist()), off)
            assert torch.equal(got, torch.from_numpy(full[off:H - off, off:W - off]).long())
            want_gray = cv2.cvtColor(full, cv2.COLOR_RGB2GRAY)
            assert torch.equal(gray_u8(torch.from_numpy(full)), torch.from_numpy(want_gray).long())
            checked += 1
    assert checked >= 18


@pytest.mark.parametrize('name', list(CASES))
def test_restatement_reproduces_fixtures(name):
    fx = _fx(name)
    images, offsets, off = _inputs(fx)
    i0, i1, h32, h64 = restate(images, offsets, off)
    assert torch.equal(h64, fx['H_true_f64'])
    _check_against_fixture(fx, i0, i1, h32)
    if fx['case']['kind'] == 'zero':
        assert torch.equal(i0, i1)


def test_division_by_255_is_correctly_rounded():
    """the kernel divides with __fdiv_rn: the reference's CPU division, unlike torch's on CUDA"""
    import numpy as np
    u8 = torch.arange(256, dtype=torch.uint8)
    assert torch.equal(by255(u8), torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255.0)))


def test_singular_configuration_takes_the_lu_failure_rule():
    """three source corners on a line: a pivot of the LU falls below 100 DBL_EPSILON, so H = [[0,0,0],[0,0,0],[0,0,1]] and the
    warp's inverse is zero (every destination pixel samples source (0, 0)).  cv2 4.13 answers with an SVD here instead."""
    H, W, off = 48, 48, 16
    o = [[0, 0], [0, 0], [-8, 7], [0, 0]]                              # (0,0), (7,7), (15,15) in crop coordinates
    dc = corners(H, W, off, True)
    assert cv_fit([[dc[i][0] + o[i][0], dc[i][1] + o[i][1]] for i in range(4)], dc) == [0.0] * 8 + [1.0]
    dw = corners(H, W, off, False)
    assert cv_fit([[dw[i][0] + o[i][0], dw[i][1] + o[i][1]] for i in range(4)], dw) == [0.0] * 8 + [1.0]
    images = pair_images(1, H, W, 9)
    _, i1, h32, _ = restate(images, torch.tensor([o]), off)
    assert torch.equal(h32[0], torch.tensor([[0.0, 0, 0], [0, 0, 0], [0, 0, 1]]))
    assert (i1 == gray_u8(images[0, 0, 0]).to(torch.uint8)).all()


def test_argument_errors():
    from openglue_b200 import synthesize_homography_pairs as syn
    img = torch.zeros(2, 40, 50, 3, dtype=torch.uint8)
    with pytest.raises(TypeError):
        syn(img.float(), 8)
    with pytest.raises(ValueError):
        syn(torch.zeros(2, 40, 50, dtype=torch.uint8), 8)
    with pytest.raises(ValueError):
        syn(torch.zeros(2, 40, 50, 4, dtype=torch.uint8), 8)
    for off in (0, -1, 20, 25):
        with pytest.raises(ValueError):
            syn(img, off)
    with pytest.raises(TypeError):
        syn(img, 2.5)
    with pytest.raises(ValueError):
        syn(img, 8, warp_offset=torch.zeros(2, 4, 3, dtype=torch.int32))
    with pytest.raises(TypeError):
        syn(img, 8, warp_offset=torch.zeros(2, 4, 2))
    for bad in (8, -9):
        wo = torch.zeros(2, 4, 2, dtype=torch.int32)
        wo[1, 2, 0] = bad
        with pytest.raises(ValueError):
            syn(img, 8, warp_offset=wo)
    with pytest.raises(RuntimeError, match='CUDA'):                    # CPU tensors are refused
        syn(img, 8, warp_offset=torch.zeros(2, 4, 2, dtype=torch.int32))
    with pytest.raises(RuntimeError, match='CUDA'):
        syn(img, 8)


def test_cabi_einval_before_any_cuda_call():
    from openglue_b200 import _cabi
    lib = _cabi.lib()
    p = C.c_void_p(16)                                                 # never dereferenced: every call below fails its checks first
    good = dict(B=2, H=40, W=50, off=8)

    def call(B=2, H=40, W=50, off=8, rgb=p, wo=p, i0=p, i1=p, h=p):
        return lib.og_homography_pairs(rgb, B, H, W, off, wo, i0, i1, h, None)
    assert good
    for kw in (dict(off=0), dict(off=-3), dict(off=20), dict(H=16, off=8), dict(B=0), dict(B=-1), dict(B=65536),
               dict(rgb=None), dict(wo=None), dict(i0=None), dict(i1=None), dict(h=None), dict(W=0)):
        assert call(**kw) == -1, kw                                    # OG_EINVAL


# ---- GPU ----
def _lib():
    from openglue_b200 import _cabi
    return _cabi.lib()


def _run_cabi(images_dev, offsets_dev, off):
    """og_homography_pairs into NaN-poisoned outputs, each followed by GUARD NaNs that must stay NaN"""
    B, H, W, _ = images_dev.shape
    h, w = H - 2 * off, W - 2 * off
    bufs = [torch.full((B * h * w + GUARD,), float('nan'), device=DEV) for _ in range(2)]
    hbuf = torch.full((B * 9 + GUARD,), float('nan'), device=DEV)
    from openglue_b200._cabi import ptr, stream
    rc = _lib().og_homography_pairs(ptr(images_dev), B, H, W, off, ptr(offsets_dev), ptr(bufs[0]), ptr(bufs[1]), ptr(hbuf), stream())
    assert rc == 0, _lib().og_last_error()
    torch.cuda.synchronize()
    for t in (*bufs, hbuf):
        assert torch.isnan(t[-GUARD:]).all(), 'a write past the end of an output'
    i0, i1 = (t[:B * h * w].view(B, h, w) for t in bufs)
    Ht = hbuf[:B * 9].view(B, 3, 3)
    for t in (i0, i1, Ht):
        assert not torch.isnan(t).any(), 'an output element was not written'
    u0, u1 = (torch.round(t.double() * 255).to(torch.uint8) for t in (i0, i1))
    assert torch.equal(by255(u0), i0) and torch.equal(by255(u1), i1)            # exactly torch.FloatTensor(u8) / 255.
    return u0, u1, Ht


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_fixture_cases_bit_equal(name):
    fx = _fx(name)
    images, offsets, off = _inputs(fx)
    u0, u1, Ht = _run_cabi(images.to(DEV), offsets.to(DEV), off)
    _check_against_fixture(fx, u0.cpu(), u1.cpu(), Ht.cpu())


@pytest.mark.gpu
@pytest.mark.parametrize('B,H,W,off', [(1, 40, 37, 8), (3, 133, 50, 10), (5, 36, 40, 14), (16, 96, 130, 24), (2, 240, 321, 60)])
def test_random_offsets_match_restatement_on_device(B, H, W, off):
    images = pair_images(B, H, W, 100 + B).to(DEV)
    g = torch.Generator().manual_seed(B * 1000 + W)
    offsets = torch.randint(-off, off, (B, 4, 2), generator=g, dtype=torch.int32)
    u0, u1, Ht = _run_cabi(images, offsets.to(DEV), off)
    r0, r1, r32, _ = restate(images, offsets, off)
    assert torch.equal(u0, r0) and torch.equal(Ht, r32.to(DEV))
    assert torch.equal(u1, r1), int((u1 != r1).sum())
    again = _run_cabi(images, offsets.to(DEV), off)
    for a, b in zip((u0, u1, Ht), again):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_singular_configuration_on_device():
    H, W, off = 48, 48, 16
    images = pair_images(2, H, W, 9).to(DEV)
    offsets = torch.tensor([[[0, 0], [0, 0], [-8, 7], [0, 0]], [[3, -2], [1, 5], [-4, 0], [2, 2]]], dtype=torch.int32)
    u0, u1, Ht = _run_cabi(images, offsets.to(DEV), off)
    r0, r1, r32, _ = restate(images, offsets, off)
    assert torch.equal(Ht[0].cpu(), torch.tensor([[0.0, 0, 0], [0, 0, 0], [0, 0, 1]]))
    assert torch.equal(u0, r0) and torch.equal(u1, r1) and torch.equal(Ht, r32.to(DEV))


@pytest.mark.gpu
def test_public_function_shapes_and_random_offsets():
    from openglue_b200 import synthesize_homography_pairs
    images = pair_images(3, 64, 98, 5).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    out = synthesize_homography_pairs(images, 16, generator=g)
    assert out['image0'].shape == (3, 1, 32, 66) and out['image1'].shape == (3, 1, 32, 66)
    assert out['transformation']['type'] == ['perspective'] * 3 and out['transformation']['H'].shape == (3, 3, 3)
    g = torch.Generator(device=DEV).manual_seed(4)
    wo = torch.randint(-16, 16, (3, 4, 2), generator=g, device=DEV, dtype=torch.int32)
    ref = synthesize_homography_pairs(images, 16, warp_offset=wo)
    assert torch.equal(out['image1'], ref['image1']) and torch.equal(out['transformation']['H'], ref['transformation']['H'])
    r0, r1, r32, _ = restate(images, wo.cpu(), 16)
    assert torch.equal(ref['image0'][:, 0], by255(r0)) and torch.equal(ref['image1'][:, 0], by255(r1))


@pytest.mark.gpu
def test_end_to_end_pretraining_size():
    """1472 x 1232, offset 256 (config/homography_pretraining.yaml): the fixture's pairs -> SuperPoint -> ground truth -> one
    training step"""
    import openglue_b200
    from openglue_b200 import SuperGlue, SuperPointNet, criterion, generate_gt_matches, synthesize_homography_pairs
    from openglue_b200.synthetic import default_config, synthetic_state_dict
    fx = _fx('hg_pretrain')
    images, offsets, off = _inputs(fx)
    images = images.to(DEV)
    pairs = synthesize_homography_pairs(images, off, warp_offset=offsets.to(DEV))
    u0, u1 = (torch.round(pairs[k][:, 0].double() * 255).to(torch.uint8).cpu() for k in ('image0', 'image1'))
    _check_against_fixture(fx, u0, u1, pairs['transformation']['H'].cpu())
    torch.manual_seed(0)
    net = SuperPointNet(max_keypoints=1024, keypoint_threshold=0.005).eval().to(DEV)
    conv = openglue_b200.get_laf_to_sideinfo_converter('none')

    def features(batch):
        with torch.no_grad():
            f0 = openglue_b200.prepare_features_output(*net(batch['image0']), conv)
            f1 = openglue_b200.prepare_features_output(*net(batch['image1']), conv)
        return f0, f1

    f0, f1 = features(pairs)
    _, y = generate_gt_matches(pairs, f0, f1, 3, 3)
    true = int((y['gt_matches0'] >= 0).sum())
    swapped = {**pairs, 'transformation': {'type': ['perspective'] * 4, 'H': pairs['transformation']['H'].transpose(1, 2).contiguous()}}
    _, yt = generate_gt_matches(swapped, f0, f1, 3, 3)
    transposed = int((yt['gt_matches0'] >= 0).sum())
    n = f0['keypoints'].shape[0] * f0['keypoints'].shape[1]
    print(f'\n{n} keypoints: {true} ground-truth matches under H_true, {transposed} under its transpose')
    assert true >= 0.1 * n and transposed <= 0.02 * n

    # one training step on these pairs equals the step on the restatement's images (the reference's item, bit for bit)
    r0, r1, r32, _ = restate(images, offsets, off)
    same = {'image0': by255(r0).unsqueeze(1).to(DEV), 'image1': by255(r1).unsqueeze(1).to(DEV),
            'transformation': {'type': ['perspective'] * 4, 'H': r32.to(DEV)}}
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=20)
    results = []
    for batch in (pairs, same):
        model = SuperGlue(dict(cfg))
        model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
        model = model.to(DEV).train()
        g0, g1 = features(batch)
        data, y_true = generate_gt_matches(batch, g0, g1, 3, 3)
        loss = criterion(y_true, model(data), margin=None)['loss']
        loss.backward()
        results.append((loss.detach(), {k: p.grad.clone() for k, p in model.named_parameters()}))
    assert torch.isfinite(results[0][0]) and torch.equal(results[0][0], results[1][0])
    for k, gr in results[0][1].items():
        assert torch.equal(gr, results[1][1][k]), k
