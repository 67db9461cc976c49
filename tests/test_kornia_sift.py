"""kornia's DoG SIFT front-end (openglue_b200.SIFT, csrc/kornia_sift.cuh) on the H100: every stage on the oracle's own inputs
(oracle/kornia_sift_oracle.py, a restatement of kornia 0.6.3), end to end against fixtures minted by the unmodified reference
(oracle/gen_golden_kornia_sift.py: tests/golden/ksift_*.pt), and the front-end's batch, padded and image-pair forms."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_kornia_sift import load_fixture  # noqa: E402
from openglue_b200 import SIFT, ImagePairMatcher, ImagePairTrainStep, _cabi  # noqa: E402
from openglue_b200._cabi import ptr  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NF = 1024
CASES = ['ksift_tiny', 'ksift_small', 'ksift_odd', 'ksift_warp', 'ksift_uniform']


def _fx(name):
    return load_fixture(os.path.join(HERE, 'golden', name + '.pt'))


def _layout(B, H, W, nf=NF):
    out = (torch.zeros(256, dtype=torch.int64)).numpy()
    n = _cabi.lib().og_ksift_workspace_layout(B, H, W, nf, out.ctypes.data, 256)
    assert n > 0, _cabi.lib().og_last_error()
    nO = int(out[0])
    octs = [tuple(int(v) for v in out[1 + 5 * o: 6 + 5 * o]) for o in range(nO)]
    return octs, int(out[n - 1])


def _view(ws, off, shape):
    n = 1
    for s in shape:
        n *= s
    return ws[off: off + 4 * n].view(torch.float32).view(*shape)


def _run_stages(img, nf=NF, dogs=None):
    """pyramid (or the given DoGs written into the workspace) and detect: (ws, octaves, det_lafs, det_resp, count)"""
    B, _, H, W = img.shape
    lib = _cabi.lib()
    octs, nbytes = _layout(B, H, W, nf)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    st = _cabi.stream(torch.device(DEV))
    _cabi.check(lib.og_ksift_pyramid(ptr(img), B, H, W, nf, ptr(ws), nbytes, st), 'og_ksift_pyramid')
    if dogs is not None:
        for (h, w, g, d, r), dog in zip(octs, dogs):
            _view(ws, d, (B, 5, h, w)).copy_(dog.reshape(B, 5, h, w))
    lafs = torch.empty(B, nf, 2, 3, device=DEV)
    resp = torch.empty(B, nf, device=DEV)
    count = torch.empty(B, dtype=torch.int32, device=DEV)
    _cabi.check(lib.og_ksift_detect(B, H, W, nf, ptr(ws), nbytes, ptr(lafs), ptr(resp), ptr(count), st), 'og_ksift_detect')
    torch.cuda.synchronize()
    return ws, octs, lafs, resp, count


def _describe(img, lafs, resp, upright, nf=NF):
    B, _, H, W = img.shape
    N = lafs.shape[1]
    octs, nbytes = _layout(B, H, W, nf)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    n = torch.full((B,), N, dtype=torch.int32, device=DEV)
    lo, sc, de, an = (torch.empty(B, N, 2, 3, device=DEV), torch.empty(B, N, device=DEV), torch.empty(B, N, 128, device=DEV),
                      torch.empty(B, N, device=DEV))
    _cabi.check(_cabi.lib().og_ksift_describe(ptr(img), B, H, W, nf, ptr(ws), nbytes, ptr(lafs.contiguous()), ptr(resp.contiguous()), N,
                                              None, ptr(n), N, int(upright), 1, ptr(lo), ptr(sc), ptr(de), ptr(an),
                                              _cabi.stream(torch.device(DEV))), 'og_ksift_describe')
    torch.cuda.synchronize()
    return lo.cpu(), sc.cpu(), de.cpu(), an.cpu()


# ------------------------------------------------------------------ stage by stage
@pytest.mark.parametrize('name', ['ksift_tiny', 'ksift_odd'])
def test_pyramid_and_dog_within_the_float32_bound(name):
    img = _fx(name)['image']
    p32, _ = KO.scale_pyramid(img)
    p64, _ = KO.scale_pyramid(img.double())
    ws, octs, *_ = _run_stages(img.to(DEV))
    assert len(octs) == len(p32)
    for o, (h, w, g, d, r) in enumerate(octs):
        g_gpu = _view(ws, g, (1, 6, h, w)).cpu().double()
        d_gpu = _view(ws, d, (1, 5, h, w)).cpu().double()
        ref, ref32 = p64[o][:, 0], p32[o][:, 0].double()
        bound = 4 * float((ref32 - ref).abs().max()) + 1e-7
        err = float((g_gpu - ref).abs().max())
        assert err <= bound, (o, err, bound)
        dref = KO.dog_response(p64[o])[:, 0]
        dbound = 4 * float((KO.dog_response(p32[o])[:, 0].double() - dref).abs().max()) + 1e-7
        assert float((d_gpu - dref).abs().max()) <= dbound, o


def _match(la, ra, lb, rb, tol_xy=1e-3, tol_s=1e-3):
    """indices i of (la, ra) with a row of (lb, rb) at the same centre, scale and response (within tolerance)"""
    ka = torch.cat([la[:, :, 2], la[:, 0, 0:1]], 1).double()        # (x, y, scale): voxels of one position differ in scale
    kb = torch.cat([lb[:, :, 2], lb[:, 0, 0:1]], 1).double()
    d = torch.cdist(ka, kb)
    j = d.argmin(1)
    ok = ((la[:, :, 2] - lb[j, :, 2]).abs().max(1).values <= tol_xy) & ((la[:, 0, 0] - lb[j, 0, 0]).abs() <= tol_s * lb[j, 0, 0].abs().clamp(min=1)) & \
         ((ra - rb[j]).abs() <= 1e-4 * rb[j].abs().clamp(min=1))
    return ok


@pytest.mark.parametrize('name', ['ksift_tiny', 'ksift_small', 'ksift_odd'])
def test_detect_on_the_oracle_dog_matches_the_fixture(name):
    fx = _fx(name)
    img = fx['image']
    pyr, _ = KO.scale_pyramid(img)
    dogs = [KO.dog_response(p) for p in pyr]
    _, _, lafs, resp, count = _run_stages(img.to(DEV), dogs=dogs)
    lafs, resp = lafs.cpu()[0], resp.cpu()[0]
    want_l, want_r = fx['det_lafs'][0], fx['det_resp'][0]
    assert int(count[0]) == NF
    # responses agree as sorted lists; the sets agree away from the top-k cut (equal-response classes at the cut may differ)
    assert float((resp - want_r).abs().max()) <= 1e-4, float((resp - want_r).abs().max())
    cut = float(want_r[-1]) + 1e-4
    above = want_r > cut
    ok = _match(want_l[above], want_r[above], lafs, resp)
    assert bool(ok.all()), (int((~ok).sum()), int(above.sum()))


@pytest.mark.parametrize('name', ['ksift_small', 'ksift_odd', 'ksift_pair'])
def test_select_on_the_oracle_detections_is_exact(name):
    fx = _fx(name)
    B, _, H, W = fx['image'].shape
    lafs, resp = fx['det_lafs'].to(DEV).contiguous(), fx['det_resp'].to(DEV).contiguous()
    count = torch.full((B,), NF, dtype=torch.int32, device=DEV)
    nb = _cabi.lib().og_ksift_select_workspace_bytes(B, NF)
    work = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    sel = torch.empty(B, NF, dtype=torch.int32, device=DEV)
    n_sel = torch.empty(B, dtype=torch.int32, device=DEV)
    _cabi.check(_cabi.lib().og_ksift_select(ptr(lafs), ptr(resp), ptr(count), B, H, W, NF, 1, 9, NF, 1, ptr(work), nb, ptr(sel),
                                            ptr(n_sel), _cabi.stream(torch.device(DEV))), 'og_ksift_select')
    N = fx['sel'].shape[1]
    assert n_sel.tolist() == [N] * B
    for b in range(B):
        assert sorted(sel[b, :N].tolist()) == sorted(fx['sel'][b].tolist()), b


@pytest.mark.parametrize('name', ['ksift_small', 'ksift_odd'])
def test_orientations_agree_to_the_bin(name):
    fx = _fx(name)
    img = fx['image']
    _, _, _, ang = _describe(img.to(DEV), fx['det_lafs'].to(DEV), fx['det_resp'].to(DEV), upright=False)
    diff = (ang[0] != fx['angles'][0]).nonzero().flatten()
    if len(diff):          # only where the oracle's two best smoothed bins are within float noise
        p = KO.extract_patches_from_pyramid(img, fx['det_lafs'][:, diff], 19).view(-1, 1, 19, 19)
        _, hist = KO.dominant_orientation(p, want_hist=True)
        top = hist.topk(2, dim=1).values
        assert bool(((top[:, 0] - top[:, 1]) <= 1e-6 * top[:, 0]).all()), (len(diff), (top[:, 0] - top[:, 1]).max())
    assert len(diff) <= NF // 100


@pytest.mark.parametrize('name', ['ksift_small', 'ksift_odd', 'ksift_warp'])
def test_descriptors_on_the_oracle_lafs(name):
    fx = _fx(name)
    lafs, resp, desc = fx['lafs'], fx['responses'], fx['descriptors'].float()
    lo, sc, de, _ = _describe(fx['image'].to(DEV), lafs.to(DEV), resp.to(DEV), upright=True)
    assert torch.equal(lo, lafs) and torch.equal(sc, resp)
    cos = torch.nn.functional.cosine_similarity(de[0], desc[0], dim=1)
    print(f'{name}: descriptor cosine min {float(cos.min()):.6f} mean {float(cos.mean()):.6f}')
    assert float(cos.min()) >= 0.999


# ------------------------------------------------------------------ end to end
# The agreement measured on an H100 (DESIGN.md): the GPU pyramid's float32 rounding differs from the oracle's, which moves the
# decisions that sit at a threshold (|offset| > 0.7, the top-k cut, nms2d between near-equal scores).  sift_tiny keeps only 9
# keypoints, so one such decision is 11 %.
MIN_AGREEMENT = {'ksift_tiny': 0.66, 'ksift_small': 0.999, 'ksift_odd': 0.998, 'ksift_warp': 0.997}


def _agreement(lafs, desc, want_l, want_d):
    """precision, recall and descriptor cosines of lafs [N,2,3] against want_l [M,2,3]: a hit is within 0.05 px, 0.1 % scale and
    0.01 rad of a reference keypoint"""
    cen = torch.cdist(lafs[:, :, 2].double(), want_l[:, :, 2].double())
    j = cen.argmin(1)
    sa, sb = KO.get_laf_scale(lafs[None])[0, :, 0, 0], KO.get_laf_scale(want_l[None])[0, :, 0, 0]
    aa = torch.atan2(lafs[:, 0, 1], lafs[:, 0, 0])
    ab = torch.atan2(want_l[:, 0, 1], want_l[:, 0, 0])
    dang = torch.remainder(aa - ab[j] + torch.pi, 2 * torch.pi) - torch.pi
    hit = (cen.min(1).values <= 0.05) & ((sa - sb[j]).abs() <= 1e-3 * sb[j]) & (dang.abs() <= 0.01)
    cos = torch.nn.functional.cosine_similarity(desc[hit], want_d[j[hit]], dim=1)
    return float(hit.float().mean()), len(set(j[hit].tolist())) / len(want_l), cos


@pytest.mark.parametrize('name', CASES)
def test_end_to_end_against_the_reference(name):
    fx = _fx(name)
    sift = SIFT(max_keypoints=NF, nms_diameter=9, rootsift=True)
    lafs, resp, desc = [t.cpu() for t in sift(fx['image'].to(DEV))]
    want_l, want_r, want_d = fx['lafs'][0], fx['responses'][0], fx['descriptors'][0].float()
    if name == 'ksift_uniform':
        assert lafs.shape == (1, 0, 2, 3) and want_r.numel() == 0
        return
    precision, recall, cos = _agreement(lafs[0], desc[0], want_l, want_d)
    print(f'{name}: N {lafs.shape[1]} / {want_r.numel()}, precision {precision:.4f}, recall {recall:.4f}, '
          f'cosine min {float(cos.min()):.5f} mean {float(cos.mean()):.6f}')
    assert precision >= MIN_AGREEMENT[name] and recall >= MIN_AGREEMENT[name]
    assert abs(lafs.shape[1] - want_r.numel()) <= 1
    assert float(cos.min()) >= 0.999


def test_forward_on_a_pair_is_min_stacked():
    fx = _fx('ksift_pair')
    img = fx['image'].to(DEV)
    sift = SIFT(max_keypoints=NF)
    lafs, resp, desc = sift(img)
    batch = sift.extract_batch(img)
    n = min(t[0].shape[1] for t in batch)
    assert lafs.shape[1] == n and abs(n - fx['lafs'].shape[1]) <= 1
    for b in range(2):
        for x, y in zip((lafs, resp, desc), batch[b]):
            assert torch.equal(x[b], y[0, :n])                  # topk(n) of a list already in response order: its first n
        precision, recall, _ = _agreement(lafs[b].cpu(), desc[b].cpu(), fx['lafs'][b], fx['descriptors'][b].float())
        assert precision >= 0.997 and recall >= 0.997, (b, precision, recall)


def test_batch_padded_repeat_and_the_non_extremum_fill():
    imgs = torch.cat([_fx('ksift_small')['image'], _fx('ksift_warp')['image']]).to(DEV)
    sift = SIFT(max_keypoints=NF)
    singles = [sift(imgs[b:b + 1]) for b in range(2)]
    batch = sift.extract_batch(imgs)
    for s, t in zip(singles, batch):
        for x, y in zip(s, t):
            assert torch.equal(x, y)
    for K in (NF, 500):
        lafs, resp, desc, num, over = sift.extract_padded(imgs, K)
        for b in range(2):
            k = batch[b][0].shape[1]
            assert int(num[b]) == min(k, K) and int(over[b]) == int(k > K)
            for x, y in zip((lafs, resp, desc), batch[b]):
                assert torch.equal(x[b, :min(k, K)], y[0, :min(k, K)])
                assert not x[b, min(k, K):].any()
    again = sift.extract_padded(imgs, NF)
    for x, y in zip(sift.extract_padded(imgs, NF), again):
        assert torch.equal(x, y)
    # the tiny image: its octaves have fewer extrema than NF, so non-extrema (|DoG|, no bonus) fill the per-octave top-k
    img = _fx('ksift_tiny')['image'].to(DEV)
    _, _, _, resp, count = _run_stages(img)
    assert int(count[0]) == NF and int((resp[0] < 5).sum()) > 0
    with pytest.raises(RuntimeError):
        sift(img.cpu())


def test_image_pair_matcher_and_train_step_replay_equal_eager():
    from test_image_matching import _matcher_parts, _pair_images
    from test_image_training import CONFIG, OUT_KEYS, _batch, _same, _state, _trainer
    _, sg, mc = _matcher_parts('sift')
    fe = SIFT(max_keypoints=300)
    graphed = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
    eager = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
    for i in range(2):
        i0, i1 = _pair_images('sift', 2, 30 + i)
        got, want = graphed(i0, i1), eager(i0, i1)
        for k in ImagePairMatcher._OUT_KEYS:
            assert torch.equal(got[k], want[k]), (i, k)
    (m_g, o_g), (m_e, o_e) = _trainer(128), _trainer(128)
    step_g = ImagePairTrainStep(fe, m_g, CONFIG, optimizer=o_g)
    step_e = ImagePairTrainStep(fe, m_e, CONFIG, optimizer=o_e, use_cuda_graph=False)
    for j in range(2):
        batch = _batch('sift', 2, 60 + j, 'perspective')
        got, ge = step_g(batch), step_e(batch)
        torch.cuda.synchronize()
        for k in OUT_KEYS:
            assert torch.equal(got[k], ge[k]), (j, k)
        _same(_state(m_g, o_g), _state(m_e, o_e))
