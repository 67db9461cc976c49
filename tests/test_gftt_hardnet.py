"""GFTT / AffNet / HardNet front-end (openglue_b200.GFTTAffNetHardNet, csrc/kornia_gftt.cuh) on the H100: stages on the oracle's
own inputs (oracle/kornia_gftt_oracle.py, a restatement of kornia 0.6.3), the patch CNNs against float64 convolutions, end to end
against fixtures minted by the unmodified reference (oracle/gen_golden_gftt_hardnet.py: tests/golden/gftt_*.pt), and the
front-end's batch, padded and image-pair forms."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_gftt_hardnet import load_fixture  # noqa: E402
from openglue_b200 import GFTTAffNetHardNet, ImagePairMatcher, ImagePairTrainStep, _cabi  # noqa: E402
from openglue_b200 import _patch_cnn as PC  # noqa: E402
from openglue_b200 import gftt_hardnet as GH  # noqa: E402
from openglue_b200._cabi import ptr  # noqa: E402
from openglue_b200._ops import _Ops  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NF = 1024


def _fx(name):
    return load_fixture(os.path.join(HERE, 'golden', name + '.pt'))


def _model(nf=NF, **kw):
    w = {'affnet': KG.synthetic_affnet_state_dict(), 'hardnet': KG.synthetic_hardnet_state_dict()}
    return GFTTAffNetHardNet(max_keypoints=nf, weights=w, **kw)


def _layout(B, H, W, nf=NF):
    out = torch.zeros(256, dtype=torch.int64).numpy()
    n = _cabi.lib().og_kgftt_workspace_layout(B, H, W, nf, out.ctypes.data, 256)
    assert n > 0, _cabi.lib().og_last_error()
    return [tuple(int(v) for v in out[1 + 5 * o: 6 + 5 * o]) for o in range(int(out[0]))]


def _view(ws, off, shape):
    n = 1
    for s in shape:
        n *= s
    return ws[off: off + 4 * n].view(torch.float32).view(*shape)


def _pyramid(m, img):
    B, _, H, W = img.shape
    ws, _ = m._workspace(img.device, B, H, W)
    _cabi.check(_cabi.lib().og_kgftt_pyramid(ptr(img), B, H, W, m.max_keypoints, ptr(ws), ws.numel(), _cabi.stream(img.device)), 'pyramid')
    return ws


# ------------------------------------------------------------------ stage by stage
def _pyramid_input(name):
    """a fixture image or batch, or a synthetic two-image batch (``synthetic_HxW``) whose octave widths are not multiples of the
    16-pixel GFTT tile and whose smallest octave sits near ScalePyramid's min_size (32)"""
    if name.startswith('synthetic_'):
        H, W = (int(v) for v in name.split('_')[1].split('x'))
        g = torch.Generator().manual_seed(H * W)
        return F.avg_pool2d(torch.rand(2, 1, H + 2, W + 2, generator=g), 3, stride=1)   # two different textures in [0, 1]
    return _fx(name)['image']


@pytest.mark.parametrize('name', ['gftt_small', 'gftt_odd', 'gftt_pair', 'synthetic_65x97', 'synthetic_33x200'])
def test_pyramid_and_gftt_responses_within_the_float32_bound(name):
    img = _pyramid_input(name)
    B = img.shape[0]
    m = _model()
    ws = _pyramid(m, img.to(DEV))
    torch.cuda.synchronize()
    p32, s32 = KO.scale_pyramid(img, double_image=False)
    p64, s64 = KO.scale_pyramid(img.double(), double_image=False)
    octs = _layout(B, *img.shape[-2:])
    assert len(octs) == len(p32)
    for o, (h, w, g, v, _) in enumerate(octs):
        ref = p64[o][:, 0]
        bound = 4 * float((p32[o][:, 0].double() - ref).abs().max()) + 1e-7
        assert float((_view(ws, g, (B, 6, h, w)).cpu().double() - ref).abs().max()) <= bound, o
        # the response of all six levels of every image (the detector reads the first five): planes [B][6] in image-major order
        r64 = KG.gftt_response(p64[o][:, 0].reshape(B * 6, 1, h, w), s64[o].reshape(-1))
        r32 = KG.gftt_response(p32[o][:, 0].reshape(B * 6, 1, h, w), s32[o].reshape(-1)).double()
        got = _view(ws, v, (B * 6, 1, h, w)).cpu().double()
        rb = 4 * float((r32 - r64).abs().max()) + 1e-9
        err = float((got - r64).abs().max())
        print(f'{name} octave {o}: level err {err:.3e}, float32 oracle {rb / 4:.3e}')
        assert err <= rb, (o, err, rb)


def test_detect_on_the_oracle_responses_matches_the_fixture():
    fx = _fx('gftt_odd')
    img = fx['image']
    m = _model()
    ws = _pyramid(m, img.to(DEV))
    pyr, sig = KO.scale_pyramid(img, double_image=False)
    for (h, w, g, v, _), p, s in zip(_layout(1, *img.shape[-2:]), pyr, sig):
        _view(ws, v, (6, 1, h, w)).copy_(KG.gftt_response(p[0].permute(1, 0, 2, 3), s.view(-1)))
    lafs, resp = torch.empty(1, NF, 2, 3, device=DEV), torch.empty(1, NF, device=DEV)
    count = torch.empty(1, dtype=torch.int32, device=DEV)
    H, W = img.shape[-2:]
    _cabi.check(_cabi.lib().og_kgftt_detect(1, H, W, NF, ptr(ws), ws.numel(), ptr(lafs), ptr(resp), ptr(count), _cabi.stream(torch.device(DEV))),
                'detect')
    lafs, resp = lafs.cpu()[0], resp.cpu()[0]
    want_l, want_r = fx['det_lafs'][0], fx['det_resp'][0]
    assert int(count[0]) == NF
    assert float((resp - want_r).abs().max()) <= 1e-6 * float(want_r.abs().max())
    # exact away from ties: rows whose response is unique in the fixture carry the same LAF
    uniq = (want_r[:, None] != want_r[None, :]).sum(1) == NF - 1
    d = (lafs[uniq] - want_l[uniq]).abs().max()
    assert float(d) <= 1e-4, float(d)


def _describe(m, img, lafs, resp, upright):
    """og_kgftt_* describe stages on the given detector rows (no selection): (lafs, scores, descriptors)"""
    B, _, H, W = img.shape
    N = lafs.shape[1]
    ws = _pyramid(m, img)
    m.upright = upright
    n = torch.full((B,), N, dtype=torch.int32, device=DEV)
    out = m._describe(img, ws, lafs.contiguous(), resp.contiguous(), None, n, N)
    torch.cuda.synchronize()
    return [t.cpu() for t in out]


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_frames_orientations_and_descriptors_on_the_oracle_lafs(precision):
    fx = _fx('gftt_small')
    img = fx['image']
    m = _model(precision=precision)
    det_l, det_r = fx['det_lafs'][:, :256], fx['det_resp'][:, :256]
    # upright: AffNet's frames alone
    lo, sc, _ = _describe(m, img.to(DEV), det_l.to(DEV), det_r.to(DEV), upright=True)
    want = fx['aff_lafs'][:, :256]
    aff64, hard64 = KG.features_in(torch.float64)
    with torch.no_grad():
        want64 = KG.affnet_shape(det_l.double(), img.double(), aff64)
    bound = 8 * float((want.double() - want64).abs().max()) + 1e-6
    err = float((lo.double() - want64).abs().max())
    print(f'{precision}: AffNet LAF err {err:.3e}, float32 oracle {bound / 8:.3e}')
    assert err <= bound and torch.equal(sc, det_r)
    # with the orienter: the fixture's angles, up to bins the oracle's two best smoothed values make a near tie
    lo_up = lo
    lo, _, de = _describe(m, img.to(DEV), det_l.to(DEV), det_r.to(DEV), upright=False)
    ang = torch.atan2(lo[0, :, 0, 1], lo[0, :, 0, 0])

    def dangle(lafs):
        a = torch.atan2(lafs[0, :, 0, 1], lafs[0, :, 0, 0])
        return (torch.remainder(ang - a + torch.pi, 2 * torch.pi) - torch.pi).abs()
    dang = dangle(KO.laf_orienter(want, img, 19))
    print(f'{precision}: {int((dang > 1e-3).sum())} of 256 orientations differ from the fixture\'s')
    assert int((dang > 1e-3).sum()) <= 256 // 50
    # on the kernel's own AffNet frames (the orienter's input, bit for bit), every angle that differs from the oracle's must be a
    # near tie of the oracle's two best smoothed bins (kornia SIFT's rule, test_kornia_sift.py)
    diff = (dangle(KO.laf_orienter(lo_up, img, 19)) > 1e-3).nonzero().flatten()
    print(f'{precision}: {len(diff)} of 256 orientations differ from the oracle\'s on the same frames')
    if len(diff):
        p = KO.extract_patches_from_pyramid(img, lo_up[:, diff], 19).view(-1, 1, 19, 19)
        _, hist = KO.dominant_orientation(p, want_hist=True)
        top = hist.topk(2, dim=1).values
        assert bool(((top[:, 0] - top[:, 1]) <= 1e-6 * top[:, 0]).all()), (len(diff), (top[:, 0] - top[:, 1]).max())
    assert len(diff) <= 256 // 50
    ok = dang <= 1e-3
    with torch.no_grad():
        d64 = KG.laf_descriptors(img.double(), lo.double(), hard64)[0]
    cos = F.cosine_similarity(de[0].double(), d64, dim=1)
    print(f'{precision}: descriptor cosine against float64 HardNet on the kernels\' LAFs: min {float(cos.min()):.7f}')
    assert float(cos.min()) >= 0.9999
    assert bool(ok.any())


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_cnns_against_float64_convolutions(precision):
    m = _model(precision=precision)
    dev = torch.device(DEV)
    ops = _Ops(dev, _cabi.OG_PREC_FP32 if precision == 'fp32' else _cabi.OG_PREC_TF32X3)
    rows = 200 if GH.CHUNK >= 200 else GH.CHUNK
    x = KG.normalize_input(torch.rand(rows, 1, 32, 32, generator=torch.Generator().manual_seed(3)))
    patches, col, a0, a1, _ = PC.cnn_buffers(m._ws, dev)
    patches[:rows * 1024].copy_(x.flatten())
    aff64, hard64 = KG.features_in(torch.float64)
    for name, net, convs, nout in (('affnet', aff64, GH.AFFNET_CONVS, 3), ('hardnet', hard64, GH.HARDNET_CONVS, 128)):
        out = torch.empty(rows, nout, device=dev)
        PC.run_cnn(ops, m._weights_on(dev)[name], patches, rows, convs, col, (a0, a1), out)
        torch.cuda.synchronize()
        with torch.no_grad():
            want = net[:19](x.double())
            want = net[19:21](want) if name == 'hardnet' else net[19](want)
        want = want.flatten(1)
        err = float((out.cpu().double() - want).abs().max()) / float(want.abs().max())
        print(f'{precision} {name}: max relative err {err:.3e}')
        assert err <= 2e-5, (name, err)


# ------------------------------------------------------------------ end to end
# The agreement measured on an H100 80GB HBM3 at 700 W (DESIGN.md, row f9): precision / recall 0.9975 / 0.9975 on gftt_small,
# 1 / 1 on gftt_odd, 0.9948 / 0.9923 on gftt_warp, the one keypoint of gftt_tiny; descriptor cosine >= 0.99999.  The rows that
# differ sit at a decision the float32 pyramid rounds differently (the top-k cut, nms2d between near-equal scores).
MIN_AGREEMENT = {'gftt_tiny': 1.0, 'gftt_small': 0.997, 'gftt_odd': 0.999, 'gftt_warp': 0.992}


def _agreement(lafs, desc, want_l, want_d):
    """precision, recall, the largest LAF difference of the hits and their descriptor cosines: a hit is within 0.05 px of a
    reference keypoint with its 2x2 part within 1 % of the reference's scale"""
    cen = torch.cdist(lafs[:, :, 2].double(), want_l[:, :, 2].double())
    j = cen.argmin(1)
    s = KO.get_laf_scale(want_l[None])[0, :, 0, 0].double()
    dshape = (lafs[:, :, :2].double() - want_l[j, :, :2].double()).abs().flatten(1).max(1).values
    hit = (cen.min(1).values <= 0.05) & (dshape <= 1e-2 * s[j])
    cos = F.cosine_similarity(desc[hit], want_d[j[hit]], dim=1)
    return float(hit.float().mean()), len(set(j[hit].tolist())) / len(want_l), float(dshape[hit].max()), cos


@pytest.mark.parametrize('name', ['gftt_tiny', 'gftt_small', 'gftt_odd', 'gftt_warp', 'gftt_uniform'])
def test_end_to_end_against_the_reference(name):
    fx = _fx(name)
    lafs, resp, desc = [t.cpu() for t in _model()(fx['image'].to(DEV))]
    want_l, want_r, want_d = fx['lafs'][0], fx['responses'][0], fx['descriptors'][0].float()
    if name == 'gftt_uniform':
        assert lafs.shape == (1, 0, 2, 3) and want_r.numel() == 0
        return
    precision, recall, dlaf, cos = _agreement(lafs[0], desc[0], want_l, want_d)
    print(f'{name}: N {lafs.shape[1]} / {want_r.numel()}, precision {precision:.4f}, recall {recall:.4f}, LAF diff {dlaf:.2e}, '
          f'cosine min {float(cos.min()):.5f} mean {float(cos.mean()):.6f}')
    assert precision >= MIN_AGREEMENT[name] and recall >= MIN_AGREEMENT[name]
    assert float(cos.min()) >= 0.9999


def test_forward_on_a_pair_is_min_stacked_and_batch_padded_identities():
    fx = _fx('gftt_pair')
    img = fx['image'].to(DEV)
    m = _model()
    lafs, resp, desc = m(img)
    batch = m.extract_batch(img)
    n = min(t[0].shape[1] for t in batch)
    assert lafs.shape[1] == n
    for b in range(2):
        for x, y in zip((lafs, resp, desc), batch[b]):
            assert torch.equal(x[b], y[0, :n])
        single = m(img[b:b + 1])
        for x, y in zip(single, batch[b]):
            assert torch.equal(x, y)
    for K in (NF, 200):
        out = m.extract_padded(img, K)
        num, over = out[3], out[4]
        for b in range(2):
            k = batch[b][0].shape[1]
            assert int(num[b]) == min(k, K) and int(over[b]) == int(k > K)
            for x, y in zip(out[:3], batch[b]):
                assert torch.equal(x[b, :min(k, K)], y[0, :min(k, K)])
                assert not x[b, min(k, K):].any()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        m.extract_padded(img, NF)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    with pytest.raises(RuntimeError):
        m(img.cpu())


def test_image_pair_matcher_and_train_step_replay_equal_eager_and_recapture_on_weight_change():
    from test_image_matching import _matcher_parts, _pair_images
    from test_image_training import CONFIG, OUT_KEYS, _batch, _same, _state, _trainer
    _, sg, mc = _matcher_parts('sift')
    fe = _model(300).to(DEV)
    graphed = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
    eager = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
    for i in range(3):
        if i == 2:                                           # a weight change: the graph is captured again
            with torch.no_grad():
                fe.descriptor.descriptor.features[15].weight.mul_(0.5)
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
