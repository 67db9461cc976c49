"""The DoG / AffNet / OriNet / HardNet front-end (openglue_b200.DoGOpenCVAffNetHardNet) on the GPU: each describe stage on the
oracle's or the fixture's inputs, end to end against the reference's fixtures (tests/golden/dogaff_*.pt, minted by
oracle/gen_golden_dog_affnet_hardnet.py), the batch and padded identities, graph replay, and the cached-feature path."""
from __future__ import annotations

import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import dog_affnet_oracle as KD  # noqa: E402
from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_dog_affnet_hardnet import load_fixture  # noqa: E402
from openglue_b200 import DoGOpenCVAffNetHardNet, ImagePairMatcher, ImagePairTrainStep, _cabi  # noqa: E402
from openglue_b200 import dog_affnet_hardnet as DA  # noqa: E402
from openglue_b200._cabi import ptr  # noqa: E402
from openglue_b200._ops import _Ops  # noqa: E402
from openglue_b200._patch_cnn import cnn_buffers, run_cnn  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NF = 2048
CASES = ['dogaff_tiny', 'dogaff_small', 'dogaff_odd', 'dogaff_warp']
# end-to-end agreement with the reference's fixtures, as measured on an H100 (see DESIGN.md, row f10)
MIN_PRECISION_RECALL = 1.0
MIN_COSINE = 0.99999


def _fx(name):
    return load_fixture(os.path.join(HERE, 'golden', name + '.pt'))


def _weights():
    return dict(affnet=KG.synthetic_affnet_state_dict(), orinet=KD.synthetic_orinet_state_dict(), hardnet=KG.synthetic_hardnet_state_dict())


def _model(nf=NF, **kw):
    return DoGOpenCVAffNetHardNet(max_keypoints=nf, weights=_weights(), **kw)


class _Stages:
    """The describe stages of one fixture image fed the fixture's keypoints, every row in one chunk"""

    def __init__(self, m, fx):
        self.m, self.img = m, fx['image'].to(DEV)
        self.kp = fx['kp'].to(DEV).contiguous()
        self.n = self.kp.shape[1]
        _, _, self.H, self.W = self.img.shape
        self.ws = m._workspace(self.img.device, 1, self.H, self.W)
        self.args = (ptr(self.img), 1, self.H, self.W, ptr(self.ws), self.ws.numel())
        self.st = _cabi.stream(self.img.device)
        self.nn = torch.tensor([self.n], dtype=torch.int32, device=DEV)
        _cabi.check(_cabi.lib().og_dogaff_pyramid(*self.args, self.st), 'pyramid')

    def affnet(self):
        lafs = torch.empty(1, self.n, 2, 3, device=DEV)
        scores = torch.empty(1, self.n, device=DEV)
        patches = torch.empty(self.n, 32, 32, device=DEV)
        sel = torch.arange(self.n, dtype=torch.int32, device=DEV)
        _cabi.check(_cabi.lib().og_dogaff_affnet_patches(*self.args, ptr(self.kp), self.n, ptr(sel), ptr(self.nn), self.n, 0, self.n, ptr(lafs),
                                                         ptr(scores), ptr(patches), self.st), 'affnet_patches')
        return lafs, scores, patches

    def frames(self, lafs_in, xy):
        lafs = lafs_in.to(DEV).float().clone().contiguous()
        patches = torch.empty(self.n, 32, 32, device=DEV)
        _cabi.check(_cabi.lib().og_dogaff_frames(*self.args, ptr(self.nn), self.n, 0, self.n, ptr(xy.float().contiguous()), ptr(lafs), ptr(patches),
                                                 self.st), 'frames')
        return lafs, patches

    def orinet(self, lafs_in, patches, precision):
        m = self.m
        ops = _Ops(self.img.device, _cabi.OG_PREC_FP32 if precision == 'fp32' else _cabi.OG_PREC_TF32X3)
        wts = m._weights_on(self.img.device)
        lafs = lafs_in.to(DEV).float().clone().contiguous()
        angle = torch.empty(1, self.n, device=DEV)
        out = torch.empty(self.n, 32, 32, device=DEV)
        _, col, a0, a1, _ = cnn_buffers(m._ws, self.img.device)
        for r0 in range(0, self.n, DA.CHUNK):
            r = min(DA.CHUNK, self.n - r0)
            act = run_cnn(ops, wts['orinet'], patches[r0:r0 + r].contiguous(), r, DA.ORINET_CONVS, col, (a0, a1), None)
            w, b = wts['orinet'][-1]
            _cabi.check(_cabi.lib().og_dogaff_orinet_head(*self.args, ptr(self.nn), self.n, r0, r, ptr(act), ptr(w), ptr(b), ptr(lafs), ptr(angle),
                                                          ptr(out[r0:r0 + r]), self.st), 'orinet_head')
        return lafs, angle, out


def _ulps(a, b):
    """max |a - b| in units of b's float32 ulp"""
    a, b = a.float(), b.float()
    ulp = torch.nextafter(b.abs(), torch.tensor(float('inf'))) - b.abs()
    return float(((a - b).abs() / ulp).max())


# ------------------------------------------------------------------ stage by stage
@pytest.mark.parametrize('name', ['dogaff_small', 'dogaff_odd'])
def test_laf_conversion_and_affnet_patches(name):
    fx = _fx(name)
    s = _Stages(_model(), fx)
    lafs, scores, patches = s.affnet()
    torch.cuda.synchronize()
    # 2 ulp, not 1: the kernel's cos and sin are correctly rounded, torch's float32 ones on the CPU only within 1 ulp, and the
    # product with the scale rounds once more.  Measured: 2 ulp on both images.
    assert _ulps(lafs.cpu(), fx['moons_lafs']) <= 2.0
    assert torch.equal(scores.cpu(), fx['scores'])
    want = KG.affnet_patches(fx['image'].double(), fx['moons_lafs'].double()).view(-1, 32, 32)
    assert float((patches.cpu().double() - want).abs().max()) < 2e-3


@pytest.mark.parametrize('name', ['dogaff_small', 'dogaff_odd'])
def test_affnet_frames_and_orinet_patches(name):
    fx = _fx(name)
    s = _Stages(_model(), fx)
    aff64 = KG.features_in(torch.float64)[0]
    moons = fx['moons_lafs']
    with torch.no_grad():
        xy64 = aff64[:-2](KG.affnet_patches(fx['image'].double(), moons.double())).view(-1, 3)   # before tanh
    want = KG.affnet_frames(torch.tanh(xy64), moons.double())
    ref32 = KG.affnet_frames(torch.tanh(xy64.float()), moons)
    bound = 8 * float((ref32.double() - want).abs().max()) + 1e-5
    lafs, patches = s.frames(moons, xy64.float().to(DEV))
    torch.cuda.synchronize()
    assert float((lafs.cpu().double() - want).abs().max()) <= bound
    pw = KD.orinet_patches(fx['image'].double(), lafs.cpu().double()).view(-1, 32, 32)
    assert float((patches.cpu().double() - pw).abs().max()) < 2e-3


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name', ['dogaff_small', 'dogaff_odd'])
def test_orinet_angles_final_lafs_and_hardnet_descriptors(name, precision):
    fx = _fx(name)
    m = _model(precision=precision)
    s = _Stages(m, fx)
    aff = fx['aff_lafs']
    p32 = KD.orinet_patches(fx['image'], aff).view(-1, 32, 32)
    lafs, angle, hp = s.orinet(aff, p32.to(DEV), precision)
    torch.cuda.synchronize()
    with torch.no_grad():
        xy = KD.orinet_in(torch.float64)(p32.double().view(-1, 1, 32, 32)).view(-1, 2)     # p32 is already standardised
        a64 = torch.atan2(xy[:, 0] + 1e-8, xy[:, 1] + 1e-8).view(1, -1)
    err = float((angle.cpu().double() - a64).abs().max())
    assert err < 1e-4, err
    want = KO.set_laf_orientation(aff.double(), KO.rad2deg(a64) + KO.get_laf_orientation(aff.double()).view_as(a64))
    assert float((lafs.cpu().double() - want).abs().max() / want.abs().max()) < 1e-5
    # HardNet on the head kernel's patches, against float64 on the same final LAFs
    ops = _Ops(s.img.device, _cabi.OG_PREC_FP32 if precision == 'fp32' else _cabi.OG_PREC_TF32X3)
    desc = torch.empty(s.n, 128, device=DEV)
    _, col, a0, a1, _ = cnn_buffers({}, s.img.device)
    for r0 in range(0, s.n, DA.CHUNK):
        r = min(DA.CHUNK, s.n - r0)
        run_cnn(ops, m._weights_on(s.img.device)['hardnet'], hp[r0:r0 + r].contiguous(), r, DA.HARDNET_CONVS, col, (a0, a1), desc[r0:r0 + r])
    _cabi.check(_cabi.lib().og_kgftt_desc_finish(ptr(desc), 1, s.n, ptr(s.nn), s.st), 'desc_finish')
    torch.cuda.synchronize()
    with torch.no_grad():
        d64 = KG.laf_descriptors(fx['image'].double(), lafs.cpu().double(), KG.features_in(torch.float64)[1])[0]
    assert float(F.cosine_similarity(desc.cpu().double(), d64, dim=-1).min()) >= 0.99999


# ------------------------------------------------------------------ end to end
def _match(kp, ref):
    """each row of kp [N, 5] against ref [M, 5] (x, y, size, angle, response), to the OpenCV SIFT tests' tolerances (the SIFT
    kernels agree with cv2 to these, not bit for bit): the index of the same keypoint, -2 for another member of its class (cv2
    repeats a keypoint at one place with its secondary orientations, and the reference's radius NMS keeps numpy argsort's
    unspecified pick among equal responses, ours the first in cv2's order), -1 for none"""
    kp, ref = kp.double(), ref.double()
    same = ((torch.cdist(kp[:, :2], ref[:, :2]) <= 0.01) & ((kp[:, None, 2] - ref[None, :, 2]).abs() <= 1e-4 * ref[None, :, 2])
            & ((kp[:, None, 4] - ref[None, :, 4]).abs() <= 1e-3 * ref[None, :, 4]))
    da = (kp[:, None, 3] - ref[None, :, 3]).abs() % 360
    exact = same & (torch.minimum(da, 360 - da) <= 0.05)
    out = torch.full((kp.shape[0],), -1, dtype=torch.int64)
    out[same.any(dim=1)] = -2
    has = exact.any(dim=1)
    out[has] = exact.float().argmax(dim=1)[has]
    return out


@pytest.mark.parametrize('name', CASES + ['dogaff_uniform'])
def test_forward_against_the_reference(name):
    fx = _fx(name)
    m = _model().to(DEV)
    img = fx['image'].to(DEV)
    lafs, scores, desc = (t.cpu() for t in m(img))
    if fx['kp'].shape[1] == 0:
        assert lafs.shape == (1, 0, 2, 3) and desc.shape == (1, 0, 128)
        return
    assert bool((scores[0, 1:] <= scores[0, :-1]).all())            # descending response
    _, kp, _, _, sel, n_sel = m._sift._detect_select(m._image(img), 1)
    kp = kp[0, sel[0, :int(n_sel[0])].long()].cpu()                  # the cv2 keypoint of every output row
    assert kp.shape[0] == scores.shape[1] and torch.equal(kp[:, 4], scores[0])
    ours, theirs = _match(kp, fx['kp'][0]), _match(fx['kp'][0], kp)
    precision, recall = float((ours != -1).double().mean()), float((theirs != -1).double().mean())
    j = torch.nonzero(ours >= 0)[:, 0]
    i = ours[j]
    cos = F.cosine_similarity(desc[0, j].double(), fx['descriptors'][0, i].double(), dim=-1)
    dl = float((lafs[0, j].double() - fx['lafs'][0, i].double()).abs().max())
    print(f'{name}: {scores.shape[1]} / {fx["kp"].shape[1]} keypoints, precision {precision:.4f}, recall {recall:.4f} '
          f'({int((ours == -2).sum())} as another member of their class); {len(j)} identical keypoints: descriptor cosine min '
          f'{float(cos.min()):.7f}, max LAF difference {dl:.2e} px')
    assert precision >= MIN_PRECISION_RECALL and recall >= MIN_PRECISION_RECALL
    assert float(cos.min()) >= MIN_COSINE and dl < 1e-3


def test_batch_and_padded_identities():
    a, b = _fx('dogaff_small'), _fx('dogaff_warp')
    img = torch.cat([a['image'], b['image']]).to(DEV)
    m = _model().to(DEV)
    batch = m.extract_batch(img)
    for i in range(2):
        single = m(img[i:i + 1])
        for x, y in zip(batch[i], single):
            assert torch.equal(x, y)
    for K in (NF, 600):
        out = m.extract_padded(img, K)
        num, over = out[3].cpu(), out[4].cpu()
        for i in range(2):
            k = batch[i][0].shape[1]
            assert int(num[i]) == min(k, K) and int(over[i]) == int(k > K)
            for x, y in zip(out[:3], batch[i]):
                assert torch.equal(x[i, :min(k, K)], y[0, :min(k, K)])
                assert not x[i, min(k, K):].any()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        m.extract_padded(img, NF)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    # a capacity before NMS too small for the image: extract_batch raises, extract_padded flags it
    small = _model(capacity=256).to(DEV)
    with pytest.raises(RuntimeError):
        small.extract_batch(img)
    assert small.extract_padded(img, 300)[4].cpu().tolist() == [1, 1]


def test_image_pair_matcher_and_train_step_replay_equal_eager_and_recapture_on_weight_change():
    from test_image_matching import _matcher_parts, _pair_images
    from test_image_training import CONFIG, OUT_KEYS, _batch, _same, _state, _trainer
    _, sg, mc = _matcher_parts('sift')
    fe = _model(300).to(DEV)
    graphed = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
    eager = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
    for i in range(3):
        if i == 2:                                           # an OriNet weight change: the graph is captured again
            with torch.no_grad():
                fe.orinet.angle_detector.features[15].weight.mul_(0.5)
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


def test_cached_features_path(tmp_path):
    """extract_features' outputs through save_features_npz -> FeatureStore -> collate_features, the path the reference intends
    these features for (extract_features.py -> train_cached.py)"""
    from oracle import collate_oracle as CO
    from oracle.gen_golden_collate import synthetic_items
    from openglue_b200.feature_cache import FeatureStore, collate_features, save_features_npz
    m = _model().to(DEV)
    names = ['dogaff_small', 'dogaff_warp']                 # one image size: the batch stacks the pairs' depth maps
    outs = {}
    for n in names:
        fx = _fx(n)
        lafs, scores, desc = (t[0].cpu() for t in m(fx['image'].to(DEV)))
        outs[n] = (lafs, scores, desc)
        H, W = fx['image'].shape[-2:]
        save_features_npz(str(tmp_path), n, lafs.numpy(), scores.numpy(), desc.numpy(), [W, H])
    store = FeatureStore(str(tmp_path), pin=False)
    assert store.names() == sorted(names)
    for n, (lafs, scores, desc) in outs.items():
        it = store[n]
        assert torch.equal(it['lafs'], lafs) and torch.equal(it['scores'], scores) and torch.equal(it['descriptors'], desc)
    items = synthetic_items((2, 512, 128, [(100, 100), (100, 100)], False, 1))
    g = torch.Generator().manual_seed(5)
    for b, pair in enumerate([names, names[::-1]]):
        for i, n in enumerate(pair):
            it = store[n]
            H, W = _fx(n)['image'].shape[-2:]
            items[b].update({f'lafs{i}': it['lafs'], f'scores{i}': it['scores'], f'descriptors{i}': it['descriptors'],
                             f'image{i}_size': it['size']})
            items[b]['transformation'][f'depth{i}'] = torch.rand(H, W, generator=g) * 10
    got = collate_features(items, 512, random=False, device=DEV)
    want = CO.stack_keypoints_batch(items, 512, None)
    torch.cuda.synchronize()
    for k in ('lafs0', 'lafs1', 'scores0', 'scores1', 'descriptors0', 'descriptors1'):
        assert torch.equal(got[k].cpu(), want[k]), k


def test_each_graph_holds_the_detector_workspaces_of_its_image_size():
    """The nested OpenCVSIFT caches the workspaces of two image sizes, ImagePairMatcher keeps four graphs: after three sizes
    the first size's workspaces have left the detector's cache, and its graph, which reads them, must still hold them"""
    from test_image_matching import _matcher_parts, _textures
    _, sg, mc = _matcher_parts('sift')
    fe = _model(300).to(DEV)
    graphed = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
    sizes = [(240, 320), (256, 336), (200, 288)]
    want = {}
    for k, (H, W) in enumerate(sizes):
        img = _textures(2, H, W, 40 + k)
        graphed(img, img.flip(-1).contiguous())
        ws = [v for key, v in fe._sift._ws.items() if key[1:] == (2, H, W)]
        assert len(ws) == 1
        want[(H, W)] = {t.data_ptr() for t in ws[0]}
    torch.cuda.synchronize()
    assert not any(key[1:] == (2,) + sizes[0] for key in fe._sift._ws)          # evicted from the detector's cache
    assert len(graphed._graphs) == len(sizes)
    for key, entry in graphed._graphs.items():
        H, W = key[0][2:]
        held = set()
        for v in entry.held[0]:
            held |= {t.data_ptr() for t in (v if isinstance(v, tuple) else (v,))}
        assert want[(H, W)] <= held, (H, W)
