"""Images to matches without a host synchronisation, on the H100: the front-ends' padded outputs (``OpenCVSIFT.extract_padded``,
``SuperPointNet[Bn].extract_padded``) against their per-image eager outputs, the overflow flags, and ``ImagePairMatcher``
(eager and graph-replayed) against ``OpenGlueMatcher`` run pair by pair."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'oracle'))

from conftest import GOLDEN_DIR  # noqa: E402
from gen_golden_superpoint import synthetic_images, synthetic_superpoint_bn_state_dict, synthetic_superpoint_state_dict  # noqa: E402
from gen_golden_superpoint_padded import CASE as PAD_CASE, NAME as PAD_NAME, padded_inputs  # noqa: E402
from gen_golden_superpoint_post import inputs_sha256, post_inputs  # noqa: E402
from test_superpoint_kernels import _probs_coarse, _same_up_to_ties, nms_threshold_borders, pixel_heat  # noqa: E402
from openglue_b200 import OpenCVSIFT, SuperGlue, SuperPointNet, SuperPointNetBn  # noqa: E402
from openglue_b200.features import ImagePairMatcher, OpenGlueMatcher, compact_matches  # noqa: E402
from openglue_b200.synthetic import default_config, synthetic_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _textures(B, H, W, seed):
    """uint8 [B,1,H,W]: noise, sinusoidal blobs and a calm gradient in turn, so the keypoint counts differ per image"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    out = []
    for b in range(B):
        ph = float(torch.rand(1, generator=g)) * 6.28
        kind = b % 3
        if kind == 0:
            img = torch.rand(H, W, generator=g) * 255
        elif kind == 1:
            img = 127 + 100 * torch.sin(xx / 9.0 + ph) * torch.cos(yy / 13.0)
        else:
            img = 127 + 40 * torch.sin(xx / 40.0 + ph) + torch.rand(H, W, generator=g) * 10
        out.append(img)
    return torch.stack(out)[:, None].round().clamp(0, 255).to(torch.uint8).to(DEV)


def _sift_images(name):
    return torch.from_numpy(np.load(os.path.join(GOLDEN_DIR, name + '.npz'))['image'])[None, None]


def _check_padded(out, singles, K):
    """out: extract_padded's tuple; singles: one (lafs, scores, desc) [1, N_b, ...] per image.  Rows [0, N_b) bit for bit, zeros past."""
    lafs, scores, desc, num, over = out
    assert lafs.shape[1] == K and num.dtype == torch.int32 and over.dtype == torch.int32
    assert over.tolist() == [0] * len(singles)
    assert num.tolist() == [s[0].shape[1] for s in singles]
    for b, s in enumerate(singles):
        n = s[0].shape[1]
        for got, want in zip((lafs, scores, desc), s):
            assert torch.equal(got[b, :n], want[0]), b
            assert (got[b, n:] == 0).all(), b


# --------------------------------------------------------------------------- 1. SIFT: extract_padded == extract_batch per image
@pytest.mark.parametrize('maxk,capacity', [(400, None), (-1, 8192)])
def test_sift_extract_padded_equals_extract_batch(maxk, capacity):
    sift = OpenCVSIFT(max_keypoints=maxk)
    batches = [torch.cat([_sift_images('sift_small'), _sift_images('sift_warp')]).to(DEV), _textures(4, 240, 320, 1)]
    for imgs in batches:
        singles = sift.extract_batch(imgs)
        assert maxk != -1 or len({s[0].shape[1] for s in singles}) > 1
        _check_padded(sift.extract_padded(imgs, capacity), singles, capacity or maxk)
    vga = _sift_images('sift_vga').to(DEV)
    _check_padded(sift.extract_padded(vga, capacity), sift.extract_batch(vga), capacity or maxk)


# --------------------------------------------------------------------------- 2. SuperPoint: extract_padded == forward per image
def _sp(cls, maxk, thr=0.01, precision='tf32x3'):
    sp = cls(max_keypoints=maxk, keypoint_threshold=thr, precision=precision)
    sd = synthetic_superpoint_bn_state_dict(7) if cls is SuperPointNetBn else synthetic_superpoint_state_dict(7)
    sp.load_state_dict(sd, strict=True)
    return sp.to(DEV).eval()


def _sp_images():
    """three 240 x 320 images with different keypoint counts: noise with blobs, its left half constant, three quarters constant"""
    img = synthetic_images(3, 240, 320, 9)
    img[1, :, :, :160] = 0.5
    img[2, :, :, 80:] = 0.5
    return img.to(DEV)


@pytest.mark.parametrize('cls', [SuperPointNet, SuperPointNetBn])
def test_superpoint_extract_padded_equals_forward(cls):
    imgs = _sp_images()
    counts = [int(cls.forward(_sp(cls, -1), imgs[b:b + 1])[0].shape[1]) for b in range(3)]
    assert len(set(counts)) == 3 and min(counts) > 0, counts
    mid = sorted(counts)[1]
    for maxk, cap in ((-1, max(counts) + 5), (mid, None), (mid, 2 * max(counts))):       # keeps all / binds for some images only
        sp = _sp(cls, maxk)
        singles = [sp(imgs[b:b + 1]) for b in range(3)]
        _check_padded(sp.extract_padded(imgs, cap), singles, cap or maxk)


@pytest.mark.parametrize('maxk', [-1, 500])
def test_superpoint_padded_post_chain_matches_reference(maxk):
    """The post-processing of extract_padded on injected layer outputs against the reference run on each image alone"""
    fx = torch.load(os.path.join(GOLDEN_DIR, PAD_NAME + '.pt'), weights_only=False)
    scores, desc = padded_inputs()
    assert inputs_sha256(scores, desc) == fx['sha256']
    c = PAD_CASE
    h, w = c['h'], c['w']
    sp = SuperPointNet(max_keypoints=maxk, nms_kernel=c['nms'], remove_borders_size=4, keypoint_threshold=c['thr']).to(DEV).eval()
    probs, coarse = _probs_coarse(scores, desc)
    K = 1024
    lafs, sc, ds, num, over = [t.cpu() for t in sp._keypoints_padded(probs, coarse, h, w, K)]
    heat = pixel_heat(scores.permute(0, 2, 3, 1))
    kept = nms_threshold_borders(heat, c['nms'], c['thr'], 4)
    ref = fx['maxk'][maxk]
    assert over.tolist() == [0, 0, 0] and num.tolist() == [r['keypoints'].shape[0] for r in ref]
    assert len(set(num.tolist())) > 1
    err = 0.0
    for b, r in enumerate(ref):
        n = int(num[b])
        kp = lafs[b, :n, :, 2]
        pos = (kp[:, 1].long() * w + kp[:, 0].long()).tolist()
        ref_pos = (r['keypoints'][:, 1].long() * w + r['keypoints'][:, 0].long()).tolist()
        cand = torch.nonzero(kept[b].view(-1))[:, 0]
        topk = maxk != -1 and maxk < cand.numel()
        _same_up_to_ties(pos, sc[b, :n].tolist(), ref_pos, r['scores'].tolist(), cand.tolist(), kept[b].view(-1)[cand].tolist(), topk)
        at = {p: i for i, p in enumerate(pos)}
        for j, d in zip(r['desc_idx'].tolist(), r['descriptors']):
            err = max(err, float((ds[b, at[ref_pos[j]]] - d).abs().max()))
        assert (lafs[b, n:] == 0).all() and (sc[b, n:] == 0).all() and (ds[b, n:] == 0).all()
    print(f'\n[padded post chain, max_keypoints {maxk}] keypoints {num.tolist()}, max |desc - reference| {err:.2e} (bound 1e-6)')
    assert err <= 1e-6


# --------------------------------------------------------------------------- 3. no host synchronisation; graph capture
def _matcher_parts(frontend, method='none', seed=3):
    side = {'none': 1, 'scale_rotation': 4}[method]
    if frontend == 'sift':
        fe, D = OpenCVSIFT(max_keypoints=300), 128
    else:
        fe, D = _sp(SuperPointNet, 256), 256
    cfg = default_config(descriptor_dim=D, num_heads=4, num_stages=2, num_iters=20, side_info_size=side)
    cfg['precision'] = 'tf32x3'
    sg = SuperGlue(cfg)
    sg.load_state_dict(synthetic_state_dict(cfg, seed=seed), strict=True)
    mc = {'superglue': {'laf_to_sideinfo_method': method}, 'inference': {'match_threshold': 0.0}}
    return fe, sg.to(DEV).eval(), mc


def _pair_images(frontend, B, seed):
    if frontend == 'sift':
        base = _textures(B, 256, 336, seed)
    else:
        base = synthetic_images(B, 256, 336, seed).to(DEV)
    return base[:, :, :240, :320].contiguous(), base[:, :, 12:252, 9:329].contiguous()


def test_no_host_synchronisation_and_graph_capture():
    sift, sp = OpenCVSIFT(max_keypoints=300), _sp(SuperPointNet, 256)
    tex, imgs = _textures(3, 240, 320, 4), _sp_images()
    eager = [sift.extract_padded(tex), sp.extract_padded(imgs)]                 # warm-up: workspaces, weights, kernel attributes
    fe, sg, mc = _matcher_parts('sift')
    m = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
    i0, i1 = _pair_images('sift', 2, 5)
    want = m(i0, i1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        again = [sift.extract_padded(tex), sp.extract_padded(imgs)]
        got = m(i0, i1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(eager, again):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert all(torch.equal(got[k], want[k]) for k in want)
    for fn in (lambda: sift.extract_padded(tex), lambda: sp.extract_padded(imgs)):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn()
        g.replay()
        torch.cuda.synchronize()
        ref = fn()
        assert all(torch.equal(x, y) for x, y in zip(out, ref))


# --------------------------------------------------------------------------- 4. overflow
def test_sift_overflow_flags_only_the_images_over_capacity():
    imgs = _textures(3, 240, 320, 2)
    sift = OpenCVSIFT(max_keypoints=-1)
    singles = sift.extract_batch(imgs)
    n = [s[0].shape[1] for s in singles]
    K = sorted(n)[1]                                                            # cuts the largest image only
    lafs, scores, desc, num, over = sift.extract_padded(imgs, K)
    assert over.tolist() == [int(x > K) for x in n] and num.tolist() == [min(x, K) for x in n] and sum(over.tolist()) == 1
    for b, s in enumerate(singles):
        k = min(n[b], K)
        for got, want in zip((lafs, scores, desc), s):
            assert torch.equal(got[b, :k], want[0, :k]), b                     # the first K in response order
    # the capacity before NMS: the selection runs on the keypoints that fitted, the images below it are unchanged
    raw = sift._detect_select(sift._image(imgs)).count.tolist()
    small = OpenCVSIFT(max_keypoints=-1, capacity=sorted(raw)[1])
    lafs, scores, desc, num, over = small.extract_padded(imgs, 8192)
    assert over.tolist() == [int(x > small.capacity) for x in raw] and sum(over.tolist()) == 1
    for b, s in enumerate(singles):
        k = int(num[b])
        assert k <= small.capacity and (lafs[b, k:] == 0).all() and torch.isfinite(desc[b]).all()
        if not over[b]:
            assert k == n[b] and torch.equal(desc[b, :k], s[2][0]) and torch.equal(lafs[b, :k], s[0][0])


def test_superpoint_overflow_flags_only_the_images_over_capacity():
    # more than 16384 non-maximum-suppression survivors in image 0 (test_post_chain_over_capacity's maps), few in image 1
    scores, desc = post_inputs(2, 720, 960, 12)
    scores[1] *= 0.005005                                                      # a survivor must exceed 0.999 to pass the threshold
    probs, coarse = _probs_coarse(scores, desc)
    sp = SuperPointNet(max_keypoints=2048, nms_kernel=5, keypoint_threshold=0.005).to(DEV).eval()
    lafs, sc, ds, num, over = sp._keypoints_padded(probs, coarse, 720, 960, 2048)
    assert over.tolist() == [1, 0] and int(num[0]) == 2048
    one = sp._keypoints(probs[720 * 960 // 64:], coarse[720 * 960 // 64:], 720, 960)
    n1 = one[0].shape[1]
    assert 0 < n1 < 2048 and int(num[1]) == n1
    for got, want in zip((lafs, sc, ds), one):
        assert torch.equal(got[1, :n1], want[0]) and (got[1, n1:] == 0).all()
    assert torch.isfinite(ds).all() and torch.isfinite(sc).all()
    # a capacity below the kept count: flagged, clamped, the first K in output order
    imgs = _sp_images()
    sp = _sp(SuperPointNet, -1)
    singles = [sp(imgs[b:b + 1]) for b in range(3)]
    n = [s[0].shape[1] for s in singles]
    K = sorted(n)[1]
    lafs, sc, ds, num, over = sp.extract_padded(imgs, K)
    assert over.tolist() == [int(x > K) for x in n] and num.tolist() == [min(x, K) for x in n]
    for b, s in enumerate(singles):
        k = min(n[b], K)
        assert torch.equal(lafs[b, :k], s[0][0, :k]) and torch.equal(ds[b, :k], s[2][0, :k])


# --------------------------------------------------------------------------- 5. ImagePairMatcher: graph == eager, pairs == OpenGlueMatcher
@pytest.mark.parametrize('method', ['none', 'scale_rotation'])
@pytest.mark.parametrize('frontend', ['sift', 'superpoint'])
def test_image_pair_matcher(frontend, method, monkeypatch):
    fe, sg, mc = _matcher_parts(frontend, method)
    captured = [0]
    orig = torch.cuda.CUDAGraph.capture_end

    def counting(self):
        captured[0] += 1
        return orig(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'capture_end', counting)
    graphed = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
    eager = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
    single = OpenGlueMatcher(fe, sg, mc)
    for i in range(3):
        i0, i1 = _pair_images(frontend, 3, 20 + i)
        got, want = graphed(i0, i1), eager(i0, i1)
        for k in ImagePairMatcher._OUT_KEYS:
            assert torch.equal(got[k], want[k]), (i, k)
        n0, n1 = got['num_keypoints0'].tolist(), got['num_keypoints1'].tolist()
        assert got['overflow0'].tolist() == [0] * 3 and got['overflow1'].tolist() == [0] * 3
        batched = compact_matches(got['matches0'], got['matching_scores0'], got['lafs0'], got['lafs1'])
        for b in range(3):
            alone = single({'image0': i0[b:b + 1], 'image1': i1[b:b + 1]})
            sel = batched['batch_indexes'] == b
            gs = {tuple(x) for x in batched['original_matching_idxs'][sel].tolist()}
            ws = {tuple(x) for x in alone['original_matching_idxs'].tolist()}
            # decisions within the parity bound of the threshold or of a tie may flip; the lists must agree on the rest
            assert len(gs ^ ws) <= max(2, len(ws) // 50), (i, b, n0[b], n1[b], len(gs), len(ws), len(gs ^ ws))
            assert len(ws) > 0
    assert captured[0] == 1
    out = graphed(i0, i1, borrow=True)
    assert out['matches0'] is graphed(i0, i1, borrow=True)['matches0']


# --------------------------------------------------------------------------- 6. a pair with an image without keypoints
def test_pair_without_keypoints_is_masked():
    fe, sg, mc = _matcher_parts('sift')
    i0, i1 = _pair_images('sift', 3, 30)
    flat = i1.clone()
    flat[1] = 128                                                               # a constant image: no SIFT keypoint
    for graph in (False, True):
        m = ImagePairMatcher(fe, sg, mc, use_cuda_graph=graph)
        ref, got = m(i0, i1), m(i0, flat)
        assert got['num_keypoints1'].tolist()[1] == 0 and got['num_keypoints0'].tolist()[1] > 0
        assert (got['matches0'][1] == -1).all() and (got['matching_scores0'][1] == 0).all()
        assert (got['matches1'][1] == -1).all() and (got['matching_scores1'][1] == 0).all()
        for k in ImagePairMatcher._OUT_KEYS:
            assert torch.isfinite(got[k].double()).all(), k
            assert torch.equal(got[k][0::2], ref[k][0::2]), k                   # pairs 0 and 2 unchanged
        assert int((got['matches0'][0::2] >= 0).sum()) > 0


# --------------------------------------------------------------------------- 7. training end to end from SuperPoint's padded output
def test_superpoint_pairs_train_end_to_end_with_every_keypoint():
    from openglue_b200 import synthesize_homography_pairs
    from openglue_b200.features import get_laf_to_sideinfo_converter, prepare_features_output
    from openglue_b200.gt_matches import IGNORE_INDEX, generate_gt_matches
    from openglue_b200.losses import criterion_with_grad
    from openglue_b200.optim import ClippedAdam
    from openglue_b200.training import GraphedTrainStep, TrainStep
    B = 3
    g = torch.Generator(device=DEV).manual_seed(7)
    low = torch.rand(B, 3, 24, 32, generator=g, device=DEV)
    imgs = (torch.nn.functional.interpolate(low, size=(288, 368), mode='bicubic', align_corners=False).clamp(0, 1) * 255)
    imgs = imgs.to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    raw = synthesize_homography_pairs(imgs, 24, generator=g)                   # 240 x 320 pairs
    sp = _sp(SuperPointNet, -1, thr=0.005)
    conv = get_laf_to_sideinfo_converter('none')
    feats, counts = [], []
    for i in (0, 1):
        image = raw[f'image{i}']
        image = image[:, None] if image.dim() == 3 else image
        counts.append([int(sp(image[b:b + 1])[0].shape[1]) for b in range(B)])
        lafs, resp, desc, n, over = sp.extract_padded(image, 2048)
        assert n.tolist() == counts[i] and over.tolist() == [0] * B                # every keypoint kept
        feats.append(prepare_features_output(lafs, resp, desc, conv))
        raw[f'num_keypoints{i}'] = n
    assert max(max(c) for c in counts) < 2048 and (len(set(counts[0])) > 1 or len(set(counts[1])) > 1), counts   # really padded
    data, y_true = generate_gt_matches(raw, feats[0], feats[1], 3.0, 5.0)
    for b in range(B):
        assert (y_true['gt_matches0'][b, counts[0][b]:] == IGNORE_INDEX).all()
    assert int((y_true['gt_matches0'] >= 0).sum()) > 0
    cfg = default_config(descriptor_dim=256, num_heads=4, num_stages=2, num_iters=20)
    cfg['precision'] = 'tf32x3'
    models = []
    for _ in range(2):
        m = SuperGlue(cfg)
        m.load_state_dict(synthetic_state_dict(cfg, seed=9), strict=True)
        models.append(m.to(DEV).train())
    m_e, m_g = models
    opt_e, opt_g = ClippedAdam(m_e.parameters(), lr=1e-3), ClippedAdam(m_g.parameters(), lr=1e-3)
    step = GraphedTrainStep(m_g, data, y_true, optimizer=opt_g)
    for j in range(3):
        st = TrainStep(m_e, data)
        scores, _, _ = st.forward()
        loss, ds = criterion_with_grad(y_true, {'scores': scores})
        gr = st.backward(ds)
        for k, p in m_e.named_parameters():
            p.grad = gr[k].reshape(p.shape).clone()
        opt_e.step()
        out = step(data, y_true)
        torch.cuda.synchronize()
        assert torch.isfinite(out['loss']) and torch.equal(out['loss'], loss['loss']), j
        for (k, pe), (_, pg) in zip(m_e.named_parameters(), m_g.named_parameters()):
            assert torch.equal(pe, pg), (j, k)
