"""SuperPoint front-end (SURVEY.md section 8, row f4) against fixtures minted from the UNMODIFIED reference module
(oracle/gen_golden_superpoint.py; kornia's nms2d restated there - kornia is not installed)."""
import os

import pytest
import torch

CASES = ['superpoint_all', 'superpoint_topk', 'superpoint_thr', 'superpoint_bn']


def _load(name):
    here = os.path.dirname(os.path.abspath(__file__))
    return torch.load(os.path.join(here, 'golden', name + '.pt'), weights_only=False)


def _decisions(heat, nms, thr, border, margin):
    """From a dense score map: which pixels the reference keeps (keep) and which of these decisions are DECISIVE - no comparison of
    the rule (x > every other value of the replicate-padded window, x > 0, x > thr) is closer than `margin`."""
    import torch.nn.functional as F
    B, H, W = heat.shape
    r = nms // 2
    xp = F.pad(heat[:, None], [r, r, r, r], mode='replicate')
    win = xp.unfold(2, nms, 1).unfold(3, nms, 1).reshape(B, H, W, nms * nms)
    others = torch.cat([win[..., :nms * nms // 2], win[..., nms * nms // 2 + 1:]], -1)
    mx = others.max(-1).values.clamp_min(0)
    gap = (heat - mx)
    keep = (gap > 0) & (heat > thr)
    decisive = (gap.abs() > margin) & ((heat - thr).abs() > margin)
    inb = torch.zeros_like(keep)
    inb[:, border:H - border, border:W - border] = True
    return keep & inb, decisive | ~inb


def _disagreements(ours, ref, keep, decisive, heat, margin):
    """Keypoints of one image, ours and the reference's (sets of (x, y)), against the per-pixel rule: a pixel whose NMS decision is
    decisive (`_decisions`) must be in both outputs or in neither - unless the output is a top-k of fewer than all kept pixels and
    the pixel's score is not above both outputs' lowest score by more than `margin` (then the cut decides, not the rule).
    Returns the number of decisive pixels on which the outputs differ."""
    H, W = heat.shape
    mask = lambda pts: torch.zeros(H * W, dtype=torch.bool).index_fill_(0, torch.tensor([y * W + x for x, y in pts], dtype=torch.long), True).view(H, W)
    m_ours, m_ref = mask(ours), mask(ref)
    decided = decisive.clone()
    if min(len(ours), len(ref)) < int(keep.sum()):
        lowest = lambda m: float(heat[m].min()) if m.any() else float('inf')
        decided &= heat > max(lowest(m_ours), lowest(m_ref)) + margin
    return int(((m_ours != m_ref) & decided).sum())


@pytest.mark.parametrize('name', CASES)
def test_superpoint_fixture_is_self_consistent(name):
    """The fixture's keypoints follow from its own dense heat map by the restated rule (this is what pins the test helper)."""
    fx = _load(name)
    batch, h, w, maxk, thr, _ = fx['case']
    keep, _ = _decisions(fx['heat_f32'], 9, thr, 4, 0.0)
    lafs, scores = fx['lafs'], fx['scores']
    assert lafs.shape[0] == batch and lafs.shape[2:] == (2, 3)
    assert torch.equal(lafs[..., :2], torch.eye(2).expand(batch, lafs.shape[1], 2, 2))
    for b in range(batch):
        xy = lafs[b, :, :, 2].long()
        assert keep[b, xy[:, 1], xy[:, 0]].all()                          # every returned keypoint is a kept pixel
        assert torch.equal(scores[b], fx['heat_f32'][b, xy[:, 1], xy[:, 0]])
        n_kept = int(keep[b].sum())
        assert lafs.shape[1] <= n_kept
        if maxk != -1 and n_kept > maxk:
            assert (scores[b][:-1] >= scores[b][1:]).all()                # top-k output is sorted
    d = fx['descriptors']
    assert (d.norm(dim=-1) - 1).abs().max() < 1e-5


def test_superpoint_bn_fold_reproduces_the_reference_layers():
    """SuperPointNetBn on the CPU: the weights the kernels are handed (BatchNorm folded into the convolution it follows, packed
    [Cout, (3 ky + kx) Cin + ci]) reproduce the dense outputs of the reference's `_forward_layers` (fixture: float64 run of the
    unmodified SuperPointNetBn) when the same schedule - conv, ReLU, max-pool, 1x1 heads, softmax, channel norm - runs in float64
    torch.  Also: the reference's state_dict loads strictly, and the checkpoint key renaming follows model.py:151-171."""
    import sys
    import torch.nn.functional as F
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    from gen_golden_superpoint import synthetic_superpoint_bn_state_dict
    from openglue_b200 import SuperPointNetBn
    fx = _load('superpoint_bn')
    batch, h, w, maxk, thr, seed = fx['case']
    model = SuperPointNetBn(max_keypoints=maxk, keypoint_threshold=thr)
    print(model.load_state_dict(synthetic_superpoint_bn_state_dict(seed), strict=True))
    model.eval()
    wts = model._weights()

    def conv(x, name, relu=True):
        wp, b = wts[name]
        co, kk = wp.shape
        k = 3 if kk == 9 * x.shape[1] else 1
        wt = wp.double().reshape(co, k, k, -1).permute(0, 3, 1, 2)
        y = F.conv2d(x, wt, b.double(), padding=k // 2)
        return y.relu() if relu else y
    x = fx['image'].double()
    for i in range(4):
        x = conv(conv(x, f'conv{i + 1}a'), f'conv{i + 1}b')
        if i != 3:
            x = F.max_pool2d(x, 2, 2)
    desc = conv(conv(x, 'convDa'), 'convDb', relu=False)
    desc = desc / desc.norm(dim=1, keepdim=True)
    cell = conv(conv(x, 'convPa'), 'convPb', relu=False).softmax(1)[:, :-1]
    heat = cell.permute(0, 2, 3, 1).reshape(batch, h // 8, w // 8, 8, 8).permute(0, 1, 3, 2, 4).reshape(batch, h, w)
    # the fold is done in float64 and rounded once to float32: ~1e-7 relative per layer
    assert float((heat - fx['heat_f64'].double()).abs().max()) <= 2e-6
    assert float((desc - fx['desc_map_f64'].double()).abs().max()) <= 2e-6
    sd = {'inc.conv.conv.0.weight': 0, 'inc.conv.conv.4.running_var': 1, 'down2.mpconv.1.conv.1.bias': 2, 'down3.mpconv.1.conv.3.weight': 3, 'convPa.weight': 4}
    assert set(SuperPointNetBn.rename_weights_keys(sd)) == {'conv1a.weight', 'bn1b.running_var', 'bn3a.bias', 'conv4b.weight', 'convPa.weight'}


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name', CASES)
def test_superpoint_matches_reference(name, precision):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    from gen_golden_superpoint import synthetic_superpoint_bn_state_dict, synthetic_superpoint_state_dict
    from openglue_b200 import SuperPointNet, SuperPointNetBn
    dev = torch.device('cuda:0')
    fx = _load(name)
    batch, h, w, maxk, thr, seed = fx['case']
    if name.endswith('_bn'):                                                             # the BatchNorm variant (model.py:132-199)
        model = SuperPointNetBn(max_keypoints=maxk, keypoint_threshold=thr, precision=precision)
        model.load_state_dict(synthetic_superpoint_bn_state_dict(seed), strict=True)
    else:
        model = SuperPointNet(max_keypoints=maxk, keypoint_threshold=thr, precision=precision)
        model.load_state_dict(synthetic_superpoint_state_dict(seed), strict=True)       # the reference module's keys, strict
    model = model.to(dev).eval()
    lafs, scores, desc = model(fx['image'].to(dev))
    # dense cell probabilities -> heat map, against the reference's fp64 layers
    probs = model.last_probs
    heat = probs[..., :64].reshape(batch, h // 8, w // 8, 8, 8).permute(0, 1, 3, 2, 4).reshape(batch, h, w).cpu()
    err = float((heat.double() - fx['heat_f64'].double()).abs().max())
    ref_err = float((fx['heat_f32'].double() - fx['heat_f64'].double()).abs().max())    # the reference's own fp32 rounding on this input
    bound = max(1e-5, 5 * ref_err)                    # (1.0e-6 .. 1.3e-6 on the plain fixtures, 3.9e-6 behind the BatchNorm scales)
    print(f'{name} {precision}: max |heat - ref64| {err:.2e} (bound {bound:.1e}, ref32-vs-ref64 {ref_err:.1e}); keypoints {tuple(lafs.shape)}')
    assert err <= bound
    # keypoints: identical wherever the reference's decision is decisive at 10x that error
    lafs, scores, desc = lafs.cpu(), scores.cpu(), desc.cpu()
    keep, decisive = _decisions(fx['heat_f64'].float(), 9, thr, 4, 10 * max(err, 1e-7))
    assert torch.equal(lafs[..., :2], torch.eye(2).expand(batch, lafs.shape[1], 2, 2))
    ref_lafs, ref_scores, ref_desc = fx['lafs'], fx['scores'], fx['descriptors']
    all_decisive = bool(decisive.all())
    if all_decisive:
        assert lafs.shape == ref_lafs.shape
    margin = 10 * max(err, 1e-7)
    for b in range(batch):
        ours = {(int(x), int(y)): j for j, (x, y) in enumerate(lafs[b, :, :, 2].tolist())}
        ref_pts = [tuple(p) for p in ref_lafs[b, :, :, 2].long().tolist()]
        for j, (x, y) in enumerate(ref_pts):
            if (x, y) in ours:
                i = ours[(x, y)]
                assert abs(float(scores[b, i]) - float(ref_scores[b, j])) <= bound + ref_err    # the fixture's scores are the reference's fp32 run
                assert (desc[b, i] - ref_desc[b, j]).abs().max() <= 1e-4
        # every pixel whose decision is decisive - by the NMS rule and, for a top-k, by the cut - is decided the same way
        bad = _disagreements(list(ours), ref_pts, keep[b], decisive[b], fx['heat_f64'][b].float(), margin)
        print(f'  image {b}: {len(ours)} / {len(ref_pts)} keypoints, {int((~decisive[b]).sum())} non-decisive pixels, {bad} decisive disagreements')
        assert bad == 0
    # ordering: where the reference's order is decided by score gaps larger than the error, ours is the same sequence
    if all_decisive:
        for b in range(batch):
            gaps = (ref_scores[b][:-1] - ref_scores[b][1:]).abs()
            if ref_lafs.shape[1] == lafs.shape[1] and (gaps > 10 * max(err, 1e-7)).all():
                assert torch.equal(lafs[b, :, :, 2], ref_lafs[b, :, :, 2])


@pytest.mark.gpu
def test_image_pair_to_matches_pipeline():
    """Front-end -> matching core, device-resident: SuperPointNet on two views of one synthetic scene (the second a shifted crop),
    keypoints / scores / descriptors handed to MatchingCore as inference.py does (keypoints = lafs[..., 2], side info = the detector
    response), mutual matches out.  Random weights: the check is plumbing (shapes, finiteness, index ranges, mutual consistency)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    from gen_golden_superpoint import synthetic_superpoint_state_dict, synthetic_images
    from openglue_b200 import MatchingCore, SuperGlue, SuperPointNet
    from openglue_b200.synthetic import default_config, synthetic_state_dict
    dev = torch.device('cuda:0')
    sp = SuperPointNet(max_keypoints=256)
    sp.load_state_dict(synthetic_superpoint_state_dict(7), strict=True)
    sp = sp.to(dev).eval()
    scene = synthetic_images(2, 256, 320, 9).to(dev)
    img0, img1 = scene[:, :, :240, :304].contiguous(), scene[:, :, 16:, 16:].contiguous()       # two 240 x 304 views, shifted by (16, 16)
    lafs0, sc0, d0 = sp(img0)
    lafs1, sc1, d1 = sp(img1)
    assert lafs0.shape[1] == 256 and lafs1.shape[1] == 256 and d0.shape == (2, 256, 256)
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=20)
    sg = SuperGlue(cfg)
    sg.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    core = MatchingCore(sg.to(dev).eval(), 0.0)
    data = {'keypoints0': lafs0[:, :, :, 2].contiguous(), 'keypoints1': lafs1[:, :, :, 2].contiguous(),
            'side_info0': sc0[..., None].contiguous(), 'side_info1': sc1[..., None].contiguous(),
            'local_descriptors0': d0, 'local_descriptors1': d1, 'image0_size': (304, 240), 'image1_size': (304, 240)}
    out = core(data, want_scores=True)
    m0, m1 = out['matches0'].cpu(), out['matches1'].cpu()
    assert torch.isfinite(out['scores']).all()
    assert m0.shape == (2, 256) and int(m0.max()) < 256 and int(m0.min()) >= -1
    for b in range(2):                                                   # mutual: matches1[matches0[i]] == i
        i = (m0[b] >= 0).nonzero()[:, 0]
        assert torch.equal(m1[b, m0[b, i]], i)
