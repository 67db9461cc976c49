"""Training on padded batches on the H100: pairs with their own keypoint counts n_b, m_b at a shared capacity N, M through
TrainStep, criterion, generate_gt_matches and GraphedTrainStep.  At full lengths the padded step must be the uniform step bit
for bit; the padding's contents must not matter; every gradient at a padding row is 0; a single pair at a larger capacity is
the step on the trimmed pair; a graph captured once replays any set of lengths as the eager step computes it.  The new
operator forms (masked BatchNorm, masked softmax, Sinkhorn with history and its backward, criterion, labels) are checked pair
by pair against float64 torch or the uniform kernels on the trimmed pair."""
import copy

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._ops import _Ops
from openglue_b200.gt_matches import IGNORE_INDEX, gt_matches
from openglue_b200.losses import criterion, criterion_with_grad
from openglue_b200.optim import ClippedAdam
from openglue_b200.superglue import SuperGlue
from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
from openglue_b200.training import GraphedTrainStep, TrainStep
from test_padded_training_host import case_config, case_state, case_batch, check_against, reference_run, train_step_run
from test_training_reference import _Check

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
KEYS = ('keypoints', 'side_info', 'local_descriptors')
CONFIGS = {
    'd256_h4': dict(descriptor_dim=256, num_heads=4, num_stages=2, num_iters=20),
    'd64_h2': dict(descriptor_dim=64, num_heads=2, num_stages=2, num_iters=20),
    'd32_h4': dict(descriptor_dim=32, num_heads=4, num_stages=1, num_iters=20),
}
OPTIONS = {'plain': {}, 'residual_offset': dict(residual=True, use_offset=True), 'no_descriptors': dict(no_descriptors=True)}


def _model(name, precision, options=(), seed=3):
    cfg = default_config(**CONFIGS[name])
    opts = OPTIONS[options] if isinstance(options, str) else {}
    if 'residual' in opts:
        cfg['residual'] = True
    if 'use_offset' in opts:
        cfg['attention_gnn']['use_offset'] = True
    if 'no_descriptors' in opts:
        cfg['no_descriptors'] = True
    cfg['precision'] = precision
    m = SuperGlue(cfg)
    sd = synthetic_state_dict(cfg, seed=seed)
    if cfg.get('residual'):
        sd['mix_coefs'] = torch.linspace(-1, 1, cfg['descriptor_dim']).reshape(-1, 1)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).train()


def _pair(d, n, m, seed, wh=(640., 480.)):
    p = synthetic_pairs(1, n, m, d, 1, seed=seed, image_wh=tuple(int(x) for x in wh))
    p['image0_size'] = p['image1_size'] = wh
    g = torch.Generator().manual_seed(seed)
    p['gt_matches0'] = torch.randint(-2, m, (1, n), generator=g)
    p['gt_matches1'] = torch.randint(-2, n, (1, m), generator=g)
    return p


def _padded(pairs, N, M, fill=0.0):
    """One padded batch (and its labels) of single-pair dicts at capacity N, M; the padding slots hold `fill`."""
    B = len(pairs)
    data, y = {}, {}
    for i, cap in ((0, N), (1, M)):
        for k in KEYS:
            src = [p[f'{k}{i}'][0] for p in pairs]
            t = torch.full((B, cap, src[0].shape[-1]), fill, dtype=torch.float32)
            for b, s in enumerate(src):
                t[b, :s.shape[0]] = s
            data[f'{k}{i}'] = t.to(DEV)
        g = torch.full((B, cap), -1, dtype=torch.int64)
        for b, p in enumerate(pairs):
            g[b, :p[f'gt_matches{i}'].shape[1]] = p[f'gt_matches{i}'][0]
        y[f'gt_matches{i}'] = g.to(DEV)
        n = torch.tensor([p[f'keypoints{i}'].shape[1] for p in pairs])
        data[f'num_keypoints{i}'] = y[f'num_keypoints{i}'] = n
        data[f'image{i}_size'] = torch.tensor([list(p[f'image{i}_size']) for p in pairs], dtype=torch.float32)
    return data, y


def _step(model, data, y):
    """eager padded / uniform step: outputs, loss, every gradient, BatchNorm buffers"""
    st = TrainStep(model, data)
    scores, c0, c1 = st.forward()
    loss, ds = criterion_with_grad(y, {'scores': scores})
    g = st.backward(ds)
    torch.cuda.synchronize()
    out = {'scores': scores, 'ctx0': c0, 'ctx1': c1, 'loss': loss['loss']}
    out.update({f'grad.{k}': v for k, v in g.items()})
    out.update({f'buf.{k}': v.clone() for k, v in model.named_buffers()})
    return out


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize('options', list(OPTIONS))
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name', list(CONFIGS))
def test_full_lengths_are_the_uniform_step_bit_for_bit(name, precision, options):
    d = CONFIGS[name]['descriptor_dim']
    pairs = [_pair(d, 96, 80, seed=s) for s in (1, 2)]
    data, y = _padded(pairs, 96, 80)
    uni = {k: v for k, v in data.items() if not k.startswith('num_keypoints') and not k.startswith('image')}
    uni['image0_size'] = uni['image1_size'] = (640., 480.)
    yu = {k: y[k] for k in ('gt_matches0', 'gt_matches1')}
    m_u, m_p = _model(name, precision, options), _model(name, precision, options)
    _equal(_step(m_u, uni, yu), _step(m_p, data, y))


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_padding_contents_do_not_matter_and_padding_gradients_are_zero(precision):
    d = 64
    pairs = [_pair(d, 70, 50, 1), _pair(d, 1, 64, 2, wh=(320., 240.)), _pair(d, 33, 9, 3)]
    N, M = 72, 64
    runs = []
    for fill in (0.0, float('nan'), 1e30):
        data, y = _padded(pairs, N, M, fill)
        runs.append(_step(_model('d64_h2', precision, 'residual_offset'), data, y))
    _equal(runs[0], runs[1])
    _equal(runs[0], runs[2])
    r = runs[0]
    for b, p in enumerate(pairs):
        n, m = p['keypoints0'].shape[1], p['keypoints1'].shape[1]
        s = r['scores'][b].clone()
        assert torch.isfinite(s[:n + 1, :m + 1]).all()
        s[:n + 1, :m + 1] = -float('inf')
        assert torch.isneginf(s).all()
        assert (r['ctx0'][b, :, n:] == 0).all() and (r['ctx1'][b, :, m:] == 0).all()
        assert (r['grad.local_descriptors0'][b, n:] == 0).all() and (r['grad.local_descriptors1'][b, m:] == 0).all()
    for k, v in r.items():
        if k.startswith('grad.'):
            assert torch.isfinite(v).all(), k


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_one_pair_at_a_larger_capacity_is_the_step_on_the_trimmed_pair(precision):
    d = 64
    p = _pair(d, 57, 41, 5)
    data, y = _padded([p], 80, 64)
    uni = {k: p[k].to(DEV) if torch.is_tensor(p[k]) else p[k] for k in p if not k.startswith('gt_')}
    yu = {k: p[k].to(DEV) for k in ('gt_matches0', 'gt_matches1')}
    got = _step(_model('d64_h2', precision, 'residual_offset'), data, y)
    ref = _step(_model('d64_h2', precision, 'residual_offset'), uni, yu)
    got['scores'] = got['scores'][:, :58, :42]
    got['ctx0'], got['ctx1'] = got['ctx0'][:, :, :57], got['ctx1'][:, :, :41]
    got['grad.local_descriptors0'] = got['grad.local_descriptors0'][:, :57]
    got['grad.local_descriptors1'] = got['grad.local_descriptors1'][:, :41]
    for k in ref:
        a, b = got[k].double(), ref[k].double()
        bound = max(2e-4 * float(b.abs().max()), 1e-5)
        assert float((a - b).abs().max()) <= bound, k


@pytest.mark.parametrize('case', ['mixed', 'mixed_offset_nodesc', 'one_pair'])
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_padded_step_against_the_reference(case, precision):
    """The padded step on the device against float64 / float32 autograd of the restated reference (B >= 3, mixed lengths, one
    pair with n_b = 1, every pair and image with its own size) or, for one pair, of the unmodified reference on the trimmed pair;
    padding filled with NaN.  Bound per tensor: |got - ref64| <= max(4 max|ref32 - ref64|, 2e-4 max|ref64|)."""
    trimmed = case == 'one_pair'
    r64 = reference_run(case, torch.float64, trimmed=trimmed)
    r32 = reference_run(case, torch.float32, trimmed=trimmed)
    model = SuperGlue(dict(case_config(case), precision=precision))
    model.load_state_dict(case_state(case), strict=True)
    got = train_step_run(case, None, model.to(DEV).train(), float('nan'))
    _, _, lens0, lens1, _, _ = case_batch(case)
    chk = _Check(f'[{case} {precision}]')
    check_against(got, [r64, r32], lens0, lens1, chk)
    chk.done()


def _eager_and_graphed(name, precision, batches):
    """the eager padded step + ClippedAdam and GraphedTrainStep (captured on the first batch) over `batches`: equal bit for bit"""
    m_e, m_g = _model(name, precision, 'residual_offset'), _model(name, precision, 'residual_offset')
    m_g.load_state_dict(copy.deepcopy(m_e.state_dict()))
    opt_e, opt_g = ClippedAdam(m_e.parameters(), lr=1e-3), ClippedAdam(m_g.parameters(), lr=1e-3)
    step = GraphedTrainStep(m_g, *batches[0], optimizer=opt_g)
    for j, (data, y) in enumerate(batches):
        st = TrainStep(m_e, data)
        scores, _, _ = st.forward()
        loss, ds = criterion_with_grad(y, {'scores': scores})
        g = st.backward(ds)
        for k, p in m_e.named_parameters():
            p.grad = g[k].reshape(p.shape).clone()
        opt_e.step()
        out = step(data, y)
        torch.cuda.synchronize()
        assert torch.equal(out['loss'], loss['loss']), j
        for (k, pe), (_, pg) in zip(m_e.named_parameters(), m_g.named_parameters()):
            assert torch.equal(pe, pg), (j, k)
        for (k, be), (_, bg) in zip(m_e.named_buffers(), m_g.named_buffers()):
            assert torch.equal(be, bg), (j, k)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_graph_captured_once_replays_new_lengths_as_the_eager_step(precision):
    d = 64
    sets = [[(60, 50), (12, 64), (64, 1)], [(64, 64), (2, 30), (40, 40)], [(1, 2), (63, 5), (30, 64)]]
    batches = []
    for j, lens in enumerate(sets):
        pairs = [_pair(d, n, m, 10 * j + b, wh=((640., 480.), (320., 241.), (97., 1000.))[b]) for b, (n, m) in enumerate(lens)]
        batches.append(_padded(pairs, 64, 64, fill=float('nan')))
    _eager_and_graphed('d64_h2', precision, batches)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_graphed_full_lengths_are_the_graphed_uniform_step_bit_for_bit(precision):
    pairs = [_pair(64, 96, 80, seed=s) for s in (1, 2)]
    data, y = _padded(pairs, 96, 80)
    uni = {k: v for k, v in data.items() if not k.startswith('num_keypoints') and not k.startswith('image')}
    uni['image0_size'] = uni['image1_size'] = (640., 480.)
    yu = {k: y[k] for k in ('gt_matches0', 'gt_matches1')}
    m_u, m_p = _model('d64_h2', precision, 'residual_offset'), _model('d64_h2', precision, 'residual_offset')
    lu, lp = GraphedTrainStep(m_u, uni, yu)(uni, yu), GraphedTrainStep(m_p, data, y)(data, y)
    torch.cuda.synchronize()
    assert torch.equal(lu['loss'], lp['loss'])
    for (k, pu), (_, pp) in zip(m_u.named_parameters(), m_p.named_parameters()):
        assert torch.equal(pu.grad, pp.grad), k
    for (k, bu), (_, bp) in zip(m_u.named_buffers(), m_p.named_buffers()):
        assert torch.equal(bu, bp), k


def test_sift_pairs_train_end_to_end_with_every_keypoint():
    """synthesize_homography_pairs -> OpenCVSIFT.extract_batch -> pad_features -> prepare_features_output -> generate_gt_matches
    -> GraphedTrainStep: every image keeps all its keypoints (lengths as the front end produces them), the labels carry them into
    the loss, and the graphed step equals the eager step."""
    from openglue_b200 import synthesize_homography_pairs
    from openglue_b200.features import get_laf_to_sideinfo_converter, pad_features, prepare_features_output
    from openglue_b200.gt_matches import generate_gt_matches
    from openglue_b200.sift import OpenCVSIFT
    B = 3
    g = torch.Generator(device=DEV).manual_seed(7)
    low = torch.rand(B, 3, 24, 32, generator=g, device=DEV)
    imgs = (torch.nn.functional.interpolate(low, size=(240, 320), mode='bicubic', align_corners=False).clamp(0, 1) * 255)
    imgs = imgs.to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    raw = synthesize_homography_pairs(imgs, 24, generator=g)
    sift = OpenCVSIFT()
    conv = get_laf_to_sideinfo_converter('none')
    feats, counts = [], []
    for i in (0, 1):
        extracted = sift.extract_batch(raw[f'image{i}'])
        counts.append([int(f[0].reshape(-1, 2, 3).shape[0]) for f in extracted])
        lafs, resp, desc, n = pad_features(extracted)
        assert n.tolist() == counts[i] and lafs.shape[1] == max(counts[i])          # every keypoint kept
        feats.append(prepare_features_output(lafs, resp, desc, conv))
        raw[f'num_keypoints{i}'] = n
    assert len(set(counts[0])) > 1 or len(set(counts[1])) > 1, counts              # the batch is really padded
    data, y_true = generate_gt_matches(raw, feats[0], feats[1], 3.0, 5.0)
    assert torch.equal(y_true['num_keypoints0'], raw['num_keypoints0'])
    for b in range(B):
        assert (y_true['gt_matches0'][b, counts[0][b]:] == IGNORE_INDEX).all()
    assert int((y_true['gt_matches0'] >= 0).sum()) > 0
    cfg = default_config(descriptor_dim=128, num_heads=4, num_stages=2, num_iters=20)
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


def test_two_runs_of_the_padded_step_are_identical():
    pairs = [_pair(32, 40, 30, 1), _pair(32, 7, 33, 2)]
    data, y = _padded(pairs, 40, 33)
    _equal(_step(_model('d32_h4', 'tf32x3'), data, y), _step(_model('d32_h4', 'tf32x3'), data, y))


def test_margin_is_refused_on_padded_batches():
    pairs = [_pair(32, 10, 12, 1), _pair(32, 4, 12, 2)]
    data, y = _padded(pairs, 10, 12)
    with pytest.raises(NotImplementedError):
        GraphedTrainStep(_model('d32_h4', 'tf32x3'), data, y, margin=0.5, metric_weight=1.0)


# ---------------------------------------------------------------------------------------------------------- operators
LENS = [37, 1, 64, 20]


def test_masked_batchnorm_forward_and_backward_against_float64():
    B, cap, cols = len(LENS), 64, 48
    g = torch.Generator().manual_seed(0)
    a = torch.randn(B * cap, cols, generator=g)
    for b, n in enumerate(LENS):
        a[b * cap + n:(b + 1) * cap] = float('nan') if b % 2 else 1e30
    gamma, beta, dy = torch.rand(cols, generator=g) + 0.5, torch.randn(cols, generator=g), torch.randn(B * cap, cols, generator=g)
    rm, rv = torch.randn(cols, generator=g), torch.rand(cols, generator=g) + 0.5
    real = torch.cat([torch.arange(b * cap, b * cap + n) for b, n in enumerate(LENS)])
    a_pad = a.clone()
    a_pad[torch.ones(B * cap, dtype=torch.bool).index_fill_(0, real, False)] = 0.0        # the kernels see finite padding
    ops = _Ops(DEV, _cabi.OG_PREC_FP32)
    lens = torch.tensor(LENS, dtype=torch.int32, device=DEV)
    rmd, rvd = rm.to(DEV), rv.to(DEV)
    y, mean, invstd = ops.bn_fwd(a_pad.to(DEV), gamma.to(DEV), beta.to(DEV), 1e-5, 0.1, rmd, rvd, lens=lens)
    da, dgam, dbet = ops.bn_bwd(dy.to(DEV), a_pad.to(DEV), gamma.to(DEV), mean, invstd, lens=lens)
    # float64 reference on the real rows: F.batch_norm with batch statistics, then autograd
    x = a[real].double().relu().requires_grad_(True)
    rm64, rv64 = rm.double(), rv.double()
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y64 = torch.nn.functional.batch_norm(x, rm64, rv64, g64, b64, training=True, momentum=0.1, eps=1e-5)
    y64.backward(dy[real].double())
    assert torch.isfinite(y).all()
    assert (y.cpu()[real].double() - y64).abs().max() < 1e-4
    assert (rmd.cpu().double() - rm64).abs().max() < 1e-5 and (rvd.cpu().double() - rv64).abs().max() < 1e-5
    assert (dgam.cpu().double() - g64.grad).abs().max() < 1e-3 and (dbet.cpu().double() - b64.grad).abs().max() < 1e-3
    dx = x.grad * (a[real] > 0).double()
    assert (da.cpu()[real].double() - dx).abs().max() < 1e-4
    pad = torch.ones(B * cap, dtype=torch.bool).index_fill_(0, real, False)
    assert (da.cpu()[pad] == 0).all()


def test_masked_softmax_forward_and_backward_against_float64():
    B, nq, cols, ld = len(LENS), 5, 64, 68
    g = torch.Generator().manual_seed(1)
    S = torch.randn(B * nq, ld, generator=g) * 3
    dP = torch.randn(B * nq, ld, generator=g)
    ops = _Ops(DEV, _cabi.OG_PREC_FP32)
    lens = torch.tensor(LENS, dtype=torch.int32, device=DEV)
    P = S.to(DEV)
    ops.softmax_rows(P, ld, B * nq, cols, klen=lens)
    dS = dP.to(DEV)
    ops.softmax_bwd_rows(P, dS, ld, B * nq, cols, 0.25, klen=lens)
    P, dS = P.cpu(), dS.cpu()
    for b, n in enumerate(LENS):
        r = slice(b * nq, (b + 1) * nq)
        s64 = S[r, :n].double().requires_grad_(True)
        p64 = torch.softmax(s64, -1)
        p64.backward(dP[r, :n].double())
        assert (P[r, :n].double() - p64).abs().max() < 1e-6
        assert (P[r, n:cols] == 0).all() and (dS[r, n:cols] == 0).all()
        assert (dS[r, :n].double() - 0.25 * s64.grad).abs().max() < 1e-5


def test_sinkhorn_with_history_and_backward_per_pair_against_the_trimmed_pair():
    N, M, iters, reg = 72, 64, 20, 1.0
    pairs = [(72, 64), (1, 30), (40, 1), (17, 59)]
    B = len(pairs)
    g = torch.Generator().manual_seed(2)
    lds = 64
    S = torch.randn(B, N, lds, generator=g)
    G = torch.randn(B, N + 1, M + 1, generator=g)
    ops = _Ops(DEV, _cabi.OG_PREC_FP32)
    lens = torch.tensor([p[0] for p in pairs] + [p[1] for p in pairs], dtype=torch.int32, device=DEV)
    dust = torch.tensor([0.7], device=DEV)
    Gp = G.clone()
    for b, (n, m) in enumerate(pairs):
        Gp[b, n + 1:] = float('nan')
        Gp[b, :, m + 1:] = float('nan')
    scores, hist = ops.sinkhorn_fwd(S.to(DEV), dust, B, N, M, iters, reg, lens=lens)
    dZ, dd = ops.sinkhorn_bwd(S.to(DEV), dust, hist, Gp.to(DEV), B, N, M, iters, reg, lens=lens)
    scores, dZ = scores.cpu(), dZ.cpu()
    dd_ref = 0.0
    for b, (n, m) in enumerate(pairs):
        lp = max(4, (m + 3) // 4 * 4)
        Sb = torch.zeros(1, n, lp)
        Sb[0, :, :m] = S[b, :n, :m]
        s1, h1 = ops.sinkhorn_fwd(Sb.to(DEV), dust, 1, n, m, iters, reg)
        Gb = G[b:b + 1, :n + 1, :m + 1].contiguous()
        z1, d1 = ops.sinkhorn_bwd(Sb.to(DEV), dust, h1, Gb.to(DEV), 1, n, m, iters, reg)
        assert (scores[b, :n + 1, :m + 1] - s1.cpu()[0]).abs().max() < 1e-4, b
        blk = scores[b].clone()
        blk[:n + 1, :m + 1] = -float('inf')
        assert torch.isneginf(blk).all()
        assert (dZ[b, :n + 1, :m + 1] - z1.cpu()[0]).abs().max() < 1e-4, b
        rest = dZ[b].clone()
        rest[:n + 1, :m + 1] = 0
        assert (rest == 0).all()
        dd_ref += float(d1)
    assert abs(float(dd) - dd_ref) <= 1e-4 * max(1.0, abs(dd_ref))


def test_criterion_with_lengths_is_the_mean_of_the_trimmed_pairs():
    pairs = [(30, 20), (1, 25), (32, 1)]
    N, M = 32, 25
    B = len(pairs)
    g = torch.Generator().manual_seed(3)
    scores = torch.randn(B, N + 1, M + 1, generator=g)
    gt0, gt1 = torch.randint(-2, M, (B, N), generator=g), torch.randint(-2, N, (B, M), generator=g)
    y = {'gt_matches0': gt0.to(DEV), 'gt_matches1': gt1.to(DEV), 'num_keypoints0': torch.tensor([p[0] for p in pairs]),
         'num_keypoints1': torch.tensor([p[1] for p in pairs])}
    sp = scores.clone()
    for b, (n, m) in enumerate(pairs):
        sp[b, n + 1:] = float('nan')
        sp[b, :, m + 1:] = float('nan')
        y['gt_matches0'][b, :n].clamp_(max=m - 1)
        y['gt_matches1'][b, :m].clamp_(max=n - 1)
    loss, ds = criterion_with_grad(y, {'scores': sp.to(DEV)})
    ds = ds.cpu()
    ref = 0.0
    for b, (n, m) in enumerate(pairs):
        yb = {'gt_matches0': y['gt_matches0'][b:b + 1, :n], 'gt_matches1': y['gt_matches1'][b:b + 1, :m]}
        lb, db = criterion_with_grad(yb, {'scores': scores[b:b + 1, :n + 1, :m + 1].to(DEV)})
        ref += float(lb['loss'])
        assert torch.allclose(ds[b, :n + 1, :m + 1] * B, db.cpu()[0], rtol=1e-6, atol=0), b
        rest = ds[b].clone()
        rest[:n + 1, :m + 1] = 0
        assert (rest == 0).all()
    assert abs(float(loss['loss']) - ref / B) <= 1e-6 * max(1.0, abs(ref))
    with pytest.raises(NotImplementedError):
        criterion(y, {'scores': sp.to(DEV), 'context_descriptors0': torch.zeros(B, 4, N, device=DEV),
                      'context_descriptors1': torch.zeros(B, 4, M, device=DEV)}, margin=0.5)


@pytest.mark.parametrize('kind', ['perspective', '3d_keypoint', '3d_image'])
def test_labels_with_lengths_are_the_labels_of_the_trimmed_pairs(kind):
    pairs = [(50, 40), (1, 40), (64, 3)]
    N, M = 64, 40
    B = len(pairs)
    g = torch.Generator().manual_seed(4)
    k0 = (torch.rand(B, N, 2, generator=g) * 100).round()
    k1 = (torch.rand(B, M, 2, generator=g) * 100).round()
    if kind == 'perspective':
        tf = {'type': [kind] * B, 'H': torch.eye(3).repeat(B, 1, 1) + 0.01 * torch.randn(B, 3, 3, generator=g)}
    else:
        K = torch.tensor([[100., 0, 50], [0, 100., 50], [0, 0, 1]]).repeat(B, 1, 1)
        R = torch.eye(3).repeat(B, 1, 1)
        T = torch.tensor([0.05, 0.0, 0.0]).repeat(B, 1)
        if kind == '3d_keypoint':
            d0, d1 = torch.rand(B, N, generator=g) + 1, torch.rand(B, M, generator=g) + 1
            d0[:, ::7] = 0.0
        else:
            d0, d1 = torch.rand(B, 101, 101, generator=g) + 1, torch.rand(B, 101, 101, generator=g) + 1
            d0[:, ::5] = 0.0
        tf = {'type': ['3d_reprojection'] * B, 'K0': K, 'K1': K, 'R': R, 'T': T, 'depth0': d0, 'depth1': d1}
    lens = torch.tensor([p[0] for p in pairs] + [p[1] for p in pairs], dtype=torch.int32, device=DEV)
    kp0, kp1 = k0.clone(), k1.clone()
    for b, (n, m) in enumerate(pairs):
        kp0[b, n:] = float('nan')
        kp1[b, m:] = float('nan')
    g0, g1 = gt_matches(kp0.to(DEV), kp1.to(DEV), tf, lens)
    g0, g1 = g0.cpu(), g1.cpu()
    for b, (n, m) in enumerate(pairs):
        tb = {k: (v[b:b + 1] if torch.is_tensor(v) else v[:1]) for k, v in tf.items()}
        if kind == '3d_keypoint':
            tb['depth0'], tb['depth1'] = tf['depth0'][b:b + 1, :n], tf['depth1'][b:b + 1, :m]
        r0, r1 = gt_matches(k0[b:b + 1, :n].to(DEV), k1[b:b + 1, :m].to(DEV), tb)
        assert torch.equal(g0[b, :n], r0.cpu()[0]) and torch.equal(g1[b, :m], r1.cpu()[0]), b
        assert (g0[b, n:] == IGNORE_INDEX).all() and (g1[b, m:] == IGNORE_INDEX).all()
