"""Training from images on the H100: ImagePairTrainStep (graph-replayed and eager) against the hand-wired eager chain
(extract_padded -> prepare_features_output -> generate_gt_matches -> TrainStep -> criterion_with_grad -> backward ->
ClippedAdam.step) bit for bit, against the extract_batch + pad_features + GraphedTrainStep path, homography pretraining against
the eager synthesis, one step against the unmodified reference and torch's optimiser, and the skip of batches the reference
skips (or BatchNorm1d refuses), decided on the device."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'oracle'))

from gen_golden_superpoint import synthetic_images, synthetic_superpoint_bn_state_dict, synthetic_superpoint_state_dict  # noqa: E402
from test_image_matching import _textures  # noqa: E402
from test_training_reference import _Check, _reference_class  # noqa: E402
from openglue_b200 import (ImagePairTrainStep, OpenCVSIFT, SuperGlue, SuperPointNet, SuperPointNetBn, _cabi,  # noqa: E402
                           synthesize_homography_pairs)
from openglue_b200._ops import _Ops  # noqa: E402
from openglue_b200.features import get_laf_to_sideinfo_converter, pad_features, prepare_features_output  # noqa: E402
from openglue_b200.gt_matches import generate_gt_matches  # noqa: E402
from openglue_b200.losses import criterion_with_grad  # noqa: E402
from openglue_b200.optim import ClippedAdam  # noqa: E402
from openglue_b200.synthetic import default_config, synthetic_state_dict  # noqa: E402
from openglue_b200.training import GraphedTrainStep, TrainStep  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
CONFIG = {'superglue': {'laf_to_sideinfo_method': 'none', 'log_transform_response': False},
          'train': {'gt_positive_threshold': 2, 'gt_negative_threshold': 7, 'margin': None, 'nll_weight': 1.0, 'metric_weight': 0.0,
                    'augmentations': {'name': 'none'}, 'lr': 1e-3, 'grad_clip': 10.0, 'scheduler_gamma': 0.99}}
OUT_KEYS = ImagePairTrainStep._OUT_KEYS


# --------------------------------------------------------------------------- helpers
def _frontend(name, maxk=None):
    if name == 'sift':
        return OpenCVSIFT(max_keypoints=maxk or 400), 128
    cls = SuperPointNet if name == 'superpoint' else SuperPointNetBn
    sp = cls(max_keypoints=maxk or 2048, keypoint_threshold=0.01)
    sp.load_state_dict(synthetic_superpoint_bn_state_dict(7) if cls is SuperPointNetBn else synthetic_superpoint_state_dict(7), strict=True)
    return sp.to(DEV).eval(), 256


def _superglue(d, seed=9):
    cfg = default_config(descriptor_dim=d, num_heads=4, num_stages=2, num_iters=20)
    cfg['precision'] = 'tf32x3'
    m = SuperGlue(cfg)
    m.load_state_dict(synthetic_state_dict(cfg, seed=seed), strict=True)
    return m.to(DEV).train()


def _trainer(d, optimizer=True):
    m = _superglue(d)
    return m, (ClippedAdam.from_config(m, CONFIG['train']) if optimizer else None)


def _pair_images(frontend, B, seed):
    """240 x 320 pairs, image1 = image0 moved by (-9, -12) px; textures whose keypoint counts differ per image"""
    if frontend == 'sift':
        base = _textures(B, 256, 336, seed)
    else:
        base = synthetic_images(B, 256, 336, seed).to(DEV)
        base[1 % B, :, :, :168] = 0.5                                           # fewer keypoints in two images
        base[2 % B, :, :, 88:] = 0.5
    return base[:, :, :240, :320].contiguous(), base[:, :, 12:252, 9:329].contiguous()


def _transformation(kind, B, h=240, w=320):
    if kind == 'perspective':
        H = torch.tensor([[1., 0., -9.], [0., 1., -12.], [0., 0., 1.]])
        return {'type': ['perspective'] * B, 'H': H.expand(B, 3, 3).contiguous().to(DEV)}
    K = torch.tensor([[300., 0., 160.], [0., 300., 120.], [0., 0., 1.]]).expand(B, 3, 3).contiguous().to(DEV)
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing='ij')
    depth = (10 + torch.sin(xx / 50) + 0.5 * torch.cos(yy / 30)).expand(B, h, w).contiguous().to(DEV)
    return {'type': ['3d_reprojection'] * B, 'K0': K, 'K1': K.clone(), 'R': torch.eye(3).expand(B, 3, 3).contiguous().to(DEV),
            'T': torch.tensor([-0.3, -0.4, 0.0]).expand(B, 3).contiguous().to(DEV), 'depth0': depth, 'depth1': depth.clone()}


def _batch(frontend, B, seed, kind='perspective'):
    i0, i1 = _pair_images(frontend, B, seed)
    return {'image0': i0, 'image1': i1, 'transformation': _transformation(kind, B)}


def _rgb(B, H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    low = torch.rand(B, 3, H // 12, W // 12, generator=g, device=DEV)
    imgs = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False).clamp(0, 1) * 255
    return imgs.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _hand_wired(fe, model, opt, batch, K):
    """the training step wired by hand from the public pieces, eagerly"""
    raw = dict(batch)
    conv = get_laf_to_sideinfo_converter('none')
    feats = []
    for i in (0, 1):
        lafs, resp, desc, n, _ = fe.extract_padded(batch[f'image{i}'], K)
        feats.append(prepare_features_output(lafs, resp, desc, conv))
        raw[f'num_keypoints{i}'] = n
    data, y = generate_gt_matches(raw, feats[0], feats[1], 2, 7)
    st = TrainStep(model, data)
    scores, _, _ = st.forward()
    loss, ds = criterion_with_grad(y, {'scores': scores})
    g = st.backward(ds)
    for k, p in model.named_parameters():
        p.grad = g[k].reshape(p.shape).clone()
    if opt is not None:
        opt.step()
    return loss['loss']


def _state(model, opt):
    """parameters, BatchNorm buffers and the optimiser's moments, step counts, lr and scheduler count"""
    t = [p.detach() for p in model.parameters()] + list(model.buffers())
    if opt is not None:
        t += opt._exp_avg + opt._exp_avg_sq + [opt._steps, opt._state]
    return [x.clone() for x in t]


def _same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i


# --------------------------------------------------------------------------- 1. replay == eager == hand-wired chain
@pytest.mark.parametrize('kind', ['perspective', '3d_reprojection'])
@pytest.mark.parametrize('frontend', ['sift', 'superpoint', 'superpoint_bn'])
def test_replay_equals_eager_and_the_hand_wired_chain(frontend, kind):
    fe, d = _frontend(frontend)
    K = fe.max_keypoints
    (m_h, o_h), (m_g, o_g), (m_e, o_e) = _trainer(d), _trainer(d), _trainer(d)
    graphed = ImagePairTrainStep(fe, m_g, CONFIG, optimizer=o_g)
    eager = ImagePairTrainStep(fe, m_e, CONFIG, optimizer=o_e, use_cuda_graph=False)
    counts = set()
    for j in range(3):
        batch = _batch(frontend, 3, 40 + j, kind)
        want = _hand_wired(fe, m_h, o_h, batch, K)
        got, ge = graphed(batch), eager(batch)
        torch.cuda.synchronize()
        assert int(got['skipped']) == 0 and torch.isfinite(want)
        assert torch.equal(got['loss'], want) and torch.equal(ge['loss'], want), j
        assert float(got['metric_loss']) == 0.0
        for k in OUT_KEYS:
            assert torch.equal(got[k], ge[k]), (j, k)
        counts |= set(got['num_keypoints0'].tolist() + got['num_keypoints1'].tolist())
        ref = _state(m_h, o_h)
        _same(ref, _state(m_g, o_g))
        _same(ref, _state(m_e, o_e))
    assert len(counts) > 1, counts                                              # the batches really are padded
    assert o_g.state_dict()['lr_scheduler']['last_epoch'] == 3


def test_sift_replay_equals_the_extract_batch_path():
    """with no overflow, a replay is test_padded_training's end-to-end path: extract_batch + pad_features + GraphedTrainStep"""
    fe, K = OpenCVSIFT(max_keypoints=400), 400
    (m_r, o_r), (m_g, o_g) = _trainer(128), _trainer(128)
    step = ImagePairTrainStep(fe, m_g, CONFIG, optimizer=o_g)
    conv = get_laf_to_sideinfo_converter('none')
    graphed = None
    for j in range(3):
        batch = _batch('sift', 3, 50 + j)
        raw = dict(batch)
        feats = []
        for i in (0, 1):
            lafs, resp, desc, n = pad_features(fe.extract_batch(batch[f'image{i}']), K)
            feats.append(prepare_features_output(lafs, resp, desc, conv))
            raw[f'num_keypoints{i}'] = n
        data, y = generate_gt_matches(raw, feats[0], feats[1], 2, 7)
        if graphed is None:
            graphed = GraphedTrainStep(m_r, data, y, optimizer=o_r)
        want = graphed(data, y)['loss']
        got = step(batch)
        torch.cuda.synchronize()
        assert got['overflow0'].tolist() == [0] * 3 and got['overflow1'].tolist() == [0] * 3
        assert got['num_keypoints0'].tolist() == raw['num_keypoints0'].tolist()
        assert torch.equal(got['loss'], want), j
        _same(_state(m_r, o_r), _state(m_g, o_g))


# --------------------------------------------------------------------------- 2. homography pretraining
@pytest.mark.parametrize('frontend', ['sift', 'superpoint'])
def test_pretrain_equals_the_eager_synthesis_and_step(frontend):
    fe, d = _frontend(frontend)
    imgs = _rgb(3, 288, 368, 11)                                                # 240 x 320 pairs at offset 24
    (m_g, o_g), (m_e, o_e) = _trainer(d), _trainer(d)
    step = ImagePairTrainStep(fe, m_g, CONFIG, optimizer=o_g)
    eager = ImagePairTrainStep(fe, m_e, CONFIG, optimizer=o_e, use_cuda_graph=False)
    offsets = []
    for j in range(3):
        got = step.pretrain(imgs, 24)
        pairs = synthesize_homography_pairs(imgs, 24, warp_offset=got['warp_offset'])
        want = eager(pairs)
        torch.cuda.synchronize()
        assert int(got['skipped']) == 0 and torch.isfinite(got['loss'])
        assert torch.equal(got['loss'], want['loss']), j
        _same(_state(m_e, o_e), _state(m_g, o_g))
        w = got['warp_offset']
        assert w.shape == (3, 4, 2) and w.dtype == torch.int32 and int(w.min()) >= -24 and int(w.max()) < 24
        offsets.append(w)
    assert not torch.equal(offsets[0], offsets[1]) and not torch.equal(offsets[1], offsets[2])


def test_pretrain_offsets_follow_the_seed():
    imgs = _rgb(2, 288, 368, 12)
    runs = []
    for _ in range(2):
        torch.cuda.manual_seed(1234)
        step = ImagePairTrainStep(OpenCVSIFT(max_keypoints=200), _superglue(128), CONFIG)
        runs.append([step.pretrain(imgs, 24)['warp_offset'] for _ in range(3)])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# --------------------------------------------------------------------------- 3. against the reference and torch's optimiser
def test_one_step_against_the_reference_and_torch_adam():
    """Every image reaches K keypoints, so padding and the reference's min_stack agree.  Loss and gradients against the unmodified
    reference's train-mode forward + criterion + autograd on the step's own front-end outputs (float64 and float32, the bound of
    the training-reference tests); the update against clip_grad_norm_ + Adam + StepLR on those gradients."""
    SG = _reference_class(True)
    from oracle.build_ref import import_reference
    _, ref_criterion, ref_gt = import_reference()
    fe, K = OpenCVSIFT(max_keypoints=40), 40
    batch = _batch('sift', 2, 70)
    m, _ = _trainer(128, optimizer=False)
    sd0 = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    out = ImagePairTrainStep(fe, m, CONFIG)(batch)
    torch.cuda.synchronize()
    assert out['num_keypoints0'].tolist() == [K, K] and out['num_keypoints1'].tolist() == [K, K] and int(out['skipped']) == 0
    grads = {k: p.grad.detach().cpu().double() for k, p in m.named_parameters()}
    conv = get_laf_to_sideinfo_converter('none')
    feats = [prepare_features_output(*fe.extract_padded(batch[f'image{i}'], K)[:3], conv) for i in (0, 1)]
    cpu = {'image0': batch['image0'].cpu().float(), 'image1': batch['image1'].cpu().float(),
           'transformation': {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in batch['transformation'].items()}}
    f32 = [{k: v.cpu() for k, v in f.items()} for f in feats]
    data, y = ref_gt(cpu, f32[0], f32[1], 2, 7)
    ref = {}
    for dtype in (torch.float64, torch.float32):
        model = SG(copy.deepcopy(m.config))
        model.load_state_dict(sd0, strict=True)
        model = model.to(dtype).train()
        d = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in data.items()}
        loss = ref_criterion(y, model(d), margin=None)['loss']
        loss.backward()
        ref[dtype] = (loss.detach().double(), {k: p.grad.detach().double() for k, p in model.named_parameters()})
    chk = _Check('[image step vs reference]')
    chk('loss', out['loss'].cpu().reshape(1), ref[torch.float64][0].reshape(1), ref[torch.float32][0].reshape(1))
    for k, g in grads.items():
        chk(f'grad {k}', g, ref[torch.float64][1][k], ref[torch.float32][1][k])
    chk.done()
    # the update: ClippedAdam in the graph against torch on the same gradients
    m2, o2 = _trainer(128)
    ImagePairTrainStep(fe, m2, CONFIG, optimizer=o2)(batch)
    tp = [sd0[k].to(DEV).clone().requires_grad_(True) for k, _ in m2.named_parameters()]
    for p, (k, _) in zip(tp, m2.named_parameters()):
        p.grad = grads[k].float().to(DEV)
    adam = torch.optim.Adam(tp, lr=CONFIG['train']['lr'])
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=CONFIG['train']['scheduler_gamma'])
    norm = torch.nn.utils.clip_grad_norm_(tp, CONFIG['train']['grad_clip'])
    adam.step()
    sched.step()
    torch.cuda.synchronize()
    assert abs(float(o2.last_grad_norm) - float(norm)) <= 1e-6 * float(norm)
    for p, (k, q) in zip(tp, m2.named_parameters()):
        assert torch.allclose(q, p, rtol=0, atol=1e-6), k
    assert o2.get_last_lr() == sched.get_last_lr()


# --------------------------------------------------------------------------- 4. the skip
def _check_skipped(out, model, opt, before):
    torch.cuda.synchronize()
    assert int(out['skipped']) == 1
    assert torch.isnan(out['loss']) and torch.isnan(out['metric_loss'])
    _same(before, _state(model, opt))
    for k, p in model.named_parameters():
        assert p.grad is not None and not p.grad.any(), k


@pytest.mark.parametrize('graph', [True, False])
def test_a_constant_image_skips_the_step(graph):
    """SIFT finds no keypoint on a constant image (the synthetic SuperPoint weights respond to the zero padding at its borders,
    so SuperPoint's skip is tested with one keypoint per side below)"""
    frontend = 'sift'
    fe, d = _frontend(frontend)
    (m, o), (m_f, o_f) = _trainer(d), _trainer(d)
    step = ImagePairTrainStep(fe, m, CONFIG, optimizer=o, use_cuda_graph=graph)
    batch = _batch(frontend, 3, 60)
    flat = batch['image1'].clone()
    flat[1] = 128 if flat.dtype == torch.uint8 else 0.5
    before = _state(m, o)
    out = step({**batch, 'image1': flat})
    assert out['num_keypoints1'].tolist()[1] == 0 and out['num_keypoints0'].tolist()[1] > 0
    _check_skipped(out, m, o, before)
    sd, torch_sd = o.state_dict(), torch.optim.Adam(m.parameters(), lr=CONFIG['train']['lr']).state_dict()
    assert sd['optimizer']['state'] == torch_sd['state'] == {}
    assert sd['optimizer']['param_groups'][0]['lr'] == CONFIG['train']['lr'] and sd['lr_scheduler']['last_epoch'] == 0
    # the next batch: what a step object that never saw the skipped batch gives
    fresh = ImagePairTrainStep(fe, m_f, CONFIG, optimizer=o_f, use_cuda_graph=graph)
    a, b = step(batch), fresh(batch)
    torch.cuda.synchronize()
    assert int(a['skipped']) == 0 and torch.isfinite(a['loss']) and torch.equal(a['loss'], b['loss'])
    _same(_state(m, o), _state(m_f, o_f))
    sd = o.state_dict()
    assert len(sd['optimizer']['state']) == len(list(m.parameters())) and sd['lr_scheduler']['last_epoch'] == 1


@pytest.mark.parametrize('optimizer', [True, False])
@pytest.mark.parametrize('frontend', ['sift', 'superpoint'])
def test_one_keypoint_per_side_skips_the_step(frontend, optimizer):
    """B = 1 with one keypoint per side: the one value per channel BatchNorm1d raises on"""
    fe, d = _frontend(frontend, maxk=1)
    m, o = _trainer(d, optimizer)
    batch = _batch(frontend, 1, 61)
    for graph in (False, True):
        step = ImagePairTrainStep(fe, m, CONFIG, optimizer=o, use_cuda_graph=graph)
        before = _state(m, o)
        out = step(batch)
        assert out['num_keypoints0'].tolist() == [1] and out['num_keypoints1'].tolist() == [1]
        _check_skipped(out, m, o, before)
        for _, p in m.named_parameters():                                       # the next step computes on real gradients
            p.grad.fill_(1.0)


def test_guard_flags():
    lib = _cabi.lib()
    cases = [([3, 4], [5, 6], 0), ([0, 4], [5, 6], 1), ([3, 4], [5, 0], 1), ([1], [1], 1), ([1], [2], 1), ([2], [2], 0),
             ([1, 1], [1, 1], 0), ([2, 0, 5], [3, 3, 3], 1), (list(range(1, 80)), list(range(2, 81)), 0)]
    for n, m_, want in cases:
        lens = torch.tensor(n + m_, dtype=torch.int32, device=DEV)
        skip = torch.full((), 7, dtype=torch.int32, device=DEV)
        _cabi.check(lib.og_train_guard(_cabi.ptr(lens), len(n), _cabi.ptr(skip), _cabi.stream(DEV)), 'og_train_guard')
        assert int(skip) == want, (n, m_)


@pytest.mark.parametrize('padded', [False, True])
def test_guarded_batchnorm_equals_the_existing_entry_points(padded):
    ops = _Ops(torch.device(DEV), _cabi.OG_PREC_TF32X3)
    g = torch.Generator(device=DEV).manual_seed(3)
    B, cap, cols = 3, 50, 64
    a = torch.randn(B * cap, cols, generator=g, device=DEV)
    gamma, beta = torch.rand(cols, generator=g, device=DEV) + 0.5, torch.randn(cols, generator=g, device=DEV)
    rm0, rv0 = torch.randn(cols, generator=g, device=DEV), torch.rand(cols, generator=g, device=DEV) + 0.5
    lens = torch.tensor([50, 7, 31], dtype=torch.int32, device=DEV) if padded else None
    lk = {'lens': lens} if padded else {}

    def run(flag):
        rm, rv = rm0.clone(), rv0.clone()
        nbt = torch.full((), 5, dtype=torch.int64, device=DEV)
        if flag == 'existing':
            y, mu, inv = ops.bn_fwd(a, gamma, beta, 1e-5, 0.1, rm, rv, **lk)
        elif flag == 'null':
            y, mu, inv = ops.empty(B * cap, cols), ops.empty(cols), ops.empty(cols)
            nb, c = (B, cap) if padded else (1, B * cap)
            _cabi.check(ops.lib.og_bn_train_fwd_guarded(_cabi.ptr(a), cols, nb, c, _cabi.ptr(lens), cols, 1, _cabi.ptr(gamma), _cabi.ptr(beta),
                                                        1e-5, 0.1, _cabi.ptr(y), cols, _cabi.ptr(mu), _cabi.ptr(inv), _cabi.ptr(rm),
                                                        _cabi.ptr(rv), None, _cabi.ptr(nbt), _cabi.ptr(ops.ws(cols)), ops.st()),
                        'og_bn_train_fwd_guarded')
        else:
            skip = torch.full((), flag, dtype=torch.int32, device=DEV)
            y, mu, inv = ops.bn_fwd(a, gamma, beta, 1e-5, 0.1, rm, rv, skip=skip, num_batches_tracked=nbt, **lk)
        torch.cuda.synchronize()
        return [y, mu, inv, rm, rv], int(nbt)
    ref, _ = run('existing')
    for flag in ('null', 0):
        got, nbt = run(flag)
        _same(ref, got)
        assert nbt == 6
    got, nbt = run(1)
    _same(ref[:3], got[:3])                                                     # the outputs either way
    _same([rm0, rv0], got[3:])                                                  # the running statistics stay
    assert nbt == 5


def test_guarded_optimiser_step_equals_the_existing_one():
    g = torch.Generator(device=DEV).manual_seed(5)
    shapes = [(300, 7), (129,), (4, 4, 3)]
    init = [torch.randn(*s, generator=g, device=DEV) for s in shapes]
    sets = [[torch.nn.Parameter(t.clone()) for t in init] for _ in range(3)]
    opts = [ClippedAdam(ps, lr=1e-2, grad_clip=1.0, lr_gamma=0.9) for ps in sets]
    zero, one = torch.zeros((), dtype=torch.int32, device=DEV), torch.ones((), dtype=torch.int32, device=DEV)
    for step in range(3):
        grads = [torch.randn(*s, generator=g, device=DEV) * (step + 1) for s in shapes]
        for ps in sets:
            for p, gr in zip(ps, grads):
                p.grad = gr.clone()
        before = [p.detach().clone() for p in sets[2]] + opts[2]._exp_avg + opts[2]._exp_avg_sq + [opts[2]._steps, opts[2]._state]
        before = [t.clone() for t in before]
        opts[0].step()
        opts[1].step(skip=zero)
        opts[2].step(skip=one)
        torch.cuda.synchronize()
        full = [[p.detach() for p in sets[i]] + [p.grad for p in sets[i]] + opts[i]._exp_avg + opts[i]._exp_avg_sq +
                [opts[i]._steps, opts[i]._state] for i in range(2)]
        _same(full[0], full[1])
        _same(before, [p.detach() for p in sets[2]] + opts[2]._exp_avg + opts[2]._exp_avg_sq + [opts[2]._steps, opts[2]._state])
        assert all(not p.grad.any() for p in sets[2])
    assert opts[2].state_dict()['optimizer']['state'] == {} and opts[2].state_dict()['lr_scheduler']['last_epoch'] == 0
    sd0, sd1 = opts[0].state_dict(), opts[1].state_dict()
    assert len(sd1['optimizer']['state']) == 3 and sd1['lr_scheduler'] == sd0['lr_scheduler']
    with pytest.raises(ValueError, match='int32'):
        opts[0].step(skip=torch.zeros((), dtype=torch.int64, device=DEV))


# --------------------------------------------------------------------------- 5. graphs: no host synchronisation, cache rules
def test_graph_cache_and_no_host_synchronisation(monkeypatch):
    captured = [0]
    orig = torch.cuda.CUDAGraph.capture_end

    def counting(self):
        captured[0] += 1
        return orig(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'capture_end', counting)
    fe = OpenCVSIFT(max_keypoints=300)
    m, o = _trainer(128)
    step = ImagePairTrainStep(fe, m, CONFIG, optimizer=o)
    b3, b2, rgb = _batch('sift', 3, 80), _batch('sift', 2, 81), _rgb(3, 288, 368, 3)
    step(b3)
    step.pretrain(rgb, 24)
    torch.cuda.synchronize()
    assert captured[0] == 2
    torch.cuda.set_sync_debug_mode('error')
    try:
        outs = [step(b3), step(b3, borrow=True), step.pretrain(rgb, 24)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert captured[0] == 2 and all(int(x['skipped']) == 0 for x in outs)
    assert outs[1]['loss'] is step(b3, borrow=True)['loss']                     # the graph's own buffers
    step(b2)                                                                    # a new shape
    assert captured[0] == 3
    step(b3)
    assert captured[0] == 3
    p = next(m.parameters())
    p.data = p.data.clone()                                                     # reallocated weights
    step(b3)
    assert captured[0] == 4
    step.max_graphs = 1
    step(b2)
    step(b3)
    assert len(step._graphs) == 1 and captured[0] == 6


def test_overflow_is_reported_and_trains_on_the_first_K_rows():
    fe, K = OpenCVSIFT(max_keypoints=400), 120                                   # capacity below max_keypoints
    (m_h, o_h), (m_g, o_g) = _trainer(128), _trainer(128)
    step = ImagePairTrainStep(fe, m_g, CONFIG, optimizer=o_g, capacity=K)
    batch = _batch('sift', 3, 90)
    singles = [fe.extract_batch(batch[f'image{i}']) for i in (0, 1)]
    out = step(batch)
    want = _hand_wired(fe, m_h, o_h, batch, K)
    torch.cuda.synchronize()
    for i in (0, 1):
        n = [s[0].shape[1] for s in singles[i]]
        assert out[f'overflow{i}'].tolist() == [int(x > K) for x in n]
        assert out[f'num_keypoints{i}'].tolist() == [min(x, K) for x in n]
    assert sum(out['overflow0'].tolist()) > 0
    assert torch.equal(out['loss'], want)
    _same(_state(m_h, o_h), _state(m_g, o_g))
