"""ClippedAdam (openglue_b200/optim.py, og_clip_adam_step): the reference's clip_grad_norm_ -> Adam -> StepLR step on the GPU,
against torch's own objects (foreach Adam on CUDA, as Lightning runs it)."""
import copy
import ctypes as C
import math

import numpy as np
import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200.optim import ClippedAdam, _torch_pair, _torch_state_dicts

LR, GAMMA, CLIP = 1e-4, 0.999994, 10.0

# the train: sections of the reference's shipped configs (config/*.yaml), restated
SHIPPED_TRAIN = {
    'config.yaml': {'lr': 1.0e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994},
    'config_cached.yaml': {'lr': 1.0e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994},
    'config_cached_sp_magicleap.yaml': {'lr': 1.0e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994},
    'homography_pretraining.yaml': {'lr': 1.0e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994},
}


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize('kw', [dict(weight_decay=0.01), dict(amsgrad=True), dict(maximize=True)])
def test_rejects_options_the_reference_never_sets(kw):
    with pytest.raises(NotImplementedError):
        ClippedAdam([torch.zeros(3)], **kw)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_rejects_cpu_parameters(dtype):
    with pytest.raises(ValueError, match='CUDA'):
        ClippedAdam([torch.nn.Parameter(torch.zeros(3, dtype=dtype))])


def test_rejects_several_groups_and_bad_hyper_parameters():
    with pytest.raises(ValueError, match='one parameter group'):
        ClippedAdam([{'params': [torch.zeros(2)]}, {'params': [torch.zeros(3)]}])
    for kw in (dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(grad_clip=0.0), dict(eps=-1.0), dict(lr_gamma=0.0)):
        with pytest.raises(ValueError):
            ClippedAdam([torch.zeros(3)], **kw)


def test_abi_rejects_bad_arguments_without_cuda():
    lib = _cabi.lib()
    assert lib.og_optim_state_bytes() == 24
    assert lib.og_optim_workspace_bytes(0) == -1 and lib.og_optim_workspace_bytes(-3) == -1
    ws_bytes = lib.og_optim_workspace_bytes(4)
    assert ws_bytes > 0
    fake = C.c_void_p(4096)                      # never dereferenced: every call below fails validation first
    good = dict(segs=fake, nseg=4, ntiles=4, b1=0.9, b2=0.999, eps=1e-8, clip=10.0, gamma=GAMMA, state=fake, ws=fake, wsb=ws_bytes)

    def call(**over):
        a = dict(good, **over)
        return lib.og_clip_adam_step(a['segs'], a['nseg'], a['ntiles'], a['b1'], a['b2'], a['eps'], a['clip'], a['gamma'], a['state'],
                                     a['ws'], a['wsb'], None)
    for over in (dict(segs=None), dict(state=None), dict(ws=None), dict(nseg=0), dict(ntiles=0), dict(clip=0.0), dict(clip=-1.0),
                 dict(b1=1.0), dict(b2=-0.5), dict(eps=-1e-8), dict(gamma=0.0)):
        assert call(**over) == -1, over          # OG_EINVAL
    assert call(wsb=ws_bytes - 1) == -4          # OG_EWORKSPACE
    out = C.c_void_p(4096)
    assert lib.og_adam_schedule(0, LR, GAMMA, 0.9, 0.999, out, out, out, None) == -1
    assert lib.og_adam_schedule(10, LR, GAMMA, 0.9, 0.999, None, out, out, None) == -1


def _layout(x):
    """key sets, value types and tensor dtypes / devices of a (nested) state dict"""
    if isinstance(x, dict):
        return {k: _layout(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return (type(x).__name__, [_layout(v) for v in x])
    if torch.is_tensor(x):
        return ('tensor', x.dtype, x.device.type, tuple(x.shape))
    return type(x).__name__


def test_state_dict_layout_equals_torch_adam_and_steplr():
    """The checkpoint dicts ClippedAdam writes have exactly the keys, value types and dtypes of torch's Adam + StepLR."""
    shapes = [(4, 3), (1,), (7,)]
    params = [torch.nn.Parameter(torch.randn(s)) for s in shapes]
    adam = torch.optim.Adam(params, lr=LR)
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=GAMMA)
    for p in params:
        p.grad = torch.randn_like(p)
    adam.step()
    sched.step()
    ref = {'optimizer': adam.state_dict(), 'lr_scheduler': sched.state_dict()}
    twins = [torch.nn.Parameter(torch.randn(s)) for s in shapes]
    states = [{'step': torch.tensor(1.0), 'exp_avg': torch.zeros(s), 'exp_avg_sq': torch.zeros(s)} for s in shapes]
    ours = _torch_state_dicts(_torch_pair(twins, LR * GAMMA, LR, (0.9, 0.999), 1e-8, GAMMA), states, 1)
    assert _layout(ours) == _layout(ref)
    assert ours['lr_scheduler'] == ref['lr_scheduler']
    assert ours['optimizer']['param_groups'] == ref['optimizer']['param_groups']


@pytest.mark.parametrize('name', sorted(SHIPPED_TRAIN))
def test_from_config_reads_the_train_section(name):
    section = dict(SHIPPED_TRAIN[name], epochs=100, steps_per_epoch=10000, precision=32)
    assert ClippedAdam.config_kwargs(section) == {'lr': 1e-4, 'grad_clip': 10.0, 'lr_gamma': 0.999994}


# ------------------------------------------------------------------------------------------------------------ GPU
DEV = 'cuda:0'


def _torch_opt(params, lr=LR, gamma=GAMMA):
    adam = torch.optim.Adam(params, lr=lr)          # foreach on CUDA: Lightning's default Adam
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=gamma)

    def step():
        norm = torch.nn.utils.clip_grad_norm_(params, CLIP)
        adam.step()
        sched.step()
        return norm
    return adam, sched, step


def _grads(shapes, k, scale, dev=DEV):
    g = torch.Generator(device=dev).manual_seed(1000 + k)
    return [torch.randn(s, device=dev, generator=g) * scale for s in shapes]


def _assert_same(ours: ClippedAdam, pa, adam, sched, pb, what):
    """p, p.grad, exp_avg, exp_avg_sq, step and lr bit for bit (NaN where torch has NaN)"""
    eq = lambda a, b, k: torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True, msg=lambda m: f'{what} {k}: {m}')
    sd = ours.state_dict()['optimizer']
    for i, (p, q) in enumerate(zip(pa, pb)):
        eq(p.detach(), q.detach(), f'param {i}')
        if q.grad is None:
            assert p.grad is None
        else:
            eq(p.grad, q.grad, f'grad {i}')
        st = adam.state.get(q)
        if not st:
            assert i not in sd['state'], (what, i)
            continue
        for key in ('exp_avg', 'exp_avg_sq', 'step'):
            eq(sd['state'][i][key], st[key], f'{key} {i}')
    assert ours.get_last_lr() == sched.get_last_lr(), what


def _pair_of_params(shapes, seed=0):
    g = torch.Generator().manual_seed(seed)
    init = [torch.randn(s, generator=g) * 0.1 for s in shapes]
    a = [torch.nn.Parameter(t.to(DEV)) for t in init]
    b = [torch.nn.Parameter(t.to(DEV)) for t in init]
    return a, b


def _run_both(shapes, steps, scale, grad_none=()):
    pa, pb = _pair_of_params(shapes)
    ours = ClippedAdam(pa)
    adam, sched, tstep = _torch_opt(pb)
    for k in range(steps):
        gs = _grads(shapes, k, scale)
        for i, (p, q, g) in enumerate(zip(pa, pb, gs)):
            p.grad = None if i in grad_none else g.clone()
            q.grad = None if i in grad_none else g.clone()
        ours.step()
        norm = tstep()
        _assert_same(ours, pa, adam, sched, pb, f'step {k + 1}')
    return ours, norm


@pytest.mark.gpu
def test_device_scalars_equal_torch_over_a_whole_training_run():
    """Steps 1 .. 1,000,000 (100 epochs x 10,000 steps): the device's fp32 step_size / bc2_sqrt and float64 lr equal what
    torch's non-capturable Adam (torch/optim/adam.py: 1 - beta ** step, (lr / bc1) * -1, bc2 ** 0.5 with Python floats, then
    fp32 in the foreach kernels) and StepLR (lr * gamma per step) compute on the host."""
    n, b1, b2 = 1_000_000, 0.9, 0.999
    lr_d = torch.empty(n, dtype=torch.float64, device=DEV)
    ss_d = torch.empty(n, dtype=torch.float32, device=DEV)
    bc_d = torch.empty(n, dtype=torch.float32, device=DEV)
    _cabi.check(_cabi.lib().og_adam_schedule(n, LR, GAMMA, b1, b2, _cabi.ptr(lr_d), _cabi.ptr(ss_d), _cabi.ptr(bc_d),
                                             _cabi.stream()), 'og_adam_schedule')
    lrs, ss, bc = [], [], []
    lr = LR
    for k in range(1, n + 1):
        step = float(k)
        lrs.append(lr)
        ss.append((lr / (1 - b1 ** step)) * -1)
        bc.append((1 - b2 ** step) ** 0.5)
        lr = lr * GAMMA
    lr_h = np.array(lrs, dtype=np.float64)
    ss_h = np.array(ss, dtype=np.float64).astype(np.float32)
    bc_h = np.array(bc, dtype=np.float64).astype(np.float32)
    for name, dev_v, host_v in (('lr', lr_d, lr_h), ('step_size', ss_d, ss_h), ('bc2_sqrt', bc_d, bc_h)):
        d = dev_v.cpu().numpy()
        bad = np.nonzero(d != host_v)[0]
        assert bad.size == 0, f'{name}: {bad.size} steps differ, first at step {bad[0] + 1}: {d[bad[0]]!r} vs {host_v[bad[0]]!r}'


@pytest.mark.gpu
def test_unclipped_steps_on_the_default_model_are_bit_identical_to_torch():
    from openglue_b200 import SuperGlue
    from openglue_b200.synthetic import default_config
    model = SuperGlue(default_config())
    shapes = [tuple(p.shape) for p in model.parameters()]
    total = sum(math.prod(s) for s in shapes)
    assert total == 11_957_249
    ours, norm = _run_both(shapes, 20, 5.0 / math.sqrt(total))
    assert 0 < float(norm) < CLIP


@pytest.mark.gpu
def test_clipped_step_scales_by_torchs_coefficient_of_our_norm():
    shapes = [(256, 256), (256,), (1,), (3, 4097), (5,)]
    pa, pb = _pair_of_params(shapes)
    ours = ClippedAdam(pa)
    adam = torch.optim.Adam(pb, lr=LR)
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=GAMMA)
    for k in range(5):
        gs = _grads(shapes, k, 1.0)
        for p, g in zip(pa, gs):
            p.grad = g.clone()
        ours.step()
        norm = ours.last_grad_norm.clone()
        ref = torch.linalg.vector_norm(torch.cat([g.double().reshape(-1) for g in gs]))
        assert abs(float(norm) - float(ref)) <= 1e-6 * float(ref), (float(norm), float(ref))
        assert float(norm) > CLIP
        coef = torch.clamp(CLIP / (norm + 1e-6), max=1.0)          # clip_grad_norm_'s fp32 formula on our norm
        for q, g in zip(pb, gs):
            q.grad = g * coef
        adam.step()
        sched.step()
        _assert_same(ours, pa, adam, sched, pb, f'step {k + 1}')


@pytest.mark.gpu
@pytest.mark.parametrize('bad', [float('inf'), float('nan')])
def test_non_finite_gradients_follow_torch(bad):
    shapes = [(64, 33), (7,), (1,)]
    pa, pb = _pair_of_params(shapes)
    ours = ClippedAdam(pa)
    adam, sched, tstep = _torch_opt(pb)
    for k in range(2):
        gs = _grads(shapes, k, 0.01)
        if k == 1:
            gs[0][3, 5] = bad
        for p, q, g in zip(pa, pb, gs):
            p.grad, q.grad = g.clone(), g.clone()
        ours.step()
        tnorm = tstep()
        _assert_same(ours, pa, adam, sched, pb, f'{bad} step {k + 1}')
    if math.isnan(bad):
        assert all(torch.isnan(p).all() for p in pa)
    torch.testing.assert_close(ours.last_grad_norm, tnorm, rtol=0, atol=0, equal_nan=True)


@pytest.mark.gpu
def test_awkward_segments_are_bit_identical_to_torch():
    # sizes around the vector width and the tile, a grad=None parameter, > 1000 segments
    shapes = [(1,), (3,), (5,), (4097,), (2 ** 20 + 1,)] + [(i % 13 + 1,) for i in range(1100)]
    ours, norm = _run_both(shapes, 3, 0.005, grad_none=(2, 600))      # norm ~5: the unclipped regime
    assert float(norm) < CLIP
    sd = ours.state_dict()['optimizer']['state']
    assert 2 not in sd and 600 not in sd and float(sd[1]['step']) == 3.0


@pytest.mark.gpu
def test_unaligned_views_are_bit_identical_to_torch():
    """Parameters and gradients that are views at 4-byte offsets of one buffer: no 16-byte alignment, the scalar path."""
    sizes = [1, 3, 4097, 5, 70000]
    offs = np.cumsum([1] + [s + 1 for s in sizes[:-1]])
    total = int(offs[-1] + sizes[-1] + 1)
    g = torch.Generator(device=DEV).manual_seed(3)
    init = torch.randn(total, device=DEV, generator=g) * 0.1
    bufs = [init.clone(), init.clone()]
    pa = [torch.nn.Parameter(bufs[0][o:o + s]) for o, s in zip(offs, sizes)]
    pb = [torch.nn.Parameter(bufs[1][o:o + s]) for o, s in zip(offs, sizes)]
    assert all(p.data_ptr() % 16 != 0 for p in pa[:2])
    ours = ClippedAdam(pa)
    adam, sched, tstep = _torch_opt(pb)
    for k in range(3):
        gbuf = [torch.randn(total, device=DEV, generator=g) * 0.01 for _ in range(1)][0]
        ga, gb = gbuf.clone(), gbuf.clone()
        for p, q, o, s in zip(pa, pb, offs, sizes):
            p.grad, q.grad = ga[o:o + s], gb[o:o + s]
        ours.step()
        tstep()
        _assert_same(ours, pa, adam, sched, pb, f'step {k + 1}')
    assert torch.equal(bufs[0], bufs[1])


SHAPES_CK = [(128, 64), (64,), (1,), (3, 4097)]


def _feed(params, k):
    for p, g in zip(params, _grads(SHAPES_CK, k, 0.01)):
        p.grad = g


@pytest.mark.gpu
@pytest.mark.parametrize('direction', ['ours_to_torch', 'torch_to_ours'])
def test_checkpoint_round_trip_is_bit_identical_to_an_uninterrupted_run(direction):
    K, N = 3, 4
    pu, _ = _pair_of_params(SHAPES_CK)
    uninterrupted = ClippedAdam(pu)
    for k in range(K + N):
        _feed(pu, k)
        uninterrupted.step()
    pa, pb = _pair_of_params(SHAPES_CK)
    if direction == 'ours_to_torch':
        first = ClippedAdam(pa)
        for k in range(K):
            _feed(pa, k)
            first.step()
        sd = copy.deepcopy(first.state_dict())
        with torch.no_grad():
            for p, q in zip(pb, pa):
                p.copy_(q)
        adam, sched, tstep = _torch_opt(pb)
        adam.load_state_dict(sd['optimizer'])
        sched.load_state_dict(sd['lr_scheduler'])
        for k in range(K, K + N):
            _feed(pb, k)
            tstep()
        final, lr = pb, sched.get_last_lr()[0]
        states = [adam.state[p] for p in pb]
    else:
        adam, sched, tstep = _torch_opt(pb)
        for k in range(K):
            _feed(pb, k)
            tstep()
        sd = copy.deepcopy({'optimizer': adam.state_dict(), 'lr_scheduler': sched.state_dict()})
        with torch.no_grad():
            for p, q in zip(pa, pb):
                p.copy_(q)
        second = ClippedAdam(pa)
        second.load_state_dict(sd)
        for k in range(K, K + N):
            _feed(pa, k)
            second.step()
        final, lr = pa, second.get_last_lr()[0]
        states = [second.state_dict()['optimizer']['state'][i] for i in range(len(pa))]
    ref = uninterrupted.state_dict()['optimizer']['state']
    for i, p in enumerate(final):
        assert torch.equal(p.detach(), pu[i].detach()), i
        for key in ('exp_avg', 'exp_avg_sq', 'step'):
            assert torch.equal(states[i][key].cpu(), ref[i][key].cpu()), (i, key)
    assert lr == uninterrupted.get_last_lr()[0]


@pytest.mark.gpu
def test_step_captured_alone_in_a_cuda_graph_and_without_host_sync():
    shapes = [(300, 7), (9,), (1,)]
    pa, pb = _pair_of_params(shapes)
    ga = _grads(shapes, 0, 0.01)
    for p, g in zip(pa, ga):
        p.grad = g.clone()
    for q, g in zip(pb, ga):
        q.grad = g.clone()
    graphed, eager = ClippedAdam(pa), ClippedAdam(pb)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        graphed.step()                      # eager first step (uploads the segment table)
        eager.step()
        eager.step()                        # and a second one with an unchanged table
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.step()
    for it in range(3):
        graph.replay()
        if it > 0:
            eager.step()
    torch.autograd.graph.increment_version(pa)
    torch.cuda.synchronize()
    for p, q in zip(pa, pb):
        assert torch.equal(p, q) and torch.equal(p.grad, q.grad)
    sa, sb = graphed.state_dict()['optimizer']['state'], eager.state_dict()['optimizer']['state']
    for i in sa:
        for key in ('exp_avg', 'exp_avg_sq', 'step'):
            assert torch.equal(sa[i][key], sb[i][key]), (i, key)
    assert float(sa[0]['step']) == 4.0
    assert graphed.get_last_lr() == eager.get_last_lr()


@pytest.mark.gpu
def test_two_identical_runs_give_identical_norms_and_parameters():
    shapes = [(512, 300), (77,), (1,), (4097,)]
    runs = []
    for _ in range(2):
        pa, _ = _pair_of_params(shapes)
        opt = ClippedAdam(pa)
        norms = []
        for k in range(3):
            for p, g in zip(pa, _grads(shapes, k, 1.0)):
                p.grad = g
            opt.step()
            norms.append(opt.last_grad_norm.clone())
        runs.append((torch.stack(norms), [p.detach().clone() for p in pa]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['train_ragged', 'train_small'])
def test_graphed_iteration_with_the_optimiser_equals_the_eager_iteration(name):
    import os
    from openglue_b200 import SuperGlue, criterion
    from openglue_b200.synthetic import synthetic_state_dict
    from openglue_b200.training import GraphedTrainStep
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', name + '.pt'), weights_only=False)
    dev = torch.device(DEV)
    sd = synthetic_state_dict(fx['config'], seed=fx['weights_seed'])
    sd.update(fx['bn_buffers'])
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    y_true = {'gt_matches0': fx['gt_matches0'].to(dev), 'gt_matches1': fx['gt_matches1'].to(dev)}
    cfg = dict(fx['config'], precision='tf32x3')
    models = []
    for _ in range(2):
        m = SuperGlue(cfg)
        m.load_state_dict(copy.deepcopy(sd), strict=True)
        models.append(m.to(dev))
    eager, graphed = models
    graphed.eval()
    with torch.no_grad():
        graphed(data)                                    # packs the eval weights once: training must invalidate them
    eager.train(), graphed.train()
    opt_e, opt_g = ClippedAdam(eager.parameters()), ClippedAdam(graphed.parameters())
    before = [p.detach().clone() for p in graphed.parameters()]
    step = GraphedTrainStep(graphed, data, y_true, optimizer=opt_g)
    for p, b in zip(graphed.parameters(), before):
        assert torch.equal(p, b)
    st0 = opt_g.state_dict()
    assert st0['optimizer']['state'] == {} and st0['lr_scheduler']['last_epoch'] == 0 and opt_g.get_last_lr() == [LR]
    for it in range(3):
        opt_e.zero_grad()
        loss_e = criterion(y_true, eager(data), margin=None)['loss']
        loss_e.backward()
        opt_e.step()
        loss_g = step(data, y_true)['loss']
        assert torch.equal(loss_e.detach(), loss_g), it
        for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
            assert torch.equal(pe, pg), (it, k)
            assert torch.equal(pe.grad, pg.grad), (it, k)
    se, sg = opt_e.state_dict(), opt_g.state_dict()
    assert se['lr_scheduler'] == sg['lr_scheduler']
    for i in se['optimizer']['state']:
        for key in ('exp_avg', 'exp_avg_sq', 'step'):
            assert torch.equal(se['optimizer']['state'][i][key], sg['optimizer']['state'][i][key]), (i, key)
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), k
    fresh = SuperGlue(cfg)
    fresh.load_state_dict(graphed.state_dict())
    fresh = fresh.to(dev).eval()
    graphed.eval()
    with torch.no_grad():
        assert torch.equal(graphed(data)['scores'], fresh(data)['scores'])
