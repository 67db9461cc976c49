"""The serving paths the headline number runs on (`pytest -m gpu` on an H100): ``MatchingCore(use_cuda_graph=True)`` replay,
borrowed outputs, host inputs and ``submit()/wait()``, in every precision.

Graph replay runs the same kernels in the same order as eager launches, so every check here is bit for bit (``torch.equal``)
against eager launches of the same weights on the same inputs; where it says "oracle" it is the float64 oracle with the bounds
and decisive-row rule of test_gpu_parity.test_forward_matches_oracle.  The graph-cache tests count captures through a
counting ``torch.cuda.CUDAGraph``: a graph kept past a change of what it baked in (weights, precision, threshold, image
size, buffer addresses) replays a stale answer, or reads freed blocks."""
import pytest
import torch

from openglue_b200.gt_matches import gt_matches
from openglue_b200.losses import criterion
from openglue_b200.superglue import MatchingCore
from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
from oracle import superglue_oracle as O
from test_gpu_parity import DEV, TOL, _model, _to_dev, check_matches

pytestmark = pytest.mark.gpu

PRECISIONS = ['fp16x3', 'tf32x3', 'fp32']
OUTPUTS = ('matches0', 'matching_scores0', 'matches1', 'matching_scores1', 'scores')
# (config kwargs, B, n, m)
CONFIGS = {
    'd256_ragged_b2': (dict(descriptor_dim=256, num_stages=2, num_iters=20), 2, 150, 97),        # head_dim 64: the fp16 GNN
    'd256_square_b1': (dict(descriptor_dim=256, num_stages=3, num_iters=20), 1, 128, 128),       # n == m: joint self layers
    'd128_h4_b3': (dict(descriptor_dim=128, num_heads=4, num_stages=2, num_iters=20, side_info_size=6), 3, 100, 173),  # head_dim 32
}


def _pairs(cfg, B, n, m, seed, family='planted'):
    return synthetic_pairs(B, n, m, cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size'], family=family, seed=seed)


def _host(data, pinned=True):
    return {k: ((v.cpu().pin_memory() if pinned else v.cpu()) if torch.is_tensor(v) else v) for k, v in data.items()}


def _setup(name, precision, seed=3):
    kw, B, n, m = CONFIGS[name]
    cfg = default_config(**kw)
    return cfg, _model(cfg, synthetic_state_dict(cfg, seed=seed), precision), (B, n, m)


def _assert_same(got, want, keys=OUTPUTS):
    for k in keys:
        g, w = got[k].cpu(), want[k].cpu()
        assert g.shape == w.shape, f'{k}: shape {tuple(g.shape)} != {tuple(w.shape)}'
        same = torch.equal(g, w)
        assert same, f'{k}: {int((g != w).sum())} elements differ, max |diff| {(g.double() - w.double()).abs().max():.3e}'


@pytest.fixture
def captures(monkeypatch):
    """Number of CUDA graphs captured since the test started."""
    count = [0]

    class CountingGraph(torch.cuda.CUDAGraph):
        def capture_end(self):
            count[0] += 1
            super().capture_end()
    monkeypatch.setattr(torch.cuda, 'CUDAGraph', CountingGraph)
    return lambda: count[0]


# --------------------------------------------------------------------------- replay against eager and the oracle
@pytest.mark.parametrize('name', CONFIGS)
@pytest.mark.parametrize('precision', PRECISIONS)
def test_graph_replay_matches_eager(name, precision):
    """Replays with new device inputs of one shape (planted and flat, so the magnitudes change too), a return to earlier
    inputs, then pinned and pageable host inputs: each equals the eager call on the same inputs."""
    cfg, model, shape = _setup(name, precision)
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    inputs = [_to_dev(_pairs(cfg, *shape, seed=s, family=f)) for s, f in ((11, 'planted'), (12, 'flat'), (13, 'planted'))]
    want = [eager(x, want_scores=True) for x in inputs]
    for i in (0, 1, 2, 0, 2):
        _assert_same(graphed(inputs[i], want_scores=True), want[i])
    for i, pinned in ((1, True), (2, False)):
        got = graphed(_host(inputs[i], pinned), want_scores=True)
        assert all(v.device.type == 'cpu' for v in got.values())
        _assert_same(got, want[i])
    assert len(graphed._graphs) == 1


@pytest.mark.parametrize('precision', PRECISIONS)
def test_graph_replay_matches_oracle(precision):
    """A replay after other inputs (the capture call and a flat batch) against the float64 oracle."""
    kw, B, n, m = CONFIGS['d256_ragged_b2']
    cfg = default_config(**kw)
    sd = synthetic_state_dict(cfg, seed=3)
    data = _pairs(cfg, B, n, m, seed=11)
    ref = O.run(sd, cfg, data, 0.2)
    ref64 = O.run(sd, cfg, data, 0.2, dtype=torch.float64)
    bound = max(TOL, 2 * float((ref['scores'].double() - ref64['scores']).abs().max()))
    graphed = MatchingCore(_model(cfg, sd, precision), 0.2, use_cuda_graph=True)
    graphed(_to_dev(data))
    graphed(_to_dev(_pairs(cfg, B, n, m, seed=12, family='flat')))
    res = graphed(_to_dev(data), want_scores=True)
    assert (res['scores'].cpu().double() - ref64['scores']).abs().max() <= bound
    check_matches(res, ref, ref64['scores'], bound)


# --------------------------------------------------------------------------- fp16 scales follow each replay's inputs
def _magnitude_steps(cfg, shape, exponents):
    base = _pairs(cfg, *shape, seed=21, family='flat')                       # unit descriptors
    steps = []
    for i, e in enumerate(exponents):
        x = dict(base)
        for k in ('local_descriptors0', 'local_descriptors1'):
            x[k] = base[k] * 2.0 ** e
        x['keypoints0'] = base['keypoints0'] * 0.9 + 32.0 * i
        x['keypoints1'] = base['keypoints1'] * 0.9 + 32.0 * (len(exponents) - 1 - i)
        steps.append(_to_dev(x))
    return steps


@pytest.mark.parametrize('exponents', [(8, 0, -8), (-8, 0, 8)], ids=['shrinking', 'growing'])
def test_fp16_replay_scales_follow_input_magnitude(exponents):
    """fp16x3 derives every operand scale from amax slots in the workspace, which each forward pass resets on the device.
    Replays with descriptors scaled by 2^8, 2^0, 2^-8 (and back) must each equal eager: a slot carried over from the previous
    inputs would give a different scale.  The reference results come from a second model with the same weights, run in the
    opposite order, so that no call here and its reference share a history of inputs."""
    cfg, model, shape = _setup('d256_ragged_b2', 'fp16x3')
    steps = _magnitude_steps(cfg, shape, exponents)
    reference = MatchingCore(_setup('d256_ragged_b2', 'fp16x3')[1], 0.2)
    want = {i: reference(steps[i], want_scores=True) for i in reversed(range(len(steps)))}
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    for i, x in enumerate(steps):
        got = graphed(x, want_scores=True)
        _assert_same(got, want[i])
        _assert_same(got, eager(x, want_scores=True))


# --------------------------------------------------------------------------- graph cache
def test_graph_cache_evicts_the_oldest_shape(captures):
    """Five shapes through a cache of four: the fifth evicts the first, which is captured again; the rest replay."""
    cfg, model, _ = _setup('d256_ragged_b2', 'fp16x3')
    shapes = [(1, 64, 48), (1, 80, 64), (2, 48, 56), (1, 96, 72), (2, 64, 40)]
    model(_to_dev(_pairs(cfg, 2, 96, 72, seed=0)))               # the largest workspace first: no call below reallocates it
    gen = model._alloc_gen
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    inputs = [_to_dev(_pairs(cfg, *s, seed=30 + i)) for i, s in enumerate(shapes)]
    want = [eager(x, want_scores=True) for x in inputs]
    assert graphed.max_graphs == 4
    for i, count in zip((0, 1, 2, 3, 4, 0, 4, 3), (1, 2, 3, 4, 5, 6, 6, 6)):
        _assert_same(graphed(inputs[i], want_scores=True), want[i])
        assert captures() == count, f'after shape {i}'
        assert len(graphed._graphs) <= graphed.max_graphs
    assert model._alloc_gen == gen


@pytest.mark.parametrize('grower', ['other_core', 'eager'])
def test_graph_recaptured_after_workspace_growth(captures, grower):
    """A larger call on the shared SuperGlue reallocates its workspace: a graph captured before must not replay."""
    cfg, model, _ = _setup('d256_ragged_b2', 'fp16x3')
    eager, core_a = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    small = [_to_dev(_pairs(cfg, 1, 64, 48, seed=s)) for s in (50, 51)]
    large = _to_dev(_pairs(cfg, 2, 160, 120, seed=52))
    _assert_same(core_a(small[0], want_scores=True), eager(small[0], want_scores=True))
    assert captures() == 1
    gen = model._alloc_gen
    if grower == 'other_core':
        got = MatchingCore(model, 0.2, use_cuda_graph=True)(large, want_scores=True)
        _assert_same(got, eager(large, want_scores=True))
    else:
        model(large)
    assert model._alloc_gen != gen
    before = captures()
    got = core_a(small[1], want_scores=True)
    assert captures() == before + 1
    _assert_same(got, eager(small[1], want_scores=True))


def _scale_in_place(model, data):
    with torch.no_grad():
        model.linear_proj.weight.mul_(1.01)
    return data


def _load_other_weights(model, data):
    model.load_state_dict(synthetic_state_dict(model.config, seed=9))
    return data


def _rebind_parameter_data(model, data):
    p = model.attention_gnn.layers[1].module.mha.in_proj_v.weight
    p.data = p.data * 1.01
    return data


def _replace_parameter(model, data):
    conv = model.attention_gnn.layers[2].module.mha.out_proj
    conv.weight = torch.nn.Parameter(conv.weight.detach() * 1.01)
    return data


def _switch_precision(model, data):
    model.config['precision'] = 'tf32x3'
    return data


def _resize_image0(model, data):
    w, h = data['image0_size']
    return {**data, 'image0_size': (w * 0.75, h)}


KEY_CHANGES = {'weights_mul_': _scale_in_place, 'load_state_dict': _load_other_weights, 'param_data_assign': _rebind_parameter_data,
               'param_replaced': _replace_parameter, 'precision': _switch_precision, 'image_size': _resize_image0}


@pytest.mark.parametrize('change', KEY_CHANGES)
def test_graph_follows_changes_it_baked_in(captures, change):
    """After a change of the weights (in place, load_state_dict, ``p.data = new``, a new Parameter object), of the precision or
    of the image size, the
    next graphed call (made before any eager call could rebuild the packed weights) is captured again, equals eager with the
    new state and differs from the old answer."""
    cfg, model, shape = _setup('d256_ragged_b2', 'fp16x3')
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    x = _to_dev(_pairs(cfg, *shape, seed=60))
    old = graphed(x, want_scores=True)
    assert captures() == 1
    x = KEY_CHANGES[change](model, x)
    got = graphed(x, want_scores=True)
    assert captures() == 2
    _assert_same(got, eager(x, want_scores=True))
    assert not torch.equal(got['scores'], old['scores'])
    _assert_same(graphed(x, want_scores=True), got)
    assert captures() == 2


def test_cores_sharing_a_model_keep_their_thresholds(captures):
    """Two graphed cores with different match_thresholds on one SuperGlue, called in turn: each equals its eager counterpart
    and the shared config keeps its threshold.  A core whose threshold is changed follows it."""
    cfg, model, shape = _setup('d256_ragged_b2', 'fp16x3')
    xs = [_to_dev(_pairs(cfg, *shape, seed=s)) for s in (70, 71)]
    ms = MatchingCore(model, 0.2)(xs[0])['matching_scores0']
    thr = float(ms[ms > 0].median())                               # drops about half of the matches at 0.2
    a, b = MatchingCore(model, 0.2, use_cuda_graph=True), MatchingCore(model, thr, use_cuda_graph=True)
    ea, eb = MatchingCore(model, 0.2), MatchingCore(model, thr)
    for x in (xs[0], xs[1], xs[0]):
        ga, gb = a(x, want_scores=True), b(x, want_scores=True)
        _assert_same(ga, ea(x, want_scores=True))
        _assert_same(gb, eb(x, want_scores=True))
    assert not torch.equal(ga['matches0'], gb['matches0'])
    assert captures() == 2
    assert 'match_threshold' not in model.config and model._ogcfg.match_threshold == pytest.approx(0.2, abs=1e-7)
    a.match_threshold = thr
    _assert_same(a(xs[1], want_scores=True), eb(xs[1], want_scores=True))
    assert captures() == 3


# --------------------------------------------------------------------------- borrowed outputs
def test_borrowed_outputs_are_the_graphs_buffers():
    """borrow=True returns the graph's output buffers (equal to eager, overwritten by the next replay, as documented);
    without it the results are copies a later replay leaves alone."""
    cfg, model, shape = _setup('d256_ragged_b2', 'fp16x3')
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    x1, x2 = (_to_dev(_pairs(cfg, *shape, seed=s)) for s in (80, 81))
    e1, e2 = eager(x1, want_scores=True), eager(x2, want_scores=True)
    r1 = graphed(x1, want_scores=True, borrow=True)
    _assert_same(r1, e1)
    c1 = graphed(x1, want_scores=True)
    r2 = graphed(x2, want_scores=True, borrow=True)
    _assert_same(r2, e2)
    assert all(r1[k].data_ptr() == r2[k].data_ptr() for k in OUTPUTS)
    _assert_same(r1, e2)
    _assert_same(c1, e1)
    assert all(c1[k].data_ptr() != r1[k].data_ptr() for k in OUTPUTS)


def test_criterion_on_borrowed_scores_matches_eager():
    """The C4 step: criterion on the graph's borrowed scores, then the next replay; each loss equals criterion on eager scores."""
    cfg, model, shape = _setup('d256_ragged_b2', 'fp16x3')
    B = shape[0]
    H = torch.tensor([[0.9, 0.0, 20.0], [0.0, 0.9, 20.0], [0.0, 0.0, 1.0]], device=DEV).repeat(B, 1, 1)
    tf = {'type': ['perspective'] * B, 'H': H}                     # the planted similarity of synthetic_pairs
    xs = [_to_dev(_pairs(cfg, *shape, seed=s)) for s in (90, 91, 92)]
    gts = []
    for x in xs:
        g0, g1 = gt_matches(x['keypoints0'], x['keypoints1'], tf)
        gts.append({'gt_matches0': g0, 'gt_matches1': g1})
    eager, graphed = MatchingCore(model, 0.2), MatchingCore(model, 0.2, use_cuda_graph=True)
    want = [criterion(y, eager(x, want_scores=True)) for x, y in zip(xs, gts)]
    got = []
    for i in (0, 1, 2, 0):
        res = graphed(xs[i], want_scores=True, borrow=True)
        got.append((i, criterion(gts[i], res)))
    for i, loss in got:
        assert torch.isfinite(loss['loss'])
        assert torch.equal(loss['loss'], want[i]['loss']) and torch.equal(loss['metric_loss'], want[i]['metric_loss'])


# --------------------------------------------------------------------------- submit() with graphs
@pytest.mark.parametrize('order', ['ABABABAB', 'ABBAABBA'])
def test_graphed_submit_matches_blocking_eager(order):
    """fp16x3 submit()/wait() with graphs, two shapes and descriptors scaled by 2^8, 2^0, 2^-8 in turn.  In 'ABBAABBA' each
    of the two input-buffer slots changes shape on every submit, so its buffers are reallocated while the other batch is in
    flight.  Every wait() result equals the blocking eager call."""
    cfg, model, _ = _setup('d256_ragged_b2', 'fp16x3')
    shapes = {'A': (1, 96, 80), 'B': (2, 64, 112)}
    batches = []
    for i, s in enumerate(order):
        x = _pairs(cfg, *shapes[s], seed=100 + i)
        for k in ('local_descriptors0', 'local_descriptors1'):
            x[k] = x[k] * 2.0 ** (8, 0, -8)[i % 3]
        batches.append(_host(x))
    blocking = MatchingCore(model, 0.2, device=DEV)
    piped = MatchingCore(model, 0.2, device=DEV, use_cuda_graph=True)
    want = [blocking(h) for h in batches]
    got, pend = [], None
    for h in batches:
        nxt = piped.submit(h)
        if pend is not None:
            got.append({k: v.clone() for k, v in pend.wait().items()})
        pend = nxt
    got.append({k: v.clone() for k, v in pend.wait().items()})
    for i, (w, g) in enumerate(zip(want, got)):
        assert all(v.device.type == 'cpu' for v in g.values())
        _assert_same(g, w, MatchingCore._OUT_KEYS)
    assert len(piped._graphs) == 2


# --------------------------------------------------------------------------- bench.py's own sequence at C3
def _check_c3(res, fx, scored=False):
    """The bounds of test_gpu_parity.test_forward_matches_reference_big for a planted fixture."""
    bound = max(TOL, 2 * fx['ref32_vs_ref64_max_abs'])
    m0, ms0 = res['matches0'].cpu(), res['matching_scores0'].cpu()
    assert torch.equal(m0, fx['matches0'])
    assert (ms0 - fx['matching_scores0']).abs().max() <= bound
    if not scored:
        return
    k, (sr, sc) = fx['scored_pairs'], fx['sample_stride']
    s = res['scores'][:k].cpu()
    assert (s[:, ::sr, ::sc].double() - fx['scores_f64_sample']).abs().max() <= bound
    assert (s[:, ::sr, ::sc] - fx['scores_f32_sample']).abs().max() <= bound
    assert (s[:, -1, :] - fx['scores_f32_lastrow']).abs().max() <= bound
    assert (s[:, :, -1] - fx['scores_f32_lastcol']).abs().max() <= bound
    assert (s.double().sum(2) - fx['scores_f64_rowsum']).abs().max() / fx['scores_f64_rowsum'].abs().max() < 2e-5
    gap = fx['row_top2_gap_f64'] > 2 * bound
    assert torch.equal(s[:, :-1, :-1].argmax(2)[gap], fx['row_argmax_f64'][gap])
    mutual = gap & (fx['matching_scores0'][:k] > 0)
    assert (ms0[:k][mutual] - fx['matching_scores0_f64'][mutual]).abs().max() <= TOL


def test_bench_call_sequence_at_c3(golden):
    """bench.py's calls on its headline configuration (C3: 16 pairs, N = M = 2048, 9 stages, fp16x3, graphs on): warm-up and
    timed borrowed device calls, blocking host calls, then submit()/wait(); every output against the reference's fixture."""
    fx = golden('C3_planted')
    model = _model(fx['config'], fx['state_dict'], 'fp16x3')
    core = MatchingCore(model, fx['match_threshold'], device=DEV, use_cuda_graph=True)
    host = _host(fx['data'])
    data = _to_dev(fx['data'])
    for _ in range(5):
        _check_c3(core(data, borrow=True), fx)
    res = core(data, want_scores=True, borrow=True)
    _check_c3(res, fx, scored=True)
    _assert_same(res, MatchingCore(model, fx['match_threshold'])(data, want_scores=True))
    for _ in range(2):
        _check_c3(core(host), fx)
    pend = None
    for _ in range(3):
        nxt = core.submit(host)
        if pend is not None:
            _check_c3(pend.wait(), fx)
        pend = nxt
    _check_c3(pend.wait(), fx)
    assert len(core._graphs) == 1
