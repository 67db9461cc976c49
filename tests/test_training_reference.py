"""The training step against the UNMODIFIED reference module (oracle/_ref, staged by ``build()``) differentiated by torch autograd
on the CPU, in float64 and float32, at any shape, config and upstream gradient - no fixtures.

Every case takes the loss ``L = sum_out <G_out, out>`` over the outputs it uses (``scores``, ``context_descriptors0/1``), each
``G_out`` a seeded random tensor, and compares the three outputs, every parameter gradient (``None`` where the reference has
``None``), the gradients of both local-descriptor inputs and every BatchNorm buffer after the step.

* CPU leg: ``TrainStep`` driven by the float64 torch double of the kernels (tests/test_training.py ``_CpuOps``) against the
  reference's float64 autograd: catches schedule mistakes (which operator on which buffer, which gradient is accumulated where).
* GPU leg: the drop-in path, ``model(data)`` in ``train()`` mode and ``.backward()``, in 'fp32' and 'tf32x3'.  Per tensor,
  elementwise: ``|got - ref64| <= max(4 max|ref32 - ref64|, 2e-4 max|ref64|)`` (2e-4: DESIGN.md section 7's gradient bound).
"""
import copy
import functools

import pytest
import torch

from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict

OUTS = ('scores', 'context_descriptors0', 'context_descriptors1')


# --------------------------------------------------------------------------------------------------------------------- cases
# name: (default_config kwargs, extra config keys, [(B, N, M), ...], seed).  Each case is one image pair per shape.
CASES = {
    'default': (dict(descriptor_dim=64, num_stages=2, num_iters=10), {}, [(2, 37, 29)], 31),          # head_dim 16; N, M % 4 != 0
    'no_desc': (dict(descriptor_dim=64, num_stages=2, num_iters=10), dict(no_descriptors=True), [(2, 50, 41)], 32),
    'no_desc_nores': (dict(descriptor_dim=64, num_stages=2, num_iters=10, residual=False), dict(no_descriptors=True),
                      [(1, 40, 40)], 33),                                                              # n == m
    'offset_nores': (dict(descriptor_dim=128, num_heads=2, num_stages=2, num_iters=10, use_offset=True, reg=0.5, residual=False), {},
                     [(2, 300, 45)], 34),                                                              # head_dim 64; 600 rows: split-K dW
    'hd32': (dict(descriptor_dim=128, num_heads=4, num_stages=2, num_iters=10, side_info_size=6), {}, [(3, 97, 130)], 35),
    'hd8': (dict(descriptor_dim=32, num_heads=4, num_stages=2, num_iters=10), {}, [(2, 21, 18)], 36),
    'enc_none': (dict(descriptor_dim=64, num_stages=2, num_iters=10, hidden_layers_sizes=(), side_info_size=0), {}, [(2, 33, 27)], 37),
    'enc_30_50': (dict(descriptor_dim=64, num_stages=2, num_iters=10, hidden_layers_sizes=(30, 50), side_info_size=0), {},
                  [(2, 33, 27)], 38),
    # N = 1 with no Sinkhorn iteration, M = 1 with one.  B = 8, so that every BatchNorm call sees 8 rows: BatchNorm1d refuses one
    # row in train mode, and over two rows its input gradient is (dy1 - dy2)(1 - s^2) / 2 with s^2 = D^2 / (D^2 + 4 eps), a
    # cancellation whose fp32 rounding (already that of var + eps) is noise of ~1e-3 relative that no fp32 run reproduces.
    'degen_t0': (dict(descriptor_dim=64, num_stages=2, num_iters=0), {}, [(8, 1, 9)], 39),
    'degen_t1': (dict(descriptor_dim=64, num_stages=2, num_iters=1), {}, [(8, 13, 1)], 40),
}
# upstream gradients: (a) all three outputs, (b) context descriptors only (scores unused), (c) scores only
SCENARIOS = {'dense': OUTS, 'ctx': OUTS[1:], 'scores': OUTS[:1]}
MATRIX = [(c, 'dense') for c in CASES] + [(c, s) for c in ('default', 'no_desc') for s in ('ctx', 'scores')]


def _config(case):
    kw, extra, _, _ = CASES[case]
    return dict(default_config(**kw), **extra)


def perturb_bn(sd, seed):
    """BatchNorm running buffers away from their initial values (as oracle/gen_golden_train.py mints its fixtures)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in sd.items():
        if k.endswith('running_mean'):
            v = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith('running_var'):
            v = 0.5 + torch.rand(v.shape, generator=g)
        out[k] = v.clone()
    return out


def _state(case):
    _, _, _, seed = CASES[case]
    return perturb_bn(synthetic_state_dict(_config(case), seed=seed), seed)


def _batches(case, variant=''):
    """[(data, G)] per batch of the case; G holds a seeded upstream gradient for each of the three outputs (fp32-representable,
    so that the float64 schedule and the reference see the same G)."""
    cfg = _config(case)
    _, _, shapes, seed = CASES[case]
    if variant == 'accumulate':          # a second batch of another shape, into the same backward
        shapes = shapes + [(1, 23, 31)]
    images = variant == 'images'
    out = []
    for i, (b, n, m) in enumerate(shapes):
        data = synthetic_pairs(b, n, m, cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size'], family='planted',
                               seed=seed + 100 * i)
        data.pop('planted_matches0')
        if images:                       # sizes from image tensors [B, 1, H, W]; the image*_size entries are wrong on purpose
            data['image0'] = torch.zeros(1).expand(b, 1, 500, 700)
            data['image1'] = torch.zeros(1).expand(b, 1, 640, 480)
            data['image0_size'] = data['image1_size'] = (2000, 1000)
        g = torch.Generator().manual_seed(seed + 100 * i + 1)
        G = {'scores': torch.randn(b, n + 1, m + 1, generator=g).double(),
             'context_descriptors0': torch.randn(b, cfg['descriptor_dim'], n, generator=g).double(),
             'context_descriptors1': torch.randn(b, cfg['descriptor_dim'], m, generator=g).double()}
        out.append((data, G))
    return out


def _frozen(variant):
    """(parameter-name prefixes without grad, local descriptors requiring grad) of a variant"""
    if variant == 'frozen':
        return ('positional_encoding.', 'attention_gnn.layers.1.'), (True, False)
    return (), (True, True)


def _reference_class(required):
    from oracle.build_ref import import_reference
    ref = import_reference()
    if ref is None:
        msg = 'oracle/_ref is not staged: run build() (python -c "import __graft_entry__ as g; g.build()") where the reference exists'
        if required:
            pytest.fail(msg)
        pytest.skip(msg)
    return ref[0]


def _run(model, batches, outs, dev, dtype, frozen=(), ld_grad=(True, True), dk=None):
    """Forward every batch through ``model`` (train mode), L = sum of <G, out> over ``outs``, one backward.  Returns the outputs per
    batch, {parameter: grad or None}, the local-descriptor gradients per batch and {buffer: value}, all on the CPU."""
    for name, p in model.named_parameters():
        if any(name.startswith(f) for f in frozen):
            p.requires_grad_(False)
    hooks = []
    if dk is not None:                   # d loss / d K of every call of every layer, for the key-bias bound (float64 run)
        for l, layer in enumerate(model.attention_gnn.layers):
            def keep(mod, inp, out, l=l):
                if out.requires_grad:
                    out.retain_grad()
                    dk.setdefault(l, []).append(out)
            hooks.append(layer.module.mha.in_proj_k.register_forward_hook(keep))
    results, lds, L = [], [], 0
    for data, G in batches:
        d = {k: (v.to(dev, dtype) if torch.is_tensor(v) and v.is_floating_point() and not k.startswith('image') else
                 v.to(dev) if torch.is_tensor(v) else v) for k, v in data.items()}
        for i in (0, 1):
            d[f'local_descriptors{i}'] = d[f'local_descriptors{i}'].clone().requires_grad_(ld_grad[i])
        y = model(d)
        for k in outs:
            L = L + (G[k].to(dev, dtype) * y[k]).sum()
        results.append({k: y[k].detach().cpu().double() for k in OUTS})
        lds.append([d[f'local_descriptors{i}'] for i in (0, 1)])
    L.backward()
    for h in hooks:
        h.remove()
    grads = {k: (None if p.grad is None else p.grad.detach().cpu().double()) for k, p in model.named_parameters()}
    dld = [[None if t.grad is None else t.grad.detach().cpu().double() for t in pair] for pair in lds]
    bufs = {k: v.detach().cpu() for k, v in model.named_buffers()}
    return dict(outs=results, grads=grads, dld=dld, bufs=bufs)


@functools.lru_cache(maxsize=None)
def _reference(case, scenario, required, variant=''):
    """The reference module's float64 and float32 runs of a case (+ per key-bias parameter: rows summed, sum |dK| per column)."""
    SG = _reference_class(required)
    cfg, sd = _config(case), _state(case)
    batches = _batches(case, variant)
    frozen, ld_grad = _frozen(variant)
    res = {}
    for dtype, tag in ((torch.float64, '64'), (torch.float32, '32')):
        model = SG(copy.deepcopy(cfg))
        model.load_state_dict(sd, strict=True)
        model = model.to(dtype).train()
        dk = {} if dtype == torch.float64 else None
        res[tag] = _run(model, batches, SCENARIOS[scenario], 'cpu', dtype, frozen, ld_grad, dk)
        if dk is not None:
            kb = {}
            for l, calls in dk.items():
                gs = [t.grad for t in calls if t.grad is not None]
                if gs:
                    kb[f'attention_gnn.layers.{l}.module.mha.in_proj_k.bias'] = (
                        sum(g.shape[0] * g.shape[2] for g in gs), sum(g.abs().sum((0, 2)) for g in gs))
            res['kbias'] = kb
    return res


# --------------------------------------------------------------------------------------------------------------------- CPU leg
@pytest.mark.parametrize('case,scenario', MATRIX)
def test_training_schedule_matches_reference_autograd_on_cpu(case, scenario):
    """TrainStep's schedule on the float64 torch double of the kernels, with upstream gradients on any of the three outputs."""
    from openglue_b200 import SuperGlue
    from openglue_b200.training import TrainStep
    from test_training import _CpuOps
    ref = _reference(case, scenario, False)['64']
    model = SuperGlue(_config(case))
    model.load_state_dict(_state(case), strict=True)
    model = model.double().train()
    (data, G), = _batches(case)
    data = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in data.items()}
    step = TrainStep(model, data, ops=_CpuOps())
    got = dict(zip(OUTS, step.forward()))
    assert (got['scores'] - ref['outs'][0]['scores']).abs().max() < 5e-6      # (the reference keeps log_a / log_b in fp32)
    for k in OUTS[1:]:
        assert (got[k] - ref['outs'][0][k]).abs().max() < 1e-9, k
    use = SCENARIOS[scenario]
    grads = step.backward(*[G[k] if k in use else None for k in OUTS])
    want = {k for k, g in ref['grads'].items() if g is not None}
    want |= {f'local_descriptors{i}' for i in (0, 1) if ref['dld'][0][i] is not None}
    assert set(grads) == want
    refs = dict(ref['grads'], local_descriptors0=ref['dld'][0][0], local_descriptors1=ref['dld'][0][1])
    for k in want:
        g, r = grads[k].reshape(refs[k].shape), refs[k]
        assert torch.isfinite(g).all(), k
        assert (g - r).abs().max() <= 2e-6 * max(1.0, float(r.abs().max())), k
    for k, v in model.named_buffers():
        r = ref['bufs'][k]
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(r), k
        else:
            assert (v - r).abs().max() <= 1e-9 * max(1.0, float(r.abs().max())), k


# --------------------------------------------------------------------------------------------------------------------- GPU leg
def _gpu_run(case, scenario, precision, variant=''):
    from openglue_b200 import SuperGlue
    dev = torch.device('cuda:0')
    model = SuperGlue(dict(_config(case), precision=precision))
    model.load_state_dict(_state(case), strict=True)
    model = model.to(dev).train()
    frozen, ld_grad = _frozen(variant)
    return _run(model, _batches(case, variant), SCENARIOS[scenario], dev, torch.float32, frozen, ld_grad)


class _Check:
    """Elementwise |got - ref64| <= max(4 max|ref32 - ref64|, 2e-4 max|ref64|) per tensor; every comparison is printed."""

    def __init__(self, label):
        self.label, self.bad = label, []

    def __call__(self, what, got, r64, r32, floor=None):
        assert got.shape == r64.shape, (what, got.shape, r64.shape)
        got, r64, r32 = got.double(), r64.double(), r32.double()
        assert torch.isfinite(got).all(), what
        bound = max(4 * float((r32 - r64).abs().max()), 2e-4 * float(r64.abs().max()))
        err = (got - r64).abs()
        if floor is not None:            # a per-column rounding floor (key-projection bias: zero in exact arithmetic)
            ok = bool((err <= torch.clamp(floor, min=bound)).all())
            bound = float(torch.clamp(floor, min=bound).max())
        else:
            ok = float(err.max()) <= bound
        print(f'{self.label} {what:60s} err {float(err.max()):.3e}  bound {bound:.3e}{"" if ok else "  FAIL"}')
        if not ok:
            self.bad.append(what)

    def done(self):
        assert not self.bad, f'{self.label}: beyond the bound: {self.bad}'


def _compare(label, got, ref):
    chk = _Check(label)
    r64, r32 = ref['64'], ref['32']
    for j, outs in enumerate(got['outs']):
        for k in OUTS:
            chk(f'batch {j} {k}', outs[k], r64['outs'][j][k], r32['outs'][j][k])
    for k, g in got['grads'].items():
        r = r64['grads'][k]
        assert (g is None) == (r is None), f'{k}: grad {"None" if g is None else "set"}, reference {"None" if r is None else "set"}'
        if g is None:
            continue
        floor = None
        if k in ref['kbias']:
            rows, sabs = ref['kbias'][k]
            floor = rows * 2.0 ** -24 * sabs
        chk(f'grad {k}', g, r, r32['grads'][k], floor)
    for j, pair in enumerate(got['dld']):
        for i in (0, 1):
            r = r64['dld'][j][i]
            assert (pair[i] is None) == (r is None), f'batch {j} local_descriptors{i}: grad presence differs from the reference'
            if r is not None:
                chk(f'batch {j} grad local_descriptors{i}', pair[i], r, r32['dld'][j][i])
    for k, v in got['bufs'].items():
        r = r64['bufs'][k]
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(r), k
        else:
            chk(f'buffer {k}', v, r, r32['bufs'][k])
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('case,scenario', MATRIX)
def test_training_step_matches_reference_autograd(case, scenario, precision):
    ref = _reference(case, scenario, True)
    _compare(f'[{case} {scenario} {precision}]', _gpu_run(case, scenario, precision), ref)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['accumulate', 'frozen', 'images'])
def test_training_autograd_usage_matches_reference(variant):
    """accumulate: two forwards (B 2 and B 1, other N, M) into one backward - summed gradients, BatchNorm buffers moved four times
    per call site; frozen: positional encoder and layer 1 without grad, local_descriptors1 without grad - they get None;
    images: image sizes from data['image0'] / data['image1'] tensors, which take precedence over image*_size."""
    ref = _reference('default', 'dense', True, variant)
    _compare(f'[{variant}]', _gpu_run('default', 'dense', 'tf32x3', variant), ref)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['offset_nores', 'default'])
def test_training_default_precision_is_tf32x3(case):
    """The default 'fp16x3' runs the training step on the tf32x3 operators: bit-identical outputs, gradients and buffers."""
    a, b = _gpu_run(case, 'dense', 'fp16x3'), _gpu_run(case, 'dense', 'tf32x3')
    for k in OUTS:
        assert torch.equal(a['outs'][0][k], b['outs'][0][k]), k
    for k in a['grads']:
        assert torch.equal(a['grads'][k], b['grads'][k]), k
    for i in (0, 1):
        assert torch.equal(a['dld'][0][i], b['dld'][0][i])
    for k in a['bufs']:
        assert torch.equal(a['bufs'][k], b['bufs'][k]), k
