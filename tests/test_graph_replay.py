"""GraphedTrainStep across calls that change what its graph baked in (`pytest -m gpu` on an H100): the image sizes of a uniform
batch, ``p.grad`` set to None by ``zero_grad()``, and a parameter re-allocated by ``p.data = ...``; and labels given as int32.
Each replay is compared bit for bit with the eager autograd step of a second model with the same weights."""
import copy
import os

import pytest
import torch

from openglue_b200 import ClippedAdam, SuperGlue, criterion
from openglue_b200.synthetic import synthetic_state_dict
from openglue_b200.training import GraphedTrainStep

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')


def _setup(name='train_ragged'):
    """a training fixture (train_ragged: 3 pairs, 96 x 131 keypoints, image sizes 960 x 720): its batch, labels and two equal
    models (eager, graphed)"""
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', name + '.pt'), weights_only=False)
    sd = synthetic_state_dict(fx['config'], seed=fx['weights_seed'])
    sd.update(fx['bn_buffers'])
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    y_true = {'gt_matches0': fx['gt_matches0'].to(DEV), 'gt_matches1': fx['gt_matches1'].to(DEV)}
    models = []
    for _ in range(2):
        m = SuperGlue(dict(fx['config'], precision='tf32x3'))
        m.load_state_dict(copy.deepcopy(sd), strict=True)
        models.append(m.to(DEV).train())
    return data, y_true, models


def _assert_same(eager, graphed, loss_e, loss_g, it):
    assert torch.equal(loss_e.detach(), loss_g), it
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.equal(pe, pg), (it, k)
        assert pg.grad is not None and torch.equal(pe.grad, pg.grad), (it, k)
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), (it, k)


def test_other_image_size_of_a_uniform_batch_raises():
    """a uniform batch's image sizes normalise the keypoints as constants of the graph: another size must not replay it"""
    data, y_true, (_, graphed) = _setup()
    step = GraphedTrainStep(graphed, data, y_true)
    step(data, y_true)
    w, h = data['image0_size']
    with pytest.raises(ValueError, match='image sizes'):
        step({**data, 'image0_size': (w * 0.75, h)}, y_true)
    step(data, y_true)


def test_gradients_after_zero_grad_set_to_none_equal_the_eager_step():
    data, y_true, (eager, graphed) = _setup()
    step = GraphedTrainStep(graphed, data, y_true)
    for it in range(3):
        eager.zero_grad()
        graphed.zero_grad()
        assert all(p.grad is None for p in graphed.parameters())
        loss_e = criterion(y_true, eager(data), margin=None)['loss']
        loss_e.backward()
        loss_g = step(data, y_true)['loss']
        _assert_same(eager, graphed, loss_e, loss_g, it)


def test_reallocated_parameter_is_captured_again(monkeypatch):
    """after p.data = p.data.clone() the next call captures once more, and the optimiser inside the graph updates the new
    storage: parameters, gradients and buffers stay equal to the eager step's"""
    captured = [0]
    orig = torch.cuda.CUDAGraph.capture_end

    def counting(self):
        captured[0] += 1
        return orig(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'capture_end', counting)
    data, y_true, (eager, graphed) = _setup()
    opt_e, opt_g = ClippedAdam(eager.parameters()), ClippedAdam(graphed.parameters())
    step = GraphedTrainStep(graphed, data, y_true, optimizer=opt_g)

    def both(it):
        opt_e.zero_grad()
        loss_e = criterion(y_true, eager(data), margin=None)['loss']
        loss_e.backward()
        opt_e.step()
        _assert_same(eager, graphed, loss_e, step(data, y_true)['loss'], it)
    both(0)
    assert captured[0] == 1
    for m in (eager, graphed):
        p = m.attention_gnn.layers[1].module.mha.in_proj_v.weight
        p.data = p.data.clone()
    for it in (1, 2):
        both(it)
        assert captured[0] == 2


def test_int32_labels_with_a_margin_equal_the_eager_step():
    """the metric loss reads the labels through an int64 pointer: labels given as int32 are held as int64 in the graph"""
    data, y_true, (eager, graphed) = _setup('train_metric')
    y32 = {k: v.to(torch.int32) for k, v in y_true.items()}
    step = GraphedTrainStep(graphed, data, y32, margin=0.5, metric_weight=0.5)
    for it in range(2):
        eager.zero_grad()
        out = criterion(y_true, eager(data), margin=0.5)
        (1.0 * out['loss'] + 0.5 * out['metric_loss']).backward()
        got = step(data, y32)
        assert float(got['metric_loss']) > 0 and torch.equal(out['metric_loss'].detach(), got['metric_loss']), it
        _assert_same(eager, graphed, out['loss'], got['loss'], it)
