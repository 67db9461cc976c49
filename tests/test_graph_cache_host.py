"""The rules of the one capture-and-replay path (openglue_b200/_graphs.py), on the CPU: a fake graph class stands in for
torch.cuda.CUDAGraph, so every step the path takes is recorded in order."""
import contextlib

import pytest
import torch

from openglue_b200 import _graphs


@pytest.fixture
def log(monkeypatch):
    events = []

    class FakeGraph:
        def replay(self):
            events.append('replay')

    @contextlib.contextmanager
    def fake_capture(graph):
        assert isinstance(graph, FakeGraph)
        events.append('capture_begin')
        yield
        events.append('capture_end')

    monkeypatch.setattr(torch.cuda, 'CUDAGraph', FakeGraph)
    monkeypatch.setattr(torch.cuda, 'graph', fake_capture)
    monkeypatch.setattr(torch.cuda, 'synchronize', lambda dev=None: events.append('synchronize'))
    return events


class Owner:
    """A graph owner as the library's four are: its own dict, max_graphs, a version and a chain."""

    def __init__(self, log, max_graphs=4):
        self.log, self._graphs, self.max_graphs, self.ver = log, {}, max_graphs, 0

    def chain(self, static):
        self.log.append('chain')
        return {'y': static['x'] * 2}

    def __call__(self, key, x, guard=None, f32=True, hold=None):
        return _graphs.run(self._graphs, self.max_graphs, key, lambda: self.ver, {'x': x}, self.chain, torch.device('cpu'), f32,
                           hold=hold, guard=guard)


def test_one_warm_up_and_one_capture_per_key(log):
    owner = Owner(log)
    out = owner('a', torch.ones(3))
    assert log == ['chain', 'synchronize', 'capture_begin', 'chain', 'capture_end', 'replay']
    assert torch.equal(out['y'], torch.full((3,), 2.0))              # warm-up and capture read the inputs' values
    for v in (3.0, 5.0):
        assert owner('a', torch.full((3,), v)) is out
        assert torch.equal(owner._graphs['a'].static['x'], torch.full((3,), v))   # each replay reads this call's inputs
    assert log[6:] == ['replay', 'replay']
    entry = owner._graphs['a']
    assert entry.out is out and entry.version == 0 and entry.held is None and entry.state is None


def test_version_change_recaptures_under_the_same_key(log):
    owner = Owner(log)
    owner('a', torch.ones(3))
    owner('b', torch.ones(3))
    first = owner._graphs['a']
    owner.ver = 1
    owner('a', torch.ones(3))
    assert log.count('capture_begin') == 3
    assert list(owner._graphs) == ['b', 'a'] and owner._graphs['a'] is not first and owner._graphs['a'].version == 1
    owner('a', torch.ones(3))
    assert log.count('capture_begin') == 3


def test_version_is_taken_after_the_capture(log):
    """the warm-up may reallocate what the version fingerprints: a version read before it would recapture on every call"""
    owner = Owner(log)

    def chain(static):
        owner.ver += 1                                               # e.g. a workspace grown by the warm-up
        return {'y': static['x']}
    owner.chain = chain
    owner('a', torch.ones(3))
    owner.chain = lambda s: pytest.fail('captured again')
    owner('a', torch.ones(3))
    assert owner._graphs['a'].version == 2


def test_fifo_eviction_at_max_graphs(log):
    owner = Owner(log, max_graphs=2)
    for key, kept in (('a', ['a']), ('b', ['a', 'b']), ('c', ['b', 'c']), ('b', ['b', 'c']), ('a', ['c', 'a'])):
        owner(key, torch.ones(3))
        assert list(owner._graphs) == kept, key
    assert log.count('capture_begin') == 4
    owner.max_graphs = 1                                             # read at call time
    owner('d', torch.ones(3))
    assert list(owner._graphs) == ['d']


def test_static_dtypes(log):
    x64, i16 = torch.ones(2, dtype=torch.float64), torch.ones(2, dtype=torch.int16)
    seen = {}

    def chain(static):
        seen.update({k: v.dtype for k, v in static.items()})
    _graphs.capture({'x': x64, 'i': i16}, chain, torch.device('cpu'), True, lambda: 0)
    assert seen == {'x': torch.float32, 'i': torch.int16}
    _graphs.capture({'x': x64, 'i': i16}, chain, torch.device('cpu'), False, lambda: 0)
    assert seen == {'x': torch.float64, 'i': torch.int16}


def test_guard_hooks_run_in_order(log):
    class Guard:
        def save(self):
            log.append('save')

        def restore(self):
            log.append('restore')

        def captured(self):
            log.append('captured')
            return 'idx'

        def replayed(self, state):
            log.append(f'replayed {state}')

    owner = Owner(log)
    owner('a', torch.ones(3), guard=Guard(), hold=lambda: log.append('hold') or 'held')
    assert log == ['save', 'chain', 'synchronize', 'restore', 'hold', 'capture_begin', 'chain', 'capture_end', 'captured', 'replay',
                   'replayed idx']
    assert owner._graphs['a'].held == 'held'
    owner('a', torch.ones(3), guard=Guard())
    assert log[11:] == ['replay', 'replayed idx']
