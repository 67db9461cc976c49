"""tools/gpu_timing.py, the timer and card record every script under tools/ uses, checked on the CPU with fake CUDA events."""
import importlib.util
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def gt(monkeypatch):
    """the module, loaded with sys.path restored afterwards, and a log of what it asks of CUDA"""
    monkeypatch.setattr(sys, 'path', list(sys.path))
    spec = importlib.util.spec_from_file_location('gpu_timing', os.path.join(ROOT, 'tools', 'gpu_timing.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    log = []

    class Event:
        made = 0

        def __init__(self, enable_timing=False):
            assert enable_timing
            self.name = ('start', 'end')[Event.made % 2]          # events_ms makes its events in pairs, start first
            Event.made += 1

        def record(self):
            log.append(('record', self.name))

        def elapsed_time(self, other):
            assert (self.name, other.name) == ('start', 'end')
            return 12.0

    monkeypatch.setattr(torch.cuda, 'Event', Event)
    monkeypatch.setattr(torch.cuda, 'synchronize', lambda device=None: log.append(('sync',)))
    mod.log = log
    return mod


@pytest.mark.parametrize('iters,warmup', [(1, 0), (4, 0), (3, 2)])
def test_events_ms_warms_up_synchronises_and_divides(gt, iters, warmup):
    ms = gt.events_ms(lambda: gt.log.append(('call',)), iters, warmup=warmup)
    assert gt.log == ([('call',)] * warmup + [('sync',), ('record', 'start')] + [('call',)] * iters
                      + [('record', 'end'), ('sync',)])
    assert ms == 12.0 / iters


def test_rounds_ms_alternates_forms_in_insertion_order(gt):
    forms = {name: (lambda name=name: gt.log.append(('call', name))) for name in ('b', 'c', 'a')}
    ms = gt.rounds_ms(forms, iters=2, rounds=3)
    assert list(ms) == ['b', 'c', 'a'] and ms == {k: [6.0] * 3 for k in forms}
    calls = [e[1] for e in gt.log if e[0] == 'call']
    assert calls == ['b', 'b', 'c', 'c', 'a', 'a'] * 3
    assert gt.log.count(('sync',)) == 2 * 3 * 3


def test_card_raises_without_cuda(gt, monkeypatch):
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    monkeypatch.setattr(subprocess, 'run', lambda *a, **k: pytest.fail('nvidia-smi queried without a CUDA device'))
    with pytest.raises(RuntimeError, match='no CUDA device'):
        gt.card()


def test_card_reads_one_query(gt, monkeypatch):
    calls = []

    def run(argv, **kw):
        calls.append(argv)
        return subprocess.CompletedProcess(argv, 0, stdout='NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n')

    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'get_device_name', lambda i: f'device {i}')
    monkeypatch.setattr(subprocess, 'run', run)
    assert gt.card(1) == {'name': 'device 1', 'power_limit': '700.00 W', 'max_sm_clock': '1980 MHz'}
    assert calls == [['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '1']]
