"""How the scripts under tools/ time work on the GPU and record the card they ran on.

Importing this module puts the repository root, oracle/ and tools/ on sys.path, so a script run as ``python tools/<script>.py``
can import the package, the oracle modules and the other scripts' workload builders.
"""
from __future__ import annotations

import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tools')]


def card(index: int = 0) -> dict:
    """The name, power limit and maximum SM clock of CUDA device `index`: a speed figure is only worth something beside them.
    Raises when there is no CUDA device or nvidia-smi cannot be queried; the query reads, it never sets."""
    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: there is no card to record')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(index)],
                       capture_output=True, text=True, timeout=60, check=True).stdout
    fields = [s.strip() for s in q.strip().split(',')]
    if len(fields) != 3:
        raise RuntimeError(f'unexpected nvidia-smi output: {q!r}')
    return {'name': torch.cuda.get_device_name(index), 'power_limit': fields[1], 'max_sm_clock': fields[2]}


def events_ms(fn, iters: int, warmup: int = 0) -> float:
    """ms per call of `fn`: CUDA events around `iters` calls, after `warmup` untimed calls.  The full-device synchronisations
    before the start event and after the end event keep work that `fn` puts on a side stream inside the window."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def rounds_ms(forms: dict, iters: int, rounds: int) -> dict:
    """{name: [ms per call in each round]}: each round times every form in `forms`' order with events_ms, so forms that are
    compared see the same drift of clocks and load."""
    ms = {name: [] for name in forms}
    for _ in range(rounds):
        for name, fn in forms.items():
            ms[name].append(events_ms(fn, iters))
    return ms
