"""Capture once, replay with static inputs: the one CUDA-graph cache of ``MatchingCore``, ``ImagePairMatcher``,
``GraphedTrainStep`` and ``ImagePairTrainStep``.  An owner keeps its graphs in a dict (key -> :class:`Entry`, in capture order)
and supplies what differs between owners: the ``key``; ``version()``, a fingerprint of the storage and values the graph baked
in (a different one captures again under the same key); the ``inputs``, copied into static buffers (float32 for floating
inputs when ``f32``, else of the input's own dtype); ``chain(static)``, the captured work; ``hold()``, storage to keep alive with
the graph; and ``guard``, training-state hooks around the warm-up and the replay (``training._WarmupGuard``)."""
from __future__ import annotations

from typing import Any, Callable, Dict, NamedTuple, Optional

import torch


class Entry(NamedTuple):
    graph: Any
    static: Dict[str, torch.Tensor]
    out: Any
    version: Any
    held: Any
    state: Any                                      # what guard.captured() returned, for guard.replayed()


def capture(inputs: Dict[str, torch.Tensor], chain: Callable, dev: torch.device, f32: bool, version: Callable,
            hold: Optional[Callable] = None, guard=None) -> Entry:
    """Static buffers, one warm-up run of ``chain``, then its capture into a new graph (not replayed)."""
    static = {k: torch.empty(v.shape, dtype=torch.float32 if v.is_floating_point() else v.dtype, device=dev) if f32
              else torch.empty_like(v) for k, v in inputs.items()}
    for k, v in inputs.items():
        static[k].copy_(v, non_blocking=True)
    if guard is not None:
        guard.save()
    chain(static)             # the warm-up builds what must not be captured: Sinkhorn tables, workspaces, kernel attributes
    torch.cuda.synchronize(dev)
    if guard is not None:
        guard.restore()
    held = None if hold is None else hold()
    graph = torch.cuda.CUDAGraph()                  # looked up at call time: tests substitute a counting class
    with torch.cuda.graph(graph):
        out = chain(static)
    state = None if guard is None else guard.captured()
    return Entry(graph, static, out, version(), held, state)    # after the warm-up, which may pack weights or grow a workspace


def run(graphs: Dict[Any, Entry], max_graphs: int, key, version: Callable, inputs: Dict[str, torch.Tensor], chain: Callable,
        dev: torch.device, f32: bool, hold: Optional[Callable] = None, guard=None):
    """Replay the graph of ``key``, capturing it first when it is missing or its version changed; the oldest capture is dropped
    beyond ``max_graphs``.  -> the graph's output buffers."""
    entry = graphs.get(key)
    if entry is not None and entry.version != version():
        del graphs[key]
        entry = None
    if entry is None:
        entry = capture(inputs, chain, dev, f32, version, hold, guard)
        while len(graphs) >= max_graphs:
            del graphs[next(iter(graphs))]
        graphs[key] = entry
    for k, v in inputs.items():
        entry.static[k].copy_(v, non_blocking=True)
    entry.graph.replay()
    if guard is not None:
        guard.replayed(entry.state)
    return entry.out
