"""Drop-in replacement for the reference's ``models.superglue.superglue.SuperGlue``.

Same constructor config, same ``state_dict`` keys and shapes (so reference checkpoints load,
reference inference.py:71-75) and the same ``forward(data) -> dict`` contract
(reference superglue.py:29-72); the arithmetic runs in libopenglue_b200.so (hand-written
sm_90a CUDA behind a C ABI, include/openglue_b200.h).  ``MatchingCore`` adds the match
extraction of ``MatchingTrainingModule.forward`` (reference models/matching_module.py:149-187).

There is no CPU or PyTorch fallback for the kernels: a missing library or a non-CUDA
device is an error, not a slow path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import _cabi, _graphs
from ._cabi import ptr, stream
from .packing import pack_weights

__all__ = ['SuperGlue', 'MatchingCore', 'PendingMatches', 'is_padded', 'padded_inputs', 'padded_lengths']

# Counts (re)registrations of parameters, buffers and submodules on any module: ``conv.weight = nn.Parameter(...)`` or
# ``bn.running_mean = t`` replaces a tensor object, which a cached list of a SuperGlue's tensors would not see.
_registrations = 0


def _count_registration(*_):
    global _registrations
    _registrations += 1


for _register in (torch.nn.modules.module.register_module_parameter_registration_hook,
                  torch.nn.modules.module.register_module_buffer_registration_hook,
                  torch.nn.modules.module.register_module_module_registration_hook):
    _register(_count_registration)


def is_padded(data: dict) -> bool:
    """Whether ``data`` is a padded batch: pairs with their own keypoint counts ``num_keypoints0`` / ``num_keypoints1``."""
    return 'num_keypoints0' in data or 'num_keypoints1' in data


def padded_lengths(data: dict, B: int, n: int, m: int) -> Dict[str, torch.Tensor]:
    """``num_keypoints0`` / ``num_keypoints1`` of a padded batch as int32 [B], where the caller keeps them.  Host lengths are
    checked against the capacities n, m; device lengths are not (the kernels clamp them into range)."""
    if 'num_keypoints0' not in data or 'num_keypoints1' not in data:
        raise ValueError('a padded batch needs both num_keypoints0 and num_keypoints1')
    out = {}
    for idx, cap in ((0, n), (1, m)):
        t = data[f'num_keypoints{idx}']
        t = t.detach() if torch.is_tensor(t) else torch.as_tensor(t)
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool or tuple(t.shape) != (B,):
            raise ValueError(f'num_keypoints{idx} must be an integer tensor of shape [{B}], got {t.dtype} {tuple(t.shape)}')
        if t.device.type == 'cpu':
            lo, hi = int(t.min()), int(t.max())
            if lo < 1 or hi > cap:
                raise ValueError(f'num_keypoints{idx} must lie in [1, {cap}] (the capacity), got values in [{lo}, {hi}]')
        out[f'num_keypoints{idx}'] = t.to(torch.int32)
    return out


def padded_inputs(data: dict, B: int, n: int, m: int) -> Dict[str, torch.Tensor]:
    """A padded batch's per-pair inputs, where the caller keeps them: ``num_keypoints0`` / ``num_keypoints1`` as int32 [B]
    (:func:`padded_lengths`) and ``image0_size`` / ``image1_size`` as float32 [B, 2] (W, H) per pair (a batch-wide size, or the
    image tensors' own, broadcast)."""
    out = padded_lengths(data, B, n, m)
    for idx in (0, 1):
        size = data.get(f'image{idx}_size')
        if 'image0' in data and 'image1' in data:
            size = None
        if torch.is_tensor(size) and size.dim() == 2:
            if tuple(size.shape) != (B, 2):
                raise ValueError(f'image{idx}_size must be [{B}, 2] (W, H per pair), got {tuple(size.shape)}')
            out[f'image{idx}_size'] = size.detach().to(torch.float32)
        else:
            w, h = SuperGlue._image_wh(data, idx)
            out[f'image{idx}_size'] = torch.tensor([[w, h]], dtype=torch.float32).expand(B, 2)
    return out


_MATCHER_KEYS = ('keypoints0', 'keypoints1', 'side_info0', 'side_info1', 'local_descriptors0', 'local_descriptors1')


def _matcher_inputs(data: dict):
    """A batch as the inputs of a captured matcher step -> ({name: tensor}, key constants): the six per-keypoint tensors plus a
    padded batch's lengths and per-pair sizes (:func:`padded_inputs`); a uniform batch's image sizes, plain floats baked into
    the graph, are the constants ``{'image0_size': (W, H), 'image1_size': (W, H)}``, read next to the tensors."""
    tensors = {k: data[k] for k in _MATCHER_KEYS}
    if is_padded(data):
        k0, k1 = tensors['keypoints0'], tensors['keypoints1']
        tensors.update(padded_inputs(data, k0.shape[0], k0.shape[1], k1.shape[1]))
        return tensors, {}
    return tensors, {'image0_size': SuperGlue._image_wh(data, 0), 'image1_size': SuperGlue._image_wh(data, 1)}


# The autograd drop-in's outputs feed losses written against the reference layout, which read every pair's dustbins at
# scores[:, -1, :] / scores[:, :, -1]: wrong for a padded pair, whose dustbins sit at its own lengths.
_TRAIN_PADDED_MSG = ('openglue_b200: SuperGlue.forward / run take padded batches (num_keypoints0 / num_keypoints1) in eval mode only. '
                     'To train on a padded batch use openglue_b200.training.GraphedTrainStep or TrainStep with openglue_b200.criterion, whose '
                     "loss reads each pair's own dustbin row and column")


def _feed_forward_params(*sizes: int) -> nn.Sequential:
    """Parameter container with the reference FeedForwardNet's key layout (models/utils.py:48-58):
    index 3i = Conv1d(k=1), 3i+1 = ReLU, 3i+2 = BatchNorm1d, last = Conv1d.  Never called."""
    layers = []
    for i in range(1, len(sizes) - 1):
        layers += [nn.Conv1d(sizes[i - 1], sizes[i], kernel_size=1), nn.ReLU(inplace=True), nn.BatchNorm1d(sizes[i])]
    layers.append(nn.Conv1d(sizes[-2], sizes[-1], kernel_size=1))
    return nn.Sequential(*layers)


class _Holder(nn.Module):
    """Plain namespace module (keeps state_dict prefixes identical to the reference's)."""


def _gnn_params(num_stages: int, d: int) -> nn.Module:
    gnn = _Holder()
    gnn.layers = nn.ModuleList()
    for _ in range(2 * num_stages):                       # even = self, odd = cross (attention_gnn.py:84-88)
        layer, module, mha = _Holder(), _Holder(), _Holder()
        for name in ('in_proj_q', 'in_proj_k', 'in_proj_v', 'out_proj'):
            setattr(mha, name, nn.Conv1d(d, d, kernel_size=1))
        module.mha = mha
        module.fc = _feed_forward_params(2 * d, 2 * d, d)
        layer.module = module
        gnn.layers.append(layer)
    return gnn


class SuperGlue(nn.Module):
    """H100-native (sm_90a) matching core behind the reference's module API.

    Extra (optional) config keys, ignored by the reference: ``precision`` ('fp16x3' (default): wgmma tensor cores,
    every contraction as three products of fp16 hi/lo operands with power-of-two tensor scales (head_dim 64; other
    shapes run as 'tf32x3') | 'tf32x3': the same scheme on tf32 hi/lo operands, half the MMA rate | 'fp32': CUDA-core
    FFMA everywhere),
    ``match_threshold`` (used by :class:`MatchingCore`).
    """

    def __init__(self, config: dict):
        super().__init__()
        self.config: dict = config
        d = config['descriptor_dim']
        pe, gnn = config['positional_encoding'], config['attention_gnn']
        if pe.get('encoder_name', 'FeedForwardNet') != 'FeedForwardNet':
            # same error type the reference raises for an unknown encoder (models/superglue/__init__.py:40-42)
            raise NameError(f"{pe['encoder_name']} positional encoder is not provided by openglue_b200 "
                            "(only 'FeedForwardNet')")
        if gnn.get('attention', 'softmax') != 'softmax':
            raise ValueError(f"Attention type {gnn['attention']} is not supported (only 'softmax').")
        if gnn.get('embed_dim', d) != d or pe.get('output_size', d) != d:
            raise ValueError('embed_dim / positional_encoding.output_size must equal descriptor_dim')
        hidden = list(pe.get('hidden_layers_sizes') or [])
        self.positional_encoding = _Holder()
        self.positional_encoding.encoder = _feed_forward_params(pe.get('side_info_size', 1) + 2, *hidden, d)
        self.attention_gnn = _gnn_params(gnn['num_stages'], d)
        self.residual = config.get('residual', False)
        if self.residual:
            self.mix_coefs = nn.parameter.Parameter(torch.zeros(d, 1))
        self.linear_proj = nn.Conv1d(d, d, kernel_size=1)
        self.dustbin_score = nn.Parameter(torch.tensor(float(config['dustbin_score_init'])))

        self._packed: Optional[torch.Tensor] = None
        self._packed_key = None
        self._packed_hi: Optional[torch.Tensor] = None
        self._packed_lo: Optional[torch.Tensor] = None
        self._packed_h16 = self._packed_l16 = self._meta16 = None
        self._workspace: Optional[torch.Tensor] = None
        self._ogcfg: Optional[_cabi.OgConfig] = None
        self.last_launches = 0

        weights_path = config.get('weights', None)
        if weights_path is not None:
            print('SuperGlue loading... ', self.load_state_dict(torch.load(str(weights_path), map_location='cpu')))

    # ------------------------------------------------------------------ weights
    def _precision(self) -> int:
        return {'fp32': _cabi.OG_PREC_FP32, 'tf32x3': _cabi.OG_PREC_TF32X3,
                'fp16x3': _cabi.OG_PREC_FP16X3}[self.config.get('precision', 'fp16x3')]

    def og_config(self) -> _cabi.OgConfig:
        return _cabi.make_config(self.config, self.config.get('match_threshold', 0.2), self._precision())

    def _bump_alloc(self) -> None:
        """Device buffers whose addresses a captured CUDA graph bakes in (workspace, packed weights and their operand
        splits) were reallocated: graphs captured against the old addresses must not be replayed."""
        self._alloc_gen = getattr(self, '_alloc_gen', 0) + 1

    def invalidate_packed(self) -> None:
        self._packed = None

    def load_state_dict(self, *args, **kwargs):
        self._packed = None
        self._tensors = None
        self._epoch = getattr(self, '_epoch', 0) + 1
        return super().load_state_dict(*args, **kwargs)

    def train(self, mode: bool = True):
        if mode:
            self._packed = None
        return super().train(mode)

    def _apply(self, fn, *args, **kwargs):               # .to() / .cuda() / .float(): storages move, the packed copy is stale
        self._packed = None
        self._tensors = None
        self._epoch = getattr(self, '_epoch', 0) + 1
        return super()._apply(fn, *args, **kwargs)

    def _weights_version(self):
        """Cheap fingerprint of the 333 parameter / buffer tensors (runs on every forward, ~50 us): in-place updates bump a
        tensor's ``_version`` (monotonic, so the sum changes), moves go through ``_apply`` / ``load_state_dict``, and the
        storage addresses of ALL tensors catch ``p.data = new`` / ``vector_to_parameters`` / EMA swaps on any of them.  The
        tensor list is collected again after any module registers a parameter, buffer or submodule (a replaced tensor)."""
        ts = getattr(self, '_tensors', None)
        if ts is None or self._tensors_at != _registrations:
            ts = self._tensors = list(self.parameters()) + list(self.buffers())
            self._tensors_at = _registrations
        ver = ptr = 0
        for i, t in enumerate(ts):
            ver += t._version
            ptr ^= t.data_ptr() * (2 * i + 1)
        return (getattr(self, '_epoch', 0), ver, ptr & 0xFFFFFFFFFFFFFFFF)

    def packed_weights(self, device: torch.device) -> torch.Tensor:
        """Folded + packed weights on ``device`` (cached; rebuilt when a parameter changes)."""
        key = (self._weights_version(), str(device), self._precision())
        if self._packed is None or self._packed_key != key:
            self._ogcfg = self.og_config()
            self._packed = pack_weights(self.state_dict(), self.config, self._ogcfg).to(device)
            self._packed_hi = self._packed_lo = None
            self._packed_h16 = self._packed_l16 = self._meta16 = None
            self._bump_alloc()
            if self._precision() != _cabi.OG_PREC_FP32:        # operand split for the tensor-core kernels
                self._packed_hi, self._packed_lo = torch.empty_like(self._packed), torch.empty_like(self._packed)
                with torch.cuda.device(device):
                    _cabi.check(_cabi.lib().og_split_tf32(ptr(self._packed), ptr(self._packed_hi), ptr(self._packed_lo), self._packed.numel(),
                                                          stream(device)), 'og_split_tf32')
            if self._precision() == _cabi.OG_PREC_FP16X3:      # fp16 hi/lo split of the GNN weights + per-tensor scales / norms
                lib = _cabi.lib()
                self._packed_h16 = torch.zeros(self._packed.numel(), dtype=torch.float16, device=device)
                self._packed_l16 = torch.zeros_like(self._packed_h16)
                self._meta16 = torch.zeros(max(int(lib.og_f16_meta_floats(self._ogcfg)), 4), dtype=torch.float32, device=device)
                with torch.cuda.device(device):
                    _cabi.check(lib.og_pack_f16(self._ogcfg, ptr(self._packed), ptr(self._packed_h16), ptr(self._packed_l16), ptr(self._meta16),
                                                stream(device)), 'og_pack_f16')
            self._packed_key = key
        return self._packed

    # ------------------------------------------------------------------ forward
    _HEAD_DIMS = (8, 16, 32, 64)                         # the head sizes the attention kernels are built for

    def _check_head_dim(self) -> None:
        """Raise before any kernel runs (and before train mode moves a BatchNorm buffer) when descriptor_dim / num_heads is not a
        head size the attention kernels are built for.  Construction and load_state_dict accept such configs, so checkpoints can
        still be loaded and converted."""
        d, H = self.config['descriptor_dim'], self.config['attention_gnn']['num_heads']
        if d % H or d // H not in self._HEAD_DIMS:
            raise ValueError(f'head_dim = descriptor_dim / num_heads = {d} / {H} is not supported: openglue_b200 builds attention '
                             f'for head_dim in {self._HEAD_DIMS}')

    @staticmethod
    def _image_wh(data: dict, idx: int):
        """reference superglue.py:35-38: image tensor [..., H, W] or image{idx}_size = (W, H)."""
        if 'image0' in data and 'image1' in data:
            sz = data[f'image{idx}'].size()
            return float(sz[-1]), float(sz[-2])
        w, h = data[f'image{idx}_size'][:2]
        return float(w), float(h)

    def run(self, data: dict, want_matches: bool, want_context: bool = True,
            match_threshold: Optional[float] = None) -> Dict[str, torch.Tensor]:
        """The eval-mode forward pass (and the matches of ``MatchingCore``).  A padded batch (``data`` with ``num_keypoints0`` /
        ``num_keypoints1``) has the capacities N, M as its keypoint dimensions; pair b owns rows [0, n_b) / [0, m_b), and its
        outputs are those of the pair run alone: ``scores[b, :n_b+1, :m_b+1]`` (dustbins at n_b and m_b), ``-inf`` elsewhere;
        matches -1 and matching scores 0 past the lengths; context-descriptor columns past them 0."""
        padded = is_padded(data)
        if self.training and padded:
            raise NotImplementedError(_TRAIN_PADDED_MSG)
        if self.training:
            raise RuntimeError('openglue_b200.SuperGlue.run is the fused eval-mode path; in train() mode call forward() '
                               '(openglue_b200.training: batch-statistics BatchNorm + the explicit backward pass)')
        self._check_head_dim()
        k0, k1 = data['keypoints0'], data['keypoints1']
        dev = k0.device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200.SuperGlue needs CUDA tensors (sm_90a); there is no CPU path')

        def prep(t, last):
            t = t.detach()
            if t.dtype != torch.float32:
                t = t.float()
            if t.shape[-1] != last:
                raise ValueError(f'expected last dimension {last}, got {tuple(t.shape)}')
            return t.contiguous()

        d = self.config['descriptor_dim']
        s_dim = self.config['positional_encoding'].get('side_info_size', 1)
        k0, k1 = prep(k0, 2), prep(k1, 2)
        d0, d1 = prep(data['local_descriptors0'], d), prep(data['local_descriptors1'], d)
        s0, s1 = prep(data['side_info0'], s_dim), prep(data['side_info1'], s_dim)
        B, n, m = k0.shape[0], k0.shape[1], k1.shape[1]
        if k1.shape[0] != B or d0.shape[:2] != (B, n) or d1.shape[:2] != (B, m) or s0.shape[:2] != (B, n) \
                or s1.shape[:2] != (B, m):
            raise ValueError('inconsistent batch / keypoint counts in data')
        if n == 0 or m == 0:
            raise ValueError('empty keypoint set')
        if padded:
            extra = padded_inputs(data, B, n, m)
            lens = torch.cat([extra['num_keypoints0'].to(dev), extra['num_keypoints1'].to(dev)])
            pair_wh = torch.cat([extra['image0_size'].to(dev), extra['image1_size'].to(dev)], 1).contiguous()
        else:
            w0, h0 = self._image_wh(data, 0)
            w1, h1 = self._image_wh(data, 1)

        lib = _cabi.lib()
        with torch.cuda.device(dev):
            packed = self.packed_weights(dev)
            cfg = self._ogcfg
            if match_threshold is not None and float(match_threshold) != cfg.match_threshold:
                cfg = _cabi.OgConfig.from_buffer_copy(cfg)             # per call: never written back into the shared config
                cfg.match_threshold = float(match_threshold)
            ws_query = lib.og_workspace_bytes_padded if padded else lib.og_workspace_bytes
            ws_bytes = _cabi.check_size(ws_query(cfg, B, n, m), 'og_workspace_bytes')
            if self._workspace is None or self._workspace.numel() < ws_bytes or self._workspace.device != dev:
                self._workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                self._bump_alloc()
            scores = torch.empty(B, n + 1, m + 1, dtype=torch.float32, device=dev)
            out = {'scores': scores}
            ctx0 = ctx1 = None
            if want_context:
                ctx0 = torch.empty(B, d, n, dtype=torch.float32, device=dev)
                ctx1 = torch.empty(B, d, m, dtype=torch.float32, device=dev)
                out['context_descriptors0'], out['context_descriptors1'] = ctx0, ctx1
            m0 = ms0 = m1 = ms1 = None
            if want_matches:
                m0 = torch.empty(B, n, dtype=torch.int64, device=dev)
                ms0 = torch.empty(B, n, dtype=torch.float32, device=dev)
                m1 = torch.empty(B, m, dtype=torch.int64, device=dev)
                ms1 = torch.empty(B, m, dtype=torch.float32, device=dev)
                out.update(matches0=m0, matching_scores0=ms0, matches1=m1, matching_scores1=ms1)
            outs = (ptr(ctx0), ptr(ctx1), ptr(scores), ptr(m0), ptr(ms0), ptr(m1), ptr(ms1), ptr(self._workspace), ws_bytes, stream(dev))
            if padded:
                rc = lib.og_superglue_forward_padded(cfg, ptr(packed), ptr(self._packed_hi), ptr(self._packed_lo), ptr(self._packed_h16),
                                                     ptr(self._packed_l16), ptr(self._meta16), B, n, m, ptr(lens), ptr(pair_wh), ptr(k0),
                                                     ptr(k1), ptr(s0), ptr(s1), ptr(d0), ptr(d1), *outs)
                _cabi.check(rc, 'og_superglue_forward_padded')
                self.last_launches = lib.og_last_forward_launches()
                return out
            wh = (C.c_float * 4)(w0, h0, w1, h1)
            tail = (B, n, m, ptr(k0), ptr(k1), ptr(s0), ptr(s1), ptr(d0), ptr(d1), wh, *outs)
            if cfg.precision == _cabi.OG_PREC_FP16X3:
                rc = lib.og_superglue_forward_f16(cfg, ptr(packed), ptr(self._packed_hi), ptr(self._packed_lo), ptr(self._packed_h16),
                                                  ptr(self._packed_l16), ptr(self._meta16), *tail)
            else:
                rc = lib.og_superglue_forward(cfg, ptr(packed), ptr(self._packed_hi), ptr(self._packed_lo), *tail)
            _cabi.check(rc, 'og_superglue_forward')
            self.last_launches = lib.og_last_forward_launches()
        return out

    def forward(self, data: dict) -> Dict[str, torch.Tensor]:
        """-> {'context_descriptors0' [B,d,N], 'context_descriptors1' [B,d,M], 'scores' [B,N+1,M+1]}.
        In ``train()`` mode the outputs are differentiable with respect to every parameter and the local descriptors
        (BatchNorm uses batch statistics and updates its running buffers, as the reference module does in training_step)."""
        if self.training:
            if is_padded(data):
                raise NotImplementedError(_TRAIN_PADDED_MSG)
            from .training import train_forward
            return train_forward(self, data)
        return self.run(data, want_matches=False)


class PendingMatches:
    """Result of :meth:`MatchingCore.submit`: host tensors that become valid at :meth:`wait`."""

    def __init__(self, result: Dict[str, torch.Tensor], done: torch.cuda.Event):
        self._result, self._done = result, done

    def wait(self) -> Dict[str, torch.Tensor]:
        self._done.synchronize()
        return self._result


class MatchingCore(nn.Module):
    """``SuperGlue`` + mutual-argmax match extraction: what ``MatchingTrainingModule.forward``
    (reference models/matching_module.py:149-187) computes from prepared features, fused into the
    same C-ABI call.  Accepts host (CPU) tensors too: they are copied to ``device`` (pinned ->
    non-blocking) and ``matches0`` / ``matching_scores0`` come back on the host.

    ``use_cuda_graph=True`` captures the whole launch schedule (~177 kernels at 9 stages) once per
    (batch, N, M) into a CUDA graph with static input / output buffers and replays it: for small
    batches the path is launch-latency-bound (1 pair, N=M=512: 3.3 ms eager).

    Padded batches (``num_keypoints0`` / ``num_keypoints1``, see :meth:`SuperGlue.run`) take every path; their lengths and
    per-pair image sizes are copied into the graph's static buffers like the other inputs, so one graph per capacity (B, N, M)
    serves every set of lengths and sizes."""

    def __init__(self, superglue: SuperGlue, match_threshold: float = 0.2, device: Optional[torch.device] = None,
                 use_cuda_graph: bool = False):
        super().__init__()
        self.superglue = superglue
        self.match_threshold = float(match_threshold)           # per core; the shared SuperGlue's config is not touched
        self.device = torch.device(device) if device is not None else None
        self.use_cuda_graph = use_cuda_graph
        self._graphs: Dict[tuple, _graphs.Entry] = {}
        self.max_graphs = 4                                     # captured shapes kept (alternating shapes do not re-capture)

    _TENSOR_KEYS = _MATCHER_KEYS
    _OUT_KEYS = ('matches0', 'matching_scores0', 'matches1', 'matching_scores1')

    def _run_graph(self, data: dict, dev: torch.device) -> Dict[str, torch.Tensor]:
        """Replay (capturing on first use) the CUDA graph for this shape; inputs are copied into its static buffers."""
        sg = self.superglue
        inputs, consts = _matcher_inputs(data)
        # the precision picks the captured kernels and packed-weight forms: a switch in config['precision'] repacks only at the
        # next run, so the version cannot see it yet
        key = (tuple(tuple(data[k].shape) for k in _MATCHER_KEYS), tuple(consts.values()), str(dev), sg._precision(),
               self.match_threshold)
        # workspace / packed weights reallocated (by a bigger call, or another core sharing the SuperGlue) or weights changed
        version = lambda: (getattr(sg, '_alloc_gen', 0), sg._weights_version())
        chain = lambda s: sg.run({**s, **consts}, want_matches=True, want_context=False, match_threshold=self.match_threshold)
        return _graphs.run(self._graphs, self.max_graphs, key, version, inputs, chain, dev, f32=True)

    def forward(self, data: dict, want_scores: bool = False, borrow: bool = False) -> Dict[str, torch.Tensor]:
        """``borrow=True`` (device input, CUDA-graph mode): return the graph's own output buffers instead of copies; they are
        overwritten by the next call on this core (use it when the results are consumed on the same stream right away)."""
        host = data['keypoints0'].device.type == 'cpu'
        dev = (self.device or torch.device('cuda', torch.cuda.current_device())) if host else data['keypoints0'].device
        keys = self._OUT_KEYS + (('scores',) if want_scores else ())
        if self.use_cuda_graph:
            with torch.cuda.device(dev):
                out = self._run_graph(data, dev)
            res = {k: out[k] for k in keys}
            if not host and not borrow:             # the graph's output buffers are overwritten by the next replay
                res = {k: v.clone() for k, v in res.items()}
        else:
            if host:
                data = dict(data)
                for k in self._TENSOR_KEYS:
                    data[k] = data[k].to(dev, non_blocking=True)
            out = self.superglue.run(data, want_matches=True, want_context=False, match_threshold=self.match_threshold)
            res = {k: out[k] for k in keys}
        if host:
            res = {k: v.to('cpu', non_blocking=True) for k, v in res.items()}
            torch.cuda.current_stream(dev).synchronize()
        return res

    # ------------------------------------------------------------------ pipelined host API
    def submit(self, data: dict) -> PendingMatches:
        """Asynchronous form of ``forward`` for HOST batches (serving loop).  The H2D copy of this batch runs on an
        upload stream into one of two device input-buffer sets while the previous batch is still computing; the
        kernels run on the current (compute) stream; the D2H copy of the matches runs on a download stream behind
        them.  ``submit`` returns at once; ``.wait()`` yields the dict ``forward`` returns for host input.  Keep at
        most two batches in flight: the result buffers of a slot are reused by the second-next ``submit``."""
        if data['keypoints0'].device.type != 'cpu':
            raise ValueError('submit() takes host (CPU, ideally pinned) tensors; use forward() for device tensors')
        dev = self.device or torch.device('cuda', torch.cuda.current_device())
        with torch.cuda.device(dev):
            if not hasattr(self, '_pipe'):
                self._pipe = {'h2d': torch.cuda.Stream(dev), 'd2h': torch.cuda.Stream(dev), 'slot': 0,
                              'bufs': [None, None], 'free': [None, None], 'out': [None, None]}
            pipe = self._pipe
            slot = pipe['slot']
            pipe['slot'] ^= 1
            compute = torch.cuda.current_stream(dev)
            shapes = tuple(tuple(data[k].shape) for k in self._TENSOR_KEYS)
            if pipe['bufs'][slot] is None or pipe['bufs'][slot][0] != shapes:
                pipe['bufs'][slot] = (shapes, {k: torch.empty(data[k].shape, dtype=torch.float32, device=dev)
                                               for k in self._TENSOR_KEYS})
                pipe['out'][slot] = None
                # fresh blocks may be recycled from tensors the compute stream is still using (the allocator only
                # orders reuse within one stream): the upload stream must not write them before that work is done
                pipe['h2d'].wait_stream(compute)
            bufs = pipe['bufs'][slot][1]
            with torch.cuda.stream(pipe['h2d']):
                if pipe['free'][slot] is not None:
                    pipe['h2d'].wait_event(pipe['free'][slot])       # the kernels that last read this buffer set are done
                for k in self._TENSOR_KEYS:
                    bufs[k].copy_(data[k], non_blocking=True)
                landed = torch.cuda.Event()
                landed.record(pipe['h2d'])
            compute.wait_event(landed)
            dev_data = dict(data)
            dev_data.update(bufs)
            if self.use_cuda_graph:
                out = self._run_graph(dev_data, dev)
            else:
                out = self.superglue.run(dev_data, want_matches=True, want_context=False, match_threshold=self.match_threshold)
            computed = torch.cuda.Event()
            computed.record(compute)
            pipe['free'][slot] = computed
            if pipe['out'][slot] is None:
                pipe['out'][slot] = {k: torch.empty(out[k].shape, dtype=out[k].dtype).pin_memory() for k in self._OUT_KEYS}
            host_out = pipe['out'][slot]
            with torch.cuda.stream(pipe['d2h']):
                pipe['d2h'].wait_event(computed)
                for k in self._OUT_KEYS:
                    host_out[k].copy_(out[k], non_blocking=True)
                done = torch.cuda.Event()
                done.record(pipe['d2h'])
            # the device-side results (graph-static, or allocator blocks of the compute stream) may be overwritten by
            # later kernels only once they have been read back: a 0.4 MB copy, so this costs the pipeline nothing
            compute.wait_event(done)
        return PendingMatches(host_out, done)
