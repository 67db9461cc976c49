"""The optimiser step of the reference's training loop on the GPU: ``configure_optimizers`` (reference
models/matching_module.py:133-147: ``Adam(lr)`` + ``StepLR(step_size=1, gamma=scheduler_gamma)``, interval 'step') and
Lightning's gradient clipping (``gradient_clip_val=grad_clip`` -> ``clip_grad_norm_``) as one ``torch.optim.Optimizer``::

    opt = ClippedAdam.from_config(model, config['train'])      # replaces configure_optimizers + gradient_clip_val
    loss.backward(); opt.step()                                # clip_grad_norm_ -> Adam.step() -> StepLR.step()

``step()`` is one call of ``og_clip_adam_step`` (two kernels, ``include/openglue_b200.h``) with no host synchronisation, so it
can be captured in a CUDA graph (``GraphedTrainStep(..., optimizer=opt)``).  The arithmetic is torch's foreach
(non-capturable) Adam bit for bit; only the gradient norm's summation order differs (a deterministic fp64 reduction, rounded
once to fp32), which changes nothing while the norm stays below ``grad_clip``.

Scope: one parameter group of float32 CUDA parameters on one device; ``weight_decay``, ``amsgrad`` and ``maximize`` (never set
by the reference) are not built.  There is no CPU path.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from . import _cabi
from ._cabi import ptr, stream

__all__ = ['ClippedAdam']

_TILE = 2048                            # OG_OPTIM_TILE; a table row is og_optim_segment: param, grad, exp_avg, exp_avg_sq, step, numel, tile0


class ClippedAdam(torch.optim.Optimizer):
    """``clip_grad_norm_(params, grad_clip)`` -> ``Adam(lr, betas, eps).step()`` -> ``StepLR(step_size=1, gamma=lr_gamma).step()``.

    State lives on the device: ``exp_avg`` / ``exp_avg_sq`` per parameter, one float32 step count per parameter (as torch keeps
    them), and the learning rate in float64.  Parameters whose ``.grad`` is None are skipped and their step does not advance,
    as in torch.  ``last_grad_norm`` is a 0-dim device tensor holding what ``clip_grad_norm_`` returned for the last step (a
    view that the next step overwrites).

    ``step(skip=flag)`` (a device int32 [] flag, as ``og_train_guard`` writes it) is the same step behind the flag: when it reads
    non-zero the gradients are zeroed and nothing else changes - parameters, moments, step counts, lr and the scheduler's count
    keep their bits - without a host synchronisation.  Which parameters then have Adam state is known on the device only;
    ``state_dict()`` reads it from their step counts.

    ``get_last_lr()``, ``state_dict()`` and ``load_state_dict()`` synchronise with the device.  ``state_dict()`` returns
    ``{'optimizer': ..., 'lr_scheduler': ...}`` in exactly the layout of torch's ``Adam.state_dict()`` / ``StepLR.state_dict()``,
    so Lightning checkpoints (``optimizer_states[0]``, ``lr_schedulers[0]``) load here and this state loads into torch's objects.

    The kernels write the parameters through raw pointers; ``step()`` bumps their autograd version counters afterwards, so
    ``SuperGlue``'s packed inference weights are rebuilt.  A replayed CUDA graph that contains ``step()`` must do the same
    (``GraphedTrainStep`` does)."""

    def __init__(self, params, lr: float = 1e-4, betas=(0.9, 0.999), eps: float = 1e-8, grad_clip: float = 10.0,
                 lr_gamma: float = 0.999994, weight_decay: float = 0.0, amsgrad: bool = False, maximize: bool = False):
        if weight_decay != 0:
            raise NotImplementedError('ClippedAdam: weight_decay is not built (the reference trains with weight_decay = 0)')
        if amsgrad:
            raise NotImplementedError('ClippedAdam: amsgrad is not built (the reference trains without it)')
        if maximize:
            raise NotImplementedError('ClippedAdam: maximize is not built (the reference minimises its loss)')
        lr, eps, grad_clip, lr_gamma = float(lr), float(eps), float(grad_clip), float(lr_gamma)
        b1, b2 = (float(b) for b in betas)
        if not (lr >= 0 and math.isfinite(lr)):
            raise ValueError(f'ClippedAdam: invalid lr {lr}')
        if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0):
            raise ValueError(f'ClippedAdam: betas {betas} must lie in [0, 1)')
        if not eps >= 0:
            raise ValueError(f'ClippedAdam: invalid eps {eps}')
        if not grad_clip > 0:
            raise ValueError(f'ClippedAdam: grad_clip = {grad_clip} must be positive (the reference clips at 10.0)')
        if not lr_gamma > 0:
            raise ValueError(f'ClippedAdam: lr_gamma = {lr_gamma} must be positive')
        super().__init__(params, dict(lr=lr, betas=(b1, b2), eps=eps, weight_decay=0.0, amsgrad=False, maximize=False))
        if len(self.param_groups) != 1:
            raise ValueError('ClippedAdam takes one parameter group (the reference optimises superglue.parameters() as one group)')
        ps: List[torch.Tensor] = self.param_groups[0]['params']
        dev = ps[0].device
        for p in ps:
            if p.device.type != 'cuda' or p.dtype != torch.float32:
                raise ValueError(f'ClippedAdam needs float32 CUDA parameters (got {p.dtype} on {p.device}); there is no CPU path')
            if p.device != dev:
                raise ValueError(f'ClippedAdam needs all parameters on one device (got {dev} and {p.device})')
            if not p.is_contiguous():
                raise ValueError('ClippedAdam needs contiguous parameters')
        self.param_groups[0]['initial_lr'] = lr
        self.grad_clip, self.lr_gamma, self.dev = grad_clip, lr_gamma, dev
        lib = _cabi.lib()
        if _cabi.check_size(lib.og_optim_state_bytes(), 'og_optim_state_bytes') != 24:
            raise _cabi.OpenGlueB200Error('og_optim_state layout differs from this binding')
        with torch.cuda.device(dev):
            self._exp_avg = [torch.zeros_like(p) for p in ps]
            self._exp_avg_sq = [torch.zeros_like(p) for p in ps]
            self._steps = torch.zeros(len(ps), dtype=torch.float32, device=dev)
            # og_optim_state {double lr; float grad_norm, clip_coef; uint32 counter, sched_steps}
            self._state = torch.zeros(3, dtype=torch.float64, device=dev)
            self._state[0].fill_(lr)
        self._stepped = [False] * len(ps)          # which parameters have Adam state (torch creates it at their first step)
        self._unsure = set()                       # parameters first stepped behind a device flag: state iff their step count > 0
        self._key = None                           # (index, param pointer, grad pointer) of the uploaded segment table
        self._table = self._table_host = self._ws = None
        self._nseg = self._ntiles = 0
        self._last_idx: List[int] = []

    @staticmethod
    def config_kwargs(train_config: dict) -> dict:
        """Constructor arguments from the reference's ``train:`` config section (lr, grad_clip, scheduler_gamma)."""
        return dict(lr=float(train_config['lr']), grad_clip=float(train_config['grad_clip']),
                    lr_gamma=float(train_config['scheduler_gamma']))

    @classmethod
    def from_config(cls, model: torch.nn.Module, train_config: dict) -> 'ClippedAdam':
        """The reference's ``configure_optimizers`` + ``gradient_clip_val`` from its ``train:`` config section."""
        return cls(model.parameters(), **cls.config_kwargs(train_config))

    # ------------------------------------------------------------------ device state views
    @property
    def _lr(self) -> torch.Tensor:
        return self._state[0]

    @property
    def last_grad_norm(self) -> torch.Tensor:
        return self._state.view(torch.float32)[2]

    @property
    def _sched_steps(self) -> torch.Tensor:
        return self._state.view(torch.int32)[5]

    def get_last_lr(self) -> List[float]:
        """StepLR.get_last_lr() (synchronises)."""
        lr = float(self._lr.item())
        self.param_groups[0]['lr'] = lr
        return [lr]

    # ------------------------------------------------------------------ the step
    def _upload_table(self, idx: List[int]) -> None:
        ps = self.param_groups[0]['params']
        rows, tile = [], 0
        step0 = self._steps.data_ptr()
        for i in idx:
            p = ps[i]
            n = p.numel()
            rows.append([p.data_ptr(), p.grad.data_ptr(), self._exp_avg[i].data_ptr(), self._exp_avg_sq[i].data_ptr(), step0 + 4 * i, n, tile])
            tile += (n + _TILE - 1) // _TILE
        if tile == 0:
            raise ValueError('ClippedAdam: every parameter with a gradient is empty')
        host = torch.tensor(rows, dtype=torch.int64).reshape(-1).pin_memory()
        if self._table is None or self._table.numel() < host.numel():
            self._table = torch.empty(host.numel(), dtype=torch.int64, device=self.dev)
        wsb = _cabi.check_size(_cabi.lib().og_optim_workspace_bytes(len(idx)), 'og_optim_workspace_bytes')
        if self._ws is None or self._ws.numel() < wsb:
            self._ws = torch.empty(wsb, dtype=torch.uint8, device=self.dev)
        self._table[:host.numel()].copy_(host, non_blocking=True)
        self._table_host = host                    # pinned: alive while the copy (or a captured copy) may still read it
        self._nseg, self._ntiles = len(idx), tile

    @torch.no_grad()
    def step(self, closure=None, skip: Optional[torch.Tensor] = None):
        if skip is not None and (not torch.is_tensor(skip) or skip.dtype != torch.int32 or skip.device != self.dev or skip.numel() != 1):
            raise ValueError(f'ClippedAdam.step: skip must be a one-element int32 tensor on {self.dev}')
        loss = None
        if closure is not None:                    # Lightning's automatic optimisation: forward + backward run inside the closure
            with torch.enable_grad():
                loss = closure()
        ps = self.param_groups[0]['params']
        idx = [i for i, p in enumerate(ps) if p.grad is not None]
        with torch.cuda.device(self.dev):
            if not idx:                            # Adam skips every parameter; StepLR still steps
                if skip is not None:
                    raise ValueError('ClippedAdam.step(skip=...) needs at least one parameter with a gradient')
                self._lr.mul_(self.lr_gamma)
                self._sched_steps.add_(1)
                return loss
            key = []
            for i in idx:
                g = ps[i].grad
                if g.dtype != torch.float32 or g.device != self.dev or g.is_sparse or not g.is_contiguous():
                    raise ValueError(f'ClippedAdam: gradient {i} must be a dense contiguous float32 tensor on {self.dev}')
                key.append((i, ps[i].data_ptr(), g.data_ptr()))
            key = tuple(key)
            if key != self._key:
                self._upload_table(idx)
                self._key = key
            b1, b2 = self.param_groups[0]['betas']
            lib = _cabi.lib()
            if skip is None:
                rc = lib.og_clip_adam_step(ptr(self._table), self._nseg, self._ntiles, b1, b2, self.param_groups[0]['eps'], self.grad_clip,
                                           self.lr_gamma, ptr(self._state), ptr(self._ws), self._ws.numel(), stream(self.dev))
                _cabi.check(rc, 'og_clip_adam_step')
            else:
                rc = lib.og_clip_adam_step_guarded(ptr(self._table), self._nseg, self._ntiles, b1, b2, self.param_groups[0]['eps'],
                                                   self.grad_clip, self.lr_gamma, ptr(self._state), ptr(self._ws), self._ws.numel(),
                                                   ptr(skip), stream(self.dev))
                _cabi.check(rc, 'og_clip_adam_step_guarded')
        self._last_idx = idx
        self._stepped_now(idx, guarded=skip is not None)
        return loss

    def _stepped_now(self, idx: List[int], guarded: bool = False) -> None:
        """Parameters ``idx`` were just updated (by step() or a graph replay that contains it): they have Adam state, and
        their version counters move so that caches keyed on them (SuperGlue's packed weights) see the new values.  ``guarded``:
        the step may have been skipped on the device, so a parameter without state gets it only if its step count moved."""
        ps = self.param_groups[0]['params']
        for i in idx:
            if guarded and not self._stepped[i]:
                self._unsure.add(i)
            else:
                self._stepped[i] = True
        torch.autograd.graph.increment_version([ps[i] for i in idx])

    def _snapshot(self):
        """Device copies of the parameters and the whole optimiser state (no synchronisation)."""
        ps = self.param_groups[0]['params']
        return ([p.detach().clone() for p in ps], [m.clone() for m in self._exp_avg], [v.clone() for v in self._exp_avg_sq],
                self._steps.clone(), self._state.clone(), list(self._stepped))

    def _restore(self, snap) -> None:
        params, ms, vs, steps, state, stepped = snap
        with torch.no_grad():
            for dst, src in zip(self.param_groups[0]['params'] + self._exp_avg + self._exp_avg_sq, params + ms + vs):
                dst.copy_(src)
            self._steps.copy_(steps)
            self._state.copy_(state)
        self._stepped = list(stepped)

    # ------------------------------------------------------------------ checkpoints
    def _torch_pair(self, lr: float):
        g = self.param_groups[0]
        return _torch_pair(g['params'], lr, g['initial_lr'], g['betas'], g['eps'], self.lr_gamma)

    def state_dict(self) -> Dict[str, dict]:
        """{'optimizer': torch Adam's state_dict, 'lr_scheduler': StepLR's} (synchronises).  Moment tensors are returned by
        reference, as torch does; the step counts are CPU float32 tensors."""
        lr = float(self._lr.item())
        steps = self._steps.cpu()
        self.param_groups[0]['lr'] = lr
        for i in list(self._unsure):               # a step behind a device flag counted only if it was not skipped
            if float(steps[i]) > 0:
                self._stepped[i] = True
                self._unsure.discard(i)
        states = [{'step': steps[i].clone(), 'exp_avg': self._exp_avg[i], 'exp_avg_sq': self._exp_avg_sq[i]} if self._stepped[i] else None
                  for i in range(len(self._stepped))]
        return _torch_state_dicts(self._torch_pair(lr), states, int(self._sched_steps.item()))

    def load_state_dict(self, state_dict: Dict[str, dict]) -> None:
        """Loads ``state_dict()``'s output or a torch Adam / StepLR pair (a Lightning checkpoint's ``optimizer_states[0]`` as
        'optimizer' and ``lr_schedulers[0]`` as 'lr_scheduler').  Synchronises."""
        opt_sd, sch_sd = state_dict['optimizer'], state_dict['lr_scheduler']
        if sch_sd.get('step_size', 1) != 1:
            raise NotImplementedError(f"ClippedAdam decays lr every step (StepLR step_size=1), got step_size={sch_sd['step_size']}")
        groups = opt_sd['param_groups']
        if len(groups) != 1:
            raise ValueError(f'ClippedAdam takes one parameter group, the state has {len(groups)}')
        g = groups[0]
        if g.get('weight_decay', 0) != 0 or g.get('amsgrad', False) or g.get('maximize', False):
            raise NotImplementedError('ClippedAdam: the state uses weight_decay / amsgrad / maximize, which are not built')
        adam, _ = self._torch_pair(float(g['lr']))
        adam.load_state_dict(opt_sd)               # validates the group sizes, moves the moments to the parameters' device
        ag = adam.param_groups[0]
        me = self.param_groups[0]
        me['lr'], me['betas'], me['eps'] = float(ag['lr']), tuple(float(b) for b in ag['betas']), float(ag['eps'])
        me['initial_lr'] = float(ag.get('initial_lr', ag['lr']))
        self.lr_gamma = float(sch_sd['gamma'])
        steps = torch.zeros(len(me['params']), dtype=torch.float32)
        self._unsure = set()
        with torch.cuda.device(self.dev):
            for i, p in enumerate(me['params']):
                st = adam.state.get(p)
                self._stepped[i] = bool(st)
                if st:
                    self._exp_avg[i].copy_(st['exp_avg'])
                    self._exp_avg_sq[i].copy_(st['exp_avg_sq'])
                    steps[i] = float(st['step'])
                else:
                    self._exp_avg[i].zero_()
                    self._exp_avg_sq[i].zero_()
            self._steps.copy_(steps)
            self._lr.fill_(me['lr'])
            self._sched_steps.fill_(int(sch_sd['last_epoch']))
            torch.cuda.synchronize(self.dev)       # the CPU step tensor above is pageable: finish before it goes


def _torch_pair(params, lr: float, initial_lr: float, betas, eps: float, gamma: float):
    """torch Adam + StepLR objects over ``params`` without state: the format of their state_dicts is the checkpoint contract."""
    adam = torch.optim.Adam(params, lr=lr, betas=betas, eps=eps)
    adam.param_groups[0]['initial_lr'] = initial_lr
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=gamma)
    return adam, sched


def _torch_state_dicts(pair, states, sched_steps: int) -> Dict[str, dict]:
    """The pair's state_dicts after ``sched_steps`` scheduler steps, with per-parameter Adam state ``states`` (None: no state)."""
    adam, sched = pair
    for p, st in zip(adam.param_groups[0]['params'], states):
        if st is not None:
            adam.state[p] = st
    lr = adam.param_groups[0]['lr']
    sched.last_epoch, sched._step_count, sched._last_lr = sched_steps, sched_steps + 1, [lr]
    return {'optimizer': adam.state_dict(), 'lr_scheduler': sched.state_dict()}
