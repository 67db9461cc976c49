"""Host-side weight preparation: fold and pack a reference ``state_dict`` into the flat fp32
buffer libopenglue_b200.so consumes (layout documented in include/openglue_b200.h).

All folds are done in float64 and rounded to fp32 once:

* eval-mode BatchNorm follows ReLU and precedes the next conv (reference models/utils.py:48-58),
  so it folds FORWARD:  W' = W . diag(s),  b' = b + W . t   with  s = gamma / sqrt(var + eps),
  t = beta - mean * s;
* ``out_proj`` (attention_gnn.py:32) is linear and feeds only ``fc.0`` (attention_gnn.py:52-55):
  W1 . [x ; Wo.o + bo] = [W1a | W1b.Wo] . [x ; o] + (b1 + W1b.bo);  with ``use_offset``
  ([x - msg ; msg]) the message half becomes (W1b - W1a);
* ``sigmoid(mix_coefs)`` (superglue.py:58-62) scales the rows of ``linear_proj``; the raw
  descriptors enter through the epilogue with weight ``1 - sigmoid(mix_coefs)``.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import _cabi

BN_EPS = 1e-5


def _bn_scale_shift(sd: Dict[str, torch.Tensor], prefix: str):
    g, b = sd[prefix + 'weight'].double(), sd[prefix + 'bias'].double()
    mu, var = sd[prefix + 'running_mean'].double(), sd[prefix + 'running_var'].double()
    s = g / torch.sqrt(var + BN_EPS)
    return s, b - mu * s


def pack_weights(state_dict: Dict[str, torch.Tensor], config: dict, ogcfg: _cabi.OgConfig,
                 dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """Return the packed CPU tensor (1-D, fp32) for ``og_superglue_forward``.  ``dtype=float64``
    keeps the folds unrounded (used by the tests to check the algebra alone)."""
    lib = _cabi.lib()
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    total = _cabi.check_size(lib.og_packed_weight_floats(ogcfg), 'og_packed_weight_floats')
    out = torch.zeros(total, dtype=dtype)
    d = int(config['descriptor_dim'])
    use_offset = bool(config['attention_gnn'].get('use_offset', False))

    def put(tid: int, index: int, t: torch.Tensor):
        off = lib.og_packed_offset(ogcfg, tid, index)
        if off < 0:
            _cabi.check(int(off), 'og_packed_offset')
        flat = t.reshape(-1).to(dtype)
        out[off:off + flat.numel()] = flat

    # keypoint encoder: conv 3i, (relu), bn 3i+2; BN i folds into conv i+1
    n_lin = ogcfg.num_hidden + 1
    s_prev = t_prev = None
    for i in range(n_lin):
        w = sd[f'positional_encoding.encoder.{3 * i}.weight'][:, :, 0].double()
        b = sd[f'positional_encoding.encoder.{3 * i}.bias'].double()
        if s_prev is not None:
            b = b + w @ t_prev
            w = w * s_prev[None, :]
        put(_cabi.OG_T_KENC_W, i, w)
        put(_cabi.OG_T_KENC_B, i, b)
        if i < n_lin - 1:
            s_prev, t_prev = _bn_scale_shift(sd, f'positional_encoding.encoder.{3 * i + 2}.')

    for layer in range(ogcfg.num_layers):
        p = f'attention_gnn.layers.{layer}.module.'
        wq, wk, wv = (sd[p + f'mha.in_proj_{c}.weight'][:, :, 0].double() for c in 'qkv')
        bq, bk, bv = (sd[p + f'mha.in_proj_{c}.bias'].double() for c in 'qkv')
        put(_cabi.OG_T_QKV_W, layer, torch.cat([wq, wk, wv], 0))
        put(_cabi.OG_T_QKV_B, layer, torch.cat([bq, bk, bv], 0))
        wo, bo = sd[p + 'mha.out_proj.weight'][:, :, 0].double(), sd[p + 'mha.out_proj.bias'].double()
        w1, b1 = sd[p + 'fc.0.weight'][:, :, 0].double(), sd[p + 'fc.0.bias'].double()
        w1a, w1b = w1[:, :d], w1[:, d:]
        wm = (w1b - w1a) if use_offset else w1b            # what multiplies the attention message
        put(_cabi.OG_T_FC1_W, layer, torch.cat([w1a, wm @ wo], 1))
        put(_cabi.OG_T_FC1_B, layer, b1 + wm @ bo)
        s, t = _bn_scale_shift(sd, p + 'fc.2.')
        w2, b2 = sd[p + 'fc.3.weight'][:, :, 0].double(), sd[p + 'fc.3.bias'].double()
        put(_cabi.OG_T_FC2_W, layer, w2 * s[None, :])
        put(_cabi.OG_T_FC2_B, layer, b2 + w2 @ t)

    wp, bp = sd['linear_proj.weight'][:, :, 0].double(), sd['linear_proj.bias'].double()
    if config.get('residual', False):
        alpha = torch.sigmoid(sd['mix_coefs'].double()).reshape(-1)
        put(_cabi.OG_T_PROJ_W, 0, wp * alpha[:, None])
        put(_cabi.OG_T_PROJ_B, 0, bp * alpha)
        put(_cabi.OG_T_PROJ_RMIX, 0, 1.0 - alpha)
    else:
        put(_cabi.OG_T_PROJ_W, 0, wp)
        put(_cabi.OG_T_PROJ_B, 0, bp)
        put(_cabi.OG_T_PROJ_RMIX, 0, torch.zeros(d, dtype=torch.float64))
    put(_cabi.OG_T_DUSTBIN, 0, sd['dustbin_score'].double().reshape(1))
    return out
