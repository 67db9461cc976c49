"""The forward Sinkhorn on score rows held on chip (sinkhorn_resident_kernel) against the streaming kernel (OG_SINK_RESIDENT=0),
its determinism, and its plan (host only)."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _ptr, stream as _stream

DEV = 'cuda:0'
PLAN_KEYS = ['resident', 'V', 'W', 'strips', 'rows_per_strip', 'pairs_per_launch', 'rows_reg', 'rows_smem', 'smem', 'occ']
SMEM_OPTIN_MAX = 227 * 1024


def _plan(B, n, m):
    out = (C.c_int64 * 10)()
    _cabi.check(_cabi.lib().og_sinkhorn_plan(B, n, m, out), 'og_sinkhorn_plan')
    return dict(zip(PLAN_KEYS, list(out)))


class _Mode:
    """og_set_sinkhorn_resident(mode) for the duration of a with-block."""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.prev = _cabi.lib().og_set_sinkhorn_resident(self.mode)

    def __exit__(self, *exc):
        _cabi.lib().og_set_sinkhorn_resident(self.prev)


def _sinkhorn(S, m, iters, mode):
    B, n, lds = S.shape
    lib = _cabi.lib()
    wsb = lib.og_sinkhorn_workspace_bytes(B, n, m)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    scores = torch.empty(B, n + 1, m + 1, device=DEV)
    with _Mode(mode):
        _cabi.check(lib.og_sinkhorn_fwd(_ptr(S), lds, n * lds, _ptr(torch.full((1,), 1.3, device=DEV)), B, n, m, iters, 1.0,
                                        _ptr(scores), _ptr(ws), wsb, _stream()), 'og_sinkhorn_fwd')
    torch.cuda.synchronize()
    return scores


def _matches(scores, threshold=0.2):
    """SuperGlue's mutual-nearest-neighbour extraction, and which of its decisions hold for any scores within `eps` of these."""
    inner = scores[:, :-1, :-1]
    top0, top1 = inner.topk(2, dim=2), inner.topk(2, dim=1)
    i0, i1 = top0.indices[..., 0], top1.indices[:, 0]
    ar0 = torch.arange(inner.shape[1], device=inner.device)[None]
    ar1 = torch.arange(inner.shape[2], device=inner.device)[None]
    mutual0 = i1.gather(1, i0) == ar0
    mutual1 = i0.gather(1, i1) == ar1
    ms0 = torch.where(mutual0, top0.values[..., 0].exp(), torch.zeros_like(top0.values[..., 0]))
    valid0 = mutual0 & (ms0 > threshold)
    valid1 = mutual1 & valid0.gather(1, i1)
    m0 = torch.where(valid0, i0, torch.full_like(i0, -1))
    m1 = torch.where(valid1, i1, torch.full_like(i1, -1))
    return m0, m1, top0, top1


@pytest.mark.gpu
@pytest.mark.parametrize('iters', [1, 20, 100])
@pytest.mark.parametrize('n,m', [(2048, 2048), (1024, 1024), (2047, 2049), (4096, 1024)])
@pytest.mark.parametrize('B', [1, 2, 3, 16])
def test_resident_matches_streaming(B, n, m, iters):
    """Scores (inputs as bench.py draws them) within 2e-5 of the streaming kernel's, the bound both meet against float64 in
    test_gpu_parity.py's test_sinkhorn_operator (the two add the column sums in different orders: a few ulps of |u| + |v|), and
    matches identical wherever a 4e-5 change of the scores cannot flip them: every decision but near-ties, whose row and column
    top-2 gaps or threshold margin are below 4e-5.  Shapes where the plan streams compare the streaming kernel with itself."""
    g = torch.Generator(device=DEV).manual_seed(B * 7919 + n + 3 * m + iters)
    lds = (m + 3) // 4 * 4
    S = torch.randn(B, n, lds, device=DEV, generator=g) * 4
    res = _sinkhorn(S, m, iters, 1)
    ref = _sinkhorn(S, m, iters, 0)
    assert torch.isfinite(res).all()
    assert float((res - ref).abs().max()) <= 2e-5
    r0, r1, top0, top1 = _matches(ref)
    o0, o1, _, _ = _matches(res)
    eps = 4e-5
    row_ok = (top0.values[..., 0] - top0.values[..., 1]) > eps
    col_ok = (top1.values[:, 0] - top1.values[:, 1]) > eps
    thr_ok = (top0.values[..., 0] - math.log(0.2)).abs() > eps
    ok0 = row_ok & col_ok.gather(1, top0.indices[..., 0]) & thr_ok
    ok1 = col_ok & ok0.gather(1, top1.indices[:, 0])
    assert ok0.float().mean() > 0.99 and ok1.float().mean() > 0.99
    assert torch.equal(o0[ok0], r0[ok0]) and torch.equal(o1[ok1], r1[ok1])


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,m,iters', [(16, 2048, 2048, 100), (3, 1024, 1024, 20), (2, 700, 513, 25)])
def test_resident_is_deterministic(B, n, m, iters):
    with _Mode(1):
        assert _plan(B, n, m)['resident'] == 1
    g = torch.Generator(device=DEV).manual_seed(11)
    lds = (m + 3) // 4 * 4
    S = torch.randn(B, n, lds, device=DEV, generator=g) * 8
    assert torch.equal(_sinkhorn(S, m, iters, 1), _sinkhorn(S, m, iters, 1))


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['uniform', 'padded', 'backward'])
@pytest.mark.parametrize('B,n,m,iters', [(16, 2048, 2048, 100), (32, 1024, 1024, 20)])
def test_streaming_is_deterministic(B, n, m, iters, form):
    """The streaming kernels (forward, padded forward at full lengths, backward) give the same bits in every run.  Their row ring
    refills a shared-memory slot by bulk copy right after the warp has read it: without the proxy fence between the two, several
    pairs of 2048 x 2048 gave run-to-run differences of up to 15 in the scores."""
    lib = _cabi.lib()
    g = torch.Generator(device=DEV).manual_seed(13)
    lds = (m + 3) // 4 * 4
    S = torch.randn(B, n, lds, device=DEV, generator=g) * 4
    dust = torch.full((1,), 1.3, device=DEV)
    wsb = lib.og_sinkhorn_workspace_bytes(B, n, m)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    lens = torch.tensor([n] * B + [m] * B, dtype=torch.int32, device=DEV)
    hist = torch.empty(lib.og_sinkhorn_hist_floats(B, n, m, iters), device=DEV)
    G = torch.randn(B, n + 1, m + 1, device=DEV, generator=g)
    bwsb = lib.og_sinkhorn_bwd_workspace_bytes(B, n, m, iters)
    bws = torch.empty(bwsb if form == 'backward' else 0, dtype=torch.uint8, device=DEV)

    def run():
        scores = torch.empty(B, n + 1, m + 1, device=DEV)
        with _Mode(0):
            if form == 'uniform':
                _cabi.check(lib.og_sinkhorn_fwd(_ptr(S), lds, n * lds, _ptr(dust), B, n, m, iters, 1.0, _ptr(scores), _ptr(ws), wsb,
                                                _stream()), 'og_sinkhorn_fwd')
            elif form == 'padded':
                _cabi.check(lib.og_sinkhorn_fwd_padded(_ptr(S), lds, n * lds, _ptr(dust), B, n, m, _ptr(lens), iters, 1.0,
                                                       _ptr(scores), _ptr(ws), wsb, _stream()), 'og_sinkhorn_fwd_padded')
            else:
                _cabi.check(lib.og_sinkhorn_train_fwd(_ptr(S), lds, n * lds, _ptr(dust), B, n, m, iters, 1.0, _ptr(scores), _ptr(hist),
                                                      _ptr(ws), wsb, _stream()), 'og_sinkhorn_train_fwd')
                dS, dd = torch.empty(B, n + 1, m + 1, device=DEV), torch.empty(1, device=DEV)
                _cabi.check(lib.og_sinkhorn_bwd(_ptr(S), lds, n * lds, _ptr(dust), B, n, m, iters, 1.0, _ptr(hist), _ptr(G), _ptr(dS),
                                                _ptr(dd), _ptr(bws), bwsb, _stream()), 'og_sinkhorn_bwd')
                scores = torch.cat([scores.flatten(), dS.flatten(), dd])
        torch.cuda.synchronize()
        return scores

    first = run()
    assert torch.isfinite(first).all()
    for _ in range(4):
        assert torch.equal(run(), first)


# BASELINE.json configs as the Sinkhorn sees them on one H100 (132 SMs): (pairs per GPU, n, m) -> resident, strips, rows per
# strip, pairs per launch.  C2's 1024-column rows pay more per held row than streaming them costs, so it streams.
BASELINE_PLANS = {
    'C1': ((1, 512, 512), (1, 65, 8, 1)),
    'C2': ((32, 1024, 1024), (0, 8, 129, 32)),
    'C3': ((16, 2048, 2048), (1, 65, 32, 2)),
    'C4': ((32, 2048, 2048), (1, 65, 32, 2)),
    'C5': ((1, 4096, 1024), (1, 129, 32, 1)),
}


def _sm_count():
    count = C.c_int(0)
    return count.value if _cabi.lib().og_device_info(C.byref(count), None, None) == 0 and count.value > 0 else 132


@pytest.mark.parametrize('config', sorted(BASELINE_PLANS))
def test_resident_plan_of_baseline_configs(config):
    (B, n, m), want = BASELINE_PLANS[config]
    with _Mode(1):
        p = _plan(B, n, m)
    if _sm_count() == 132:
        assert (p['resident'], p['strips'], p['rows_per_strip'], p['pairs_per_launch']) == want, p
    if not p['resident']:
        return
    G = 8 // p['W']
    assert p['occ'] == 1
    assert p['strips'] * p['pairs_per_launch'] <= _sm_count()                 # one CTA per SM, all co-resident
    assert p['strips'] * p['rows_per_strip'] >= n + 1 > (p['strips'] - 1) * p['rows_per_strip']
    assert G * (p['rows_reg'] + p['rows_smem']) >= p['rows_per_strip']        # every row of a strip is held
    assert p['rows_reg'] * p['V'] * 4 <= 96                                   # the registers the kernel holds rows in
    assert p['smem'] <= SMEM_OPTIN_MAX
    launches = math.ceil(B / p['pairs_per_launch'])
    assert B <= launches * p['pairs_per_launch'] < B + launches               # pairs spread evenly over the launches


@pytest.mark.parametrize('B,n,m', [(16, 2047, 2049), (1, 64, 8192), (2, 100, 4096), (3, 2048, 2048), (16, 1024, 1024)])
def test_streaming_where_residency_does_not_fit(B, n, m):
    with _Mode(1):
        assert _plan(B, n, m)['resident'] == 0


def test_switch_selects_streaming():
    with _Mode(0):
        p = _plan(2, 2048, 2048)
        assert p['resident'] == 0 and p['rows_reg'] == 0 and p['rows_smem'] == 0
    with _Mode(1):
        assert _plan(2, 2048, 2048)['resident'] == 1


def test_workspace_covers_both_forms():
    lib = _cabi.lib()
    for B, n, m in [(1, 2048, 2048), (16, 2048, 2048), (1, 512, 512), (32, 1024, 1024), (1, 4096, 1024)]:
        with _Mode(1):
            p = _plan(B, n, m)
        mpad = (m + 1 + 3) // 4 * 4
        partial_rows = max(2 * B * 32, 2 * (p['strips'] + 1) * p['pairs_per_launch'])
        assert lib.og_sinkhorn_workspace_bytes(B, n, m) >= 256 * 128 + B * (n + 1) * 4 + partial_rows * mpad * 4


def test_resident_kernels_do_not_spill():
    """Static check of the built library (cuobjdump, no GPU; OG_LIB names another build): the resident kernels keep their rows in
    registers without touching local memory (STL / LDL: spills)."""
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    path = os.environ.get('OG_LIB') or _cabi.LIB_PATH
    assert os.path.exists(path), f'library not built: {path}'
    res = subprocess.run([tool, '-sass', path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    funcs, cur = {}, None
    for line in res.stdout.splitlines():
        mt = re.match(r'\s*Function : (\S+)', line)
        if mt:
            cur = funcs.setdefault(mt.group(1), []) if 'sinkhorn_resident_kernel' in mt.group(1) else None
            continue
        mt = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P(?:\d+|T)\s+)?([A-Z0-9_.]+)', line)
        if mt and cur is not None:
            cur.append(mt.group(1).split('.')[0])
    assert len(funcs) == 3, sorted(funcs)                # <4,1>, <4,2>, <8,2>
    for name, ops in funcs.items():
        assert 'STL' not in ops and 'LDL' not in ops, name
