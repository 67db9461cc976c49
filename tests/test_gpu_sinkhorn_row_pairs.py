"""The resident Sinkhorn's two-rows-at-a-time sweep against the streaming kernel at shapes chosen for how the rows of a warp pair
up: odd and even rows per warp, one row per warp, the dustbin row (the strip's last, so the last row of its warp) as the second
row of a pair and alone, all rows in registers (rows_smem = 0) and some in shared memory, W = 1 and 2, B = 1, 2 and 3.  The
comparison is test_resident_matches_streaming's (2e-5, decisive matches identical), plus determinism."""
import pytest
import torch

import test_gpu_sinkhorn_resident as resident
from test_gpu_sinkhorn_resident import DEV, _Mode, _plan, _sinkhorn

# (B, n, m, iters)
CASES = [
    (1, 64, 2048, 20),       # one row per warp (none in some warps), V = 8
    (1, 65, 2047, 20),
    (1, 127, 1001, 20),      # one row per warp, V = 4
    (1, 1004, 1001, 20),     # 1 and 2 rows per warp, all in registers, V = 4
    (1, 2040, 2048, 30),     # 2, 3 and 4 rows per warp, the dustbin alone in shared memory
    (1, 2044, 2048, 20),     # 3 and 4 rows per warp, the dustbin second of a pair
    (1, 2047, 2048, 100),
    (2, 2046, 2047, 25),
    (2, 2040, 1001, 20),     # 6, 7 and 8 rows per warp, V = 4
    (3, 1023, 2048, 25),
    (1, 2040, 500, 20),      # W = 1, all rows in registers
    (2, 4095, 500, 20),      # W = 1, the dustbin alone in registers while other warps hold rows in shared memory
    (3, 4095, 500, 20),      # W = 1, 6, 7, 11 and 12 rows per warp
]


def _warp_rows(p, n):
    """Rows per warp, and where the dustbin row falls ('second' of a pair or 'alone'), from the plan's strips."""
    G = 8 // p['W']
    counts, dustbin = set(), set()
    for strip in range(p['strips']):
        r0 = strip * p['rows_per_strip']
        r1 = min(r0 + p['rows_per_strip'], n + 1)
        for grp in range(G):
            rows = list(range(r0 + grp, r1, G))
            counts.add(len(rows))
            if n in rows:
                dustbin.add('second' if rows.index(n) % 2 else 'alone')
    return counts, dustbin


def test_cases_cover_the_row_pairing():
    """Host only: every case runs resident, and together they reach each way the rows of a warp pair up."""
    seen = {'B': set(), 'W': set(), 'rows_smem>0': set(), 'rows': set(), 'dustbin': set()}
    with _Mode(1):
        for B, n, m, _ in CASES:
            p = _plan(B, n, m)
            assert p['resident'] == 1, (B, n, m, p)
            counts, dustbin = _warp_rows(p, n)
            seen['B'].add(B)
            seen['W'].add(p['W'])
            seen['rows_smem>0'].add(p['rows_smem'] > 0)
            seen['rows'] |= counts
            seen['dustbin'] |= dustbin
    assert seen['B'] == {1, 2, 3} and seen['W'] == {1, 2} and seen['rows_smem>0'] == {False, True}
    assert 1 in seen['rows'] and any(r > 1 and r % 2 for r in seen['rows']) and any(r > 0 and r % 2 == 0 for r in seen['rows'])
    assert seen['dustbin'] == {'second', 'alone'}


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,m,iters', CASES)
def test_row_pairs_match_streaming(B, n, m, iters):
    resident.test_resident_matches_streaming(B, n, m, iters)


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,m,iters', CASES[::3])
def test_row_pairs_deterministic(B, n, m, iters):
    g = torch.Generator(device=DEV).manual_seed(B + n + m)
    lds = (m + 3) // 4 * 4
    S = torch.randn(B, n, lds, device=DEV, generator=g) * 8
    assert torch.equal(_sinkhorn(S, m, iters, 1), _sinkhorn(S, m, iters, 1))
