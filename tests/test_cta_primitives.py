"""The CTA-level conventions the tests pin bit for bit - the fixed-order block sum, the last-CTA finish of a grid-wide sum, the
bitonic sort network and its power-of-two length - are each written once, in csrc/common.cuh, and every kernel that needs one
calls it there.  CPU, on the sources.
"""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'openglue_b200', 'csrc')


def _files_matching(pattern):
    rx = re.compile(pattern)
    hits = []
    for name in sorted(os.listdir(CSRC)):
        if name.endswith(('.cu', '.cuh')):
            with open(os.path.join(CSRC, name)) as f:
                if rx.search(f.read()):
                    hits.append(name)
    return hits


def test_bitonic_network_is_written_once():
    assert _files_matching(r'for \(int size = 2; size <= \w+; size <<= 1\)') == ['common.cuh']
    assert _files_matching(r'while \(\w+ < \w+\) \w+ <<= 1;') == ['common.cuh']          # pow2_ceil


def test_block_sum_is_defined_once():
    assert _files_matching(r'__device__[^;{(]*\b\w*(block|cta)_sum\w*\s*\(') == ['common.cuh']
    assert _files_matching(r'\+= red\[w\];') == ['common.cuh']                            # the warp totals in warp order


def test_last_cta_arrival_is_written_once():
    assert _files_matching(r'atomicAdd\([^;]*\)\s*==') == ['common.cuh']
