"""Time og_sinkhorn_fwd with the resident kernel against the streaming kernel, the two alternating in one process.

    python tools/sinkhorn_timing.py [--launches 20] [--rounds 3] [--out DIR] [--against OTHER_LIB]

For each shape (the BASELINE workloads' Sinkhorn, one pair at the headline size, and two pairs of 2048 x 4096 for the band
2048 < m <= 4096, which only the streaming kernel runs) it prints the plan of each form, the median over `rounds` rounds of the
mean CUDA-event time of `launches` back-to-back launches, the largest score difference between the two forms and whether two
resident launches gave identical bits.  --against measures the same shapes in a second process on
another build of the library (OG_LIB, such as a parent commit's) and prints both builds' times and whether their streaming
outputs are bit-identical.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys

import torch

from gpu_timing import card, events_ms  # first: it makes the package importable
from openglue_b200 import _cabi
from openglue_b200._cabi import ptr, stream

# (label, pairs, n, m, iterations)
SHAPES = [('C3', 16, 2048, 2048, 100), ('C2', 32, 1024, 1024, 100), ('C5', 1, 4096, 1024, 50), ('C1', 1, 512, 512, 20),
          ('1 pair 2048', 1, 2048, 2048, 100), ('2048x4096', 2, 2048, 4096, 100)]


def plan(lib, B, n, m):
    out = (C.c_int64 * 10)()
    _cabi.check(lib.og_sinkhorn_plan(B, n, m, out), 'og_sinkhorn_plan')
    keys = ['resident', 'V', 'W', 'strips', 'rows_per_strip', 'pairs_per_launch', 'rows_reg', 'rows_smem', 'smem', 'occ']
    return dict(zip(keys, list(out)))


def measure(launches, rounds, quiet=False):
    lib = _cabi.lib()
    dev = 'cuda:0'
    results = []
    for label, B, n, m, T in SHAPES:
        g = torch.Generator(device=dev).manual_seed(7)
        lds = (m + 3) // 4 * 4
        S = torch.randn(B, n, lds, device=dev, generator=g) * 4
        dust = torch.ones(1, device=dev)
        wsb = lib.og_sinkhorn_workspace_bytes(B, n, m)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        outs = {1: torch.empty(B, n + 1, m + 1, device=dev), 0: torch.empty(B, n + 1, m + 1, device=dev)}

        def run(mode, out):
            lib.og_set_sinkhorn_resident(mode)
            _cabi.check(lib.og_sinkhorn_fwd(ptr(S), lds, n * lds, ptr(dust), B, n, m, T, 1.0, ptr(out), ptr(ws), wsb, stream()),
                        'og_sinkhorn_fwd')

        plans = {}
        for mode in (1, 0):
            lib.og_set_sinkhorn_resident(mode)
            plans[mode] = plan(lib, B, n, m)
            run(mode, outs[mode])
        again = torch.empty_like(outs[1])
        run(1, again)
        torch.cuda.synchronize()
        times = {1: [], 0: []}
        for _ in range(rounds):
            for mode in (1, 0):
                lib.og_set_sinkhorn_resident(mode)
                times[mode].append(events_ms(lambda: run(mode, outs[mode]), launches))
        lib.og_set_sinkhorn_resident(1)
        r = {'shape': label, 'pairs': B, 'n': n, 'm': m, 'iters': T,
             'ms_resident': statistics.median(times[1]), 'ms_streaming': statistics.median(times[0]),
             'ms_resident_rounds': times[1], 'ms_streaming_rounds': times[0],
             'max_abs_diff': float((outs[1] - outs[0]).abs().max()), 'resident_bit_identical': bool(torch.equal(outs[1], again)),
             'sha256_resident': hashlib.sha256(outs[1].cpu().numpy().tobytes()).hexdigest(),
             'sha256_streaming': hashlib.sha256(outs[0].cpu().numpy().tobytes()).hexdigest(),
             'plan_resident': plans[1], 'plan_streaming': plans[0]}
        r['hbm_gbs_streaming'] = (T + 1) * 4 * (n + 1) * (m + 1) * B / (r['ms_streaming'] * 1e-3) / 1e9
        if not quiet:
            print(f"{label:12s} B={B:3d} {n}x{m} T={T:3d}: resident {r['ms_resident']:.3f} ms, streaming {r['ms_streaming']:.3f} ms "
                  f"({r['ms_streaming'] / r['ms_resident']:.2f}x), max|d| {r['max_abs_diff']:.2e}, "
                  f"deterministic {r['resident_bit_identical']}, plan {plans[1]}")
        results.append(r)
        del S, ws, outs, again
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--against', help='another build of the library, timed in a second process')
    ap.add_argument('--json', action='store_true', help='print the measurements of this build as one JSON list')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    if args.json:
        print(json.dumps(measure(args.launches, args.rounds, quiet=True)))
        return
    gpu = card()
    print(json.dumps({'card': gpu}))
    results = measure(args.launches, args.rounds)
    against = None
    if args.against:
        env = dict(os.environ, OG_LIB=os.path.abspath(args.against))
        res = subprocess.run([sys.executable, os.path.abspath(__file__), '--json', '--launches', str(args.launches),
                              '--rounds', str(args.rounds)], env=env, capture_output=True, text=True, check=True)
        against = json.loads(res.stdout.strip().splitlines()[-1])
        print(f'against {args.against}:')
        for r, o in zip(results, against):
            print(f"{r['shape']:12s} resident {r['ms_resident']:.3f} ms against {o['ms_resident']:.3f} ms "
                  f"({o['ms_resident'] / r['ms_resident']:.3f}x), streaming {r['ms_streaming']:.3f} against {o['ms_streaming']:.3f} ms, "
                  f"streaming outputs bit-identical {r['sha256_streaming'] == o['sha256_streaming']}, "
                  f"resident outputs bit-identical {r['sha256_resident'] == o['sha256_resident']}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'sinkhorn_timing.json'), 'w') as f:
            json.dump({'card': gpu, 'launches': args.launches, 'rounds': args.rounds, 'results': results,
                       'against': args.against, 'against_results': against}, f, indent=1)


if __name__ == '__main__':
    main()
