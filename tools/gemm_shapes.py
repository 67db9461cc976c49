"""Times every GEMM shape of one C3 step (16 pairs, 2048 keypoints per image, d = 256) through the C ABI: CUDA events over 50
launches of one shape after a warm-up, on cuda:0.  Prints one JSON line per shape: time, algorithmic TFLOP/s, the MMA share (three
MMAs per product against the data-sheet dense rate of an H100 SXM: 989 TFLOP/s fp16, 495 TFLOP/s tf32), bytes (fp32 A, the outputs
and the residual, the B hi / lo operands) and GB/s.

    python tools/gemm_shapes.py [--against OTHER_LIB]

--against runs the same shapes in a second process on another build of the library (OG_LIB, such as a parent commit's) and prints
both builds side by side.  Not imported by bench.py."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

from gpu_timing import card, events_ms

PEAK = {'f16': 989e12, 'tf32': 495e12}
N, PAIRS, D = 2048, 16, 256
SEQ = 2 * PAIRS                                          # sequences of a self layer (both images)


# name, form, rows, k1, k2, nout, output kind, batch (V^T and the score GEMM: per sequence / pair)
SHAPES = [
    ('self Y (Q|K|V size)', 'f16', SEQ * N, D, 0, 3 * D, 'y', 1),
    ('self K', 'f16', SEQ * N, D, 0, D, 'k', 1),
    ('self Vt', 'f16', N, D, 0, D, 'vt', SEQ),
    ('self fc1', 'f16', SEQ * N, D, D, 2 * D, 'relu', 1),
    ('self fc2', 'f16', SEQ * N, 2 * D, 0, D, 'resid', 1),
    ('cross Q', 'f16', PAIRS * N, D, 0, D, 'y', 1),
    ('cross Y (K|V size)', 'f16', PAIRS * N, D, 0, 2 * D, 'y', 1),
    ('cross fc1', 'f16', PAIRS * N, D, D, 2 * D, 'relu', 1),
    ('cross fc2', 'f16', PAIRS * N, 2 * D, 0, D, 'resid', 1),
    ('final projection', 'tf32', PAIRS * N, D, 0, D, 'y', 1),
    ('score', 'tf32', N, D, 0, N, 'score', PAIRS),
]


def measure(iters=50):
    import torch
    from openglue_b200 import _cabi
    from openglue_b200._cabi import ptr as _p, stream as _st
    dev = 'cuda:0'
    lib = _cabi.lib()
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for name, form, rows, k1, k2, nout, kind, batch in SHAPES:
        K = k1 + k2
        A = torch.randn(batch, rows, k1, generator=g, device=dev)
        A2 = torch.randn(batch, rows, k2, generator=g, device=dev) if k2 else None
        wb = batch if kind == 'score' else 1
        W = torch.randn(wb * nout, K, generator=g, device=dev) / 16
        bias = torch.randn(nout, generator=g, device=dev)
        a = _cabi.OgLinearArgs()
        a.A, a.lda, a.strideA, a.k1, a.k2, a.ldw = A.data_ptr(), k1, rows * k1, k1, k2, K
        if k2:
            a.A2, a.lda2, a.strideA2 = A2.data_ptr(), k2, rows * k2
        a.strideW = nout * K if kind == 'score' else 0
        a.bias = bias.data_ptr() if kind != 'score' else None
        a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, 1.0, int(kind == 'relu')
        nbytes = A.numel() * 4 + (A2.numel() * 4 if k2 else 0)
        keep = []
        if form == 'tf32':
            Whi, Wlo = torch.empty_like(W), torch.empty_like(W)
            _cabi.check(lib.og_split_tf32(_p(W), _p(Whi), _p(Wlo), W.numel(), _st()), 'split_tf32')
            Y = torch.empty(batch, rows, nout, device=dev)
            a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
            nbytes += Y.numel() * 4 + W.numel() * 8
            call = lambda: lib.og_linear_tc_fwd(C.byref(a), _p(Whi), _p(Wlo), None, None, None, None, 0, _st())
        else:
            Wh, Wl = torch.empty(W.shape, dtype=torch.float16, device=dev), torch.empty(W.shape, dtype=torch.float16, device=dev)
            meta, amax, scale = torch.zeros(4, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev)
            _cabi.check(lib.og_weight_split_f16(_p(W), _p(bias), W.shape[0], K, _p(Wh), _p(Wl), _p(meta), _st()), 'split16')
            _cabi.check(lib.og_amax(_p(A), A.numel(), _p(amax), _st()), 'amax')
            nbytes += W.numel() * 4
            outs = [None] * 4
            amax_out = None
            if kind in ('y', 'relu', 'resid'):
                Y = torch.randn(batch, rows, nout, generator=g, device=dev)
                a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
                nbytes += Y.numel() * 4
                if kind == 'resid':                      # fc2: the residual is Y itself
                    a.R, a.ldr, a.strideR = Y.data_ptr(), nout, rows * nout
                    nbytes += Y.numel() * 4
                amax_out = torch.zeros(1, device=dev)
                keep.append(Y)
            elif kind == 'k':
                Yh, Yl = (torch.empty(batch, rows, nout, dtype=torch.float16, device=dev) for _ in range(2))
                a.ldy, a.strideY = nout, rows * nout
                outs[:2] = [_p(Yh), _p(Yl)]
                nbytes += Yh.numel() * 4
                keep += [Yh, Yl]
            else:                                        # V^T: [sequence, nout, ldyt]
                Yth, Ytl = (torch.empty(batch, nout, rows, dtype=torch.float16, device=dev) for _ in range(2))
                a.ldyt, a.strideYt = rows, nout * rows
                outs[2:] = [_p(Yth), _p(Ytl)]
                nbytes += Yth.numel() * 4
                keep += [Yth, Ytl]
            call = lambda: lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(amax), _p(amax_out), _p(scale), *outs, 0, _st())
        for _ in range(5):
            _cabi.check(call(), name)
        ms = events_ms(call, iters)
        flop = 2.0 * batch * rows * K * nout
        out.append({'shape': name, 'rows': batch * rows, 'K': K, 'nout': nout, 'form': form, 'ms': round(ms, 4),
                    'tflops': round(flop / ms / 1e9, 1), 'mma_share': round(3 * flop / (ms * 1e-3) / PEAK[form], 3),
                    'mbytes': round(nbytes / 1e6), 'gbps': round(nbytes / ms / 1e6)})
        del keep
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--against', help='another build of the library, timed in a second process')
    ap.add_argument('--json', action='store_true', help='print the measurements of this build as one JSON list')
    args = ap.parse_args()
    if args.json:
        print(json.dumps(measure()))
        return
    print(json.dumps({'card': card()}))
    runs = {'this': measure()}
    if args.against:
        env = dict(os.environ, OG_LIB=os.path.abspath(args.against))
        res = subprocess.run([sys.executable, os.path.abspath(__file__), '--json'], env=env, capture_output=True, text=True, check=True)
        runs['against'] = json.loads(res.stdout.strip().splitlines()[-1])
    for i, row in enumerate(runs['this']):
        line = {'this': row}
        if 'against' in runs:
            line['against'] = {k: runs['against'][i][k] for k in ('ms', 'tflops', 'mma_share', 'gbps')}
        print(json.dumps(line))


if __name__ == '__main__':
    main()
