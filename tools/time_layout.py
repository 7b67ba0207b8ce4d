"""Times K8 (csrc/layout.cuh): copies between strided views and broadcast arithmetic on device-resident operands, against a
2 GiB device copy measured in the same run, and against the kernels K8 could replace (k_transpose and k_binop_rows at
tools/time_local.py's np_sgn shape, timed alternately with K8 on the same operands).

Shapes at the byte size of 10^8 128-bit elements (n = 2*10^8 / L elements of L limbs): x[:, ::2] of (n/100, 100), x[::-1],
a 2-D transpose, swapaxes(1, 3) of a 4-D array, concatenate of two (n/100, 50) pieces on the last axis, x[..., I] with
every other index, and (n/100, 1) * (n/100, 100) against K1 on equal shapes.  Algorithmic bytes: what is read plus what
is written.  Prints the card's name and power limit, then one JSON line per shape: best-of CUDA-event time after warm-up,
GB/s and the fraction of the copy rate.

    python tools/time_layout.py [--reps 10] [--quick]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mpyc_b200                                   # noqa: E402
from mpyc_b200 import _cabi, device as dev, layout  # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {1: 2**64 - 189, 2: 2**128 - 173, 4: 2**256 - 189}


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best * 1e-3


def copy_rate(reps):
    n = 2**31 // 8
    a = torch.empty(n, dtype=torch.int64, device='cuda')
    b = torch.empty_like(a)
    return 2 * 2**31 / timed(lambda: b.copy_(a), reps)


def report(what, L, nbytes, secs, copy, **extra):
    rate = nbytes / secs
    print(json.dumps({'what': what, 'L': L, 'ms': round(secs * 1e3, 4), 'GBps': round(rate / 1e9, 1),
                      'frac_of_copy': round(rate / copy, 3), **extra}), flush=True)


def copy_fn(src, view, dst):
    s, d = layout.collapse(view, layout.View.full(view.shape))
    return lambda: dev.copy_view(src, s, dst, d)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--quick', action='store_true', help='a hundredth of the sizes (rehearsal)')
    a = ap.parse_args()
    print(f'card: {card()}', flush=True)
    copy = copy_rate(a.reps)
    print(json.dumps({'what': 'device copy 2 GiB', 'GBps': round(copy / 1e9, 1)}), flush=True)
    scale = 100 if a.quick else 1
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        E = 8 * L
        n = 2 * 10**8 // L // scale // 100 * 100
        x = DeviceArray.random(ctx, n, seed=1)
        out = DeviceArray.empty(ctx, n)
        R = n // 100
        view = layout.getitem_plan((R, 100), (slice(None), slice(None, None, 2)))[0]
        report('x[:, ::2] of (n/100, 100)', L, 2 * E * n // 2, timed(copy_fn(x, view, out), a.reps), copy)
        report('x[::-1]', L, 2 * E * n, timed(copy_fn(x, layout.flip_view((n,)), out), a.reps), copy)
        side = int(n ** 0.5)
        report('transpose (s, s)', L, 2 * E * side * side, timed(copy_fn(x, layout.permuted((side, side), (1, 0)), out), a.reps), copy,
               s=side)
        s4 = (R // 100, 10, 10, 100)
        report('swapaxes(1, 3) of (n/10^4, 10, 10, 100)', L, 2 * E * n,
               timed(copy_fn(x, layout.permuted(s4, layout.swapaxes_axes(4, 1, 3)), out), a.reps), copy)
        half = DeviceArray(ctx, x.t[:n // 2])
        other = DeviceArray(ctx, x.t[n // 2:])
        out_shape, items = layout.concatenate_plan([(R, 50), (R, 50)], -1)
        plans = [(src, layout.collapse(s, d)) for src, (_, s, d) in zip((half, other), items)]
        report('concatenate two (n/100, 50) on axis -1', L, 2 * E * n,
               timed(lambda: [dev.copy_view(src, s, out, d) for src, (s, d) in plans], a.reps), copy)
        view = layout.getitem_plan((R, 100), (Ellipsis, np.arange(0, 100, 2)))[0]
        report('x[..., I], I = every other index', L, 2 * E * n // 2, timed(copy_fn(x, view, out), a.reps), copy)
        col = DeviceArray(ctx, x.t[:R])
        shape, vc, vm = layout.broadcast_views((R, 1), (R, 100))
        cc, cm = layout.collapse(vc, vm)
        report('(n/100, 1) * (n/100, 100) k_binop_view', L, E * (2 * n + R), timed(lambda: dev.binop_view(col, cc, x, cm, _cabi.OP_MUL), a.reps),
               copy)
        report('(n/100, 100) * (n/100, 100) K1', L, 3 * E * n, timed(lambda: x._binop(out, _cabi.OP_MUL), a.reps), copy)
        del x, out, half, other, col
        # old vs new at tools/time_local.py's shape: (cols, 38) -> (38, cols) and v (cols,) - M (38, cols); alternated
        m = (1 << 30) // E // scale
        rows = 38
        cols = m // rows
        A = DeviceArray.random(ctx, rows * cols, seed=5, stream_id=1)
        V = DeviceArray.random(ctx, cols, seed=5, stream_id=3)
        T = DeviceArray.empty(ctx, rows * cols)
        new_t = copy_fn(A, layout.permuted((cols, rows), (1, 0)), T)
        shape, vv, vm = layout.broadcast_views((cols,), (rows, cols))
        cv, cm = layout.collapse(vv, vm)
        best = {'transpose k_transpose': 1e9, 'transpose K8': 1e9, 'binop_rows k_binop_rows': 1e9, 'binop_rows K8': 1e9}
        for _ in range(3):
            best['transpose k_transpose'] = min(best['transpose k_transpose'], timed(lambda: dev.transpose(A, cols, rows), a.reps))
            best['transpose K8'] = min(best['transpose K8'], timed(new_t, a.reps))
            best['binop_rows k_binop_rows'] = min(best['binop_rows k_binop_rows'],
                                                  timed(lambda: dev.binop_rows(A, V, _cabi.OP_SUB, rows, cols, reflected=True), a.reps))
            best['binop_rows K8'] = min(best['binop_rows K8'], timed(lambda: dev.binop_view(V, cv, A, cm, _cabi.OP_SUB), a.reps))
        for what, secs in best.items():
            nbytes = 2 * E * rows * cols if what.startswith('transpose') else (2 * rows + 1) * E * cols
            report(what + ' (time_local shape)', L, nbytes, secs, copy, rows=rows, cols=cols)
        del A, V, T


if __name__ == '__main__':
    main()
