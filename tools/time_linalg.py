"""Times K9 (csrc/linalg.cuh): det, solve (nrhs = 1) and inv of one n x n matrix at n in {64, 256, 1024, 2048} for L = 1, 2
and 4 (2^64-189, 2^128-173, 2^256-189), and batched det of (10^5, 4, 4) and (10^4, 16, 16) stacks.  Kernel time is the
best-of CUDA-event time of the whole C-ABI call after warm-up (solve and inv synchronise once, at the end, to read the
singular flag).  Modular multiplications are counted from the algorithm:
  det    sum_k 2 (n-1-k)^2                  (rows below the pivot, columns right of it)
  solve  sum_k 2 (n-1) (n-1-k + nrhs)       (Gauss-Jordan: every other row)
  plus the pivot products, one Fermat inversion (~1.5 bits(p) products) and the row scaling.
For contrast, the reference's own gauss_det / gauss_inv from oracle/_ref (pure Python, CPU) at n = 64 and 128, when that
copy exists.  --caller also times one mpc.np_det of a 256 x 256 secint matrix under install(resident=True), 1 party: with
the K9 hooks (the determinant of the opened L @ (U @ A) on the device) and without them (the reference's gauss_det on the
settled array); both calls must return the same determinant.  Prints the card's name and power limit, then one JSON line
per measurement.

    python tools/time_linalg.py [--reps 3] [--quick] [--caller]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev                # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {1: 2**64 - 189, 2: 2**128 - 173, 4: 2**256 - 189}


def timed(fn, reps):
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


def muls(op, n, nrhs, bits):
    if op == 'det':
        return sum(2 * (n - 1 - k) ** 2 for k in range(n)) + 2 * n + 1.5 * bits
    return sum(2 * (n - 1) * (n - 1 - k + nrhs) for k in range(n)) + 3 * n + 1.5 * bits + 2 * n * nrhs


def report(**rec):
    print(json.dumps(rec), flush=True)


def reference_times(ns):
    ref = os.path.join(ROOT, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'mpyc')):
        report(what='reference', note='oracle/_ref not present: not measured')
        return
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc import finfields
    sys.argv = argv
    F = finfields.GF(2**127 - 1).array
    rng = np.random.default_rng(1)
    for n in ns:
        A = F(np.array([int(v) for v in rng.integers(0, 2**62, size=n * n)], dtype=object).reshape(n, n))
        for op, fn in (('det', np.linalg.det), ('inv', np.linalg.inv)):
            t0 = time.perf_counter()
            fn(A)
            report(what='reference', op=op, n=n, p='2^127-1', s=round(time.perf_counter() - t0, 4), device='cpu')


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--quick', action='store_true', help='n <= 256 only')
    ap.add_argument('--caller', action='store_true', help='only the mpc.np_det measurement')
    a = ap.parse_args()
    print(f'card: {card()}', flush=True)
    if a.caller:
        caller()
        return
    sizes = (64, 256) if a.quick else (64, 256, 1024, 2048)
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        for n in sizes:
            A = DeviceArray.random(ctx, n * n, seed=n)
            B = DeviceArray.random(ctx, n, seed=n + 1)
            reps = a.reps if n < 2048 else 1
            for op, fn, nrhs in (('det', lambda: dev.det(A, 1, n), 0), ('solve', lambda: dev.solve(A, B, n, 1), 1),
                                 ('inv', lambda: dev.inv(A, n), n)):
                s = timed(fn, reps)
                m = muls(op if op == 'det' else 'solve', n, nrhs, p.bit_length())
                report(what=op, L=L, n=n, ms=round(s * 1e3, 3), Gmul_per_s=round(m / s / 1e9, 2))
        for batch, n in ((10**5, 4), (10**4, 16)):
            A = DeviceArray.random(ctx, batch * n * n, seed=batch)
            s = timed(lambda: dev.det(A, batch, n), a.reps)
            m = batch * muls('det', n, 0, 0) + 3 * batch   # + Montgomery-trick inversion per matrix
            report(what='det_batch', L=L, batch=batch, n=n, ms=round(s * 1e3, 3), Gmul_per_s=round(m / s / 1e9, 2))
    reference_times((64, 128))


def caller(n=256):
    sys.path.insert(0, ROOT)
    from oracle import reference
    ref = reference.path()
    if ref is None:
        report(what='np_det', note='no reference: not measured')
        return
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc.runtime import mpc
    sys.argv = argv
    from mpyc_b200 import install, resident
    install.install(resident=True, operators_min_size=1)
    secint = mpc.SecInt(64)
    mpc.run(mpc.start())
    rng = np.random.default_rng(2)
    A = mpc.input(secint.array(rng.integers(-100, 100, size=(n, n)).astype(object)))[0]
    mpc.run(mpc.gather(A))

    def one():
        t0 = time.perf_counter()
        d = mpc.run(mpc.output(mpc.np_det(A)))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, int(d)
    one()
    hooked, d1 = min((one() for _ in range(3)), key=lambda r: r[0])
    hooks, resident.LINALG_FUNCTIONS = resident.LINALG_FUNCTIONS, ()   # np.linalg.det back to the reference's gauss_det
    try:
        settled, d2 = one()
    finally:
        resident.LINALG_FUNCTIONS = hooks
    assert d1 == d2, (d1, d2)
    report(what='np_det', n=n, parties=1, hooked_ms=round(hooked * 1e3, 1), settled_ms=round(settled * 1e3, 1))
    mpc.run(mpc.shutdown())


if __name__ == '__main__':
    main()
