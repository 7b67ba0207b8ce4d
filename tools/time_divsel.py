"""Times K11: `x / y` (ff_div, one Montgomery-trick pass) against ff_inv followed by a K1 product, and np.where (k_select)
of device arrays, at n = 10^6 and 10^7 for L = 2 and 4 (2^128-173, 2^256-189), best-of CUDA-event time of the C-ABI call
after warm-up.  Bandwidth counts the bytes the call must move: division 3 n elements (num, den, out) plus the prefix
products written and read back (2 n); select 2 n elements plus n mask bytes (one side read per element).  At n = 10^6
the settled reference path -- NumPy object arithmetic with Python-int inverses, what FiniteFieldArray.__truediv__ and
np.where ran before the hooks -- is timed once on the host for comparison.  Checks that both forms give the same values on
a sample.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/time_divsel.py [--reps 10]
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
from mpyc_b200 import codec, device as dev         # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {2: 2**128 - 173, 4: 2**256 - 189}


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


def host_ints(a: DeviceArray, idx):
    t = a.t[torch.from_numpy(idx).to(a.t.device)].cpu().numpy().view(np.uint64)
    return [int(v) for v in codec.limbs_to_ints(t, a.ctx)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    print('card', card(), flush=True)
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        E = 8 * L
        for n in (10**6, 10**7):
            x, y = DeviceArray.random(ctx, n, 1), DeviceArray.random(ctx, n, 2)
            mask = torch.randint(0, 2, (n,), dtype=torch.uint8, device='cuda')
            t_div = timed(lambda: dev.divide(x, y), args.reps)
            t_inv = timed(lambda: x * y.reciprocal(), args.reps)
            t_sel = timed(lambda: dev.select(mask, x, (1, 0), y, (1, 0)), args.reps)
            t_aff = timed(lambda: dev.select(mask, x, (p - 1, 1), y, (1, 0)), args.reps)
            q, s = dev.divide(x, y), dev.select(mask, x, (1, 0), y, (1, 0))
            assert q.count_mismatch(x * y.reciprocal()) == 0
            rec = {'L': L, 'n': n, 'div_s': t_div, 'inv_then_mul_s': t_inv, 'div_GBps': 5 * n * E / t_div / 1e9,
                   'select_s': t_sel, 'select_affine_s': t_aff, 'select_GBps': (2 * n * E + n) / t_sel / 1e9}
            if n == 10**6:                                     # the settled reference path, on the host
                idx = np.arange(n)
                xs, ys = host_ints(x, idx), host_ints(y, idx)
                m = mask.cpu().numpy().astype(bool)
                X, Y = np.array(xs, dtype=object), np.array(ys, dtype=object)
                t0 = time.perf_counter()
                ref_div = X * np.vectorize(lambda v: pow(v, -1, p), otypes='O')(Y) % p
                rec['reference_div_s'] = time.perf_counter() - t0
                t0 = time.perf_counter()
                ref_sel = np.where(m, X, Y)
                rec['reference_where_s'] = time.perf_counter() - t0
                sample = np.random.default_rng(0).integers(0, n, size=1000)
                assert host_ints(q, sample) == [int(v) for v in ref_div[sample]]
                assert host_ints(s, sample) == [int(v) for v in ref_sel[sample]]
            print(json.dumps(rec), flush=True)


if __name__ == '__main__':
    main()
