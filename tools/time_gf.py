"""Times K15 (csrc/gf_local.cuh) on device-resident GF(2^8) bytes: k_gf_bits_compose of (n, 8) bit rows and
k_gf_matmul_batched of the S-box shape (8, 8) @ (n, 8, 1), n = 10^6 and 10^7 rows, the best of 5 windows of 50 back-to-back C-ABI
calls between CUDA events after warm-up, with the bytes each call reads and writes per second; K1's k_gf_matmul on the same product as one 2-D
(8, 8) @ (8, n) in the same run for contrast.  Prints the card's name, power limit and max SM clock, then one JSON line
per measurement.

    python tools/time_gf.py [--reps 5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev                # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from stream_probe import card                      # noqa: E402


def best(fn, reps, loops=50):
    """Best over reps of the mean time of `loops` back-to-back calls between one pair of CUDA events."""
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(loops):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3 / loops)
    return min(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    ctx = mpyc_b200.context_for(283, binary=True)
    rng = np.random.default_rng(0)
    A = DeviceArray.from_limbs(ctx, rng.integers(0, 256, size=64, dtype=np.uint8))
    for n in (10**6, 10**7):
        bits = DeviceArray.from_limbs(ctx, rng.integers(0, 2, size=8 * n, dtype=np.uint8))
        t = best(lambda: dev.gf_bits_compose(bits, n, 8), args.reps)
        print(json.dumps({'kernel': 'k_gf_bits_compose', 'n': n, 'l': 8, 'seconds': t, 'GB_per_s': 9 * n / t / 1e9}), flush=True)
        t = best(lambda: dev.gf_matmul_batched(A, False, bits, True, n, 8, 8, 1), args.reps)
        print(json.dumps({'kernel': 'k_gf_matmul_batched', 'shape': f'(8,8)@({n},8,1)', 'seconds': t,
                          'GB_per_s': 16 * n / t / 1e9}), flush=True)
        cols = DeviceArray(ctx, bits.t.view(n, 8).t().contiguous().view(-1))
        t = best(lambda: dev.matmul(ctx, A, cols, 8, 8, n), args.reps)
        print(json.dumps({'kernel': 'k_gf_matmul', 'shape': f'(8,8)@(8,{n})', 'seconds': t, 'GB_per_s': 16 * n / t / 1e9}),
              flush=True)


if __name__ == '__main__':
    main()
