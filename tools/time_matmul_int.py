"""Times K14 (csrc/matmul_int.cuh): a field matrix times a public int64 matrix, against K1c on the same matrix converted to
limbs, on device-resident operands; best-of CUDA-event time of the C-ABI call after warm-up, the two kernels timed
alternately.  Shapes (r, k, c): (1, 3136, 1024) and (128, 3136, 1024) (np_cnnmnist's dense layer, one image and a batch),
(1024, 1024, 1024), (10^6, 100, 1) (a scoring pass, rows form) and W on the left (1024, 10^5, 1).  Primes 2^64 - 189,
2^128 - 173, 2^256 - 189 and a generic 64-bit prime.  Also the host time of the conversion K1c needs (int64 entries to
canonical limbs, vectorised NumPy), and one caller-level `x @ W` of a limb-backed field array through install's hook
against the reference's own __matmul__ on the settled object array (needs the reference; reported as not measured
without it).  Each K14 result is compared with K1c's.  Prints the card's name, power limit and max SM clock, then one JSON
line per measurement.

    python tools/time_matmul_int.py [--reps 5]
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
import ctypes                                      # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray, _stream_ptr   # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {'P64': 2**64 - 189, 'P128': 2**128 - 173, 'P256': 2**256 - 189, 'P64G': 9409569905028393239}
SHAPES = [(1, 3136, 1024, False), (128, 3136, 1024, False), (1024, 1024, 1024, False), (10**6, 100, 1, False),
          (1024, 10**5, 1, True)]


def report(**rec):
    print(json.dumps(rec), flush=True)


def to_limbs(w, p, L):
    """int64 entries -> canonical residues as (n, L) uint64 limbs: w for w >= 0, p - |w| otherwise (multi-limb borrow)."""
    w = w.reshape(-1)
    neg = w < 0
    mag = np.where(neg, (-(w + 1)).astype(np.uint64) + np.uint64(1), w.astype(np.uint64))
    out = np.zeros((w.size, L), dtype=np.uint64)
    out[:, 0] = np.where(neg, np.uint64(p & (2**64 - 1)) - mag, mag)
    borrow = neg & (mag > np.uint64(p & (2**64 - 1)))
    for i in range(1, L):
        pi = np.uint64((p >> (64 * i)) & (2**64 - 1))
        out[:, i] = np.where(neg, pi - borrow.astype(np.uint64), 0)
        borrow = neg & borrow & (pi == 0)
    return out


def event_time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def caller_level(reps):
    from oracle import reference
    path = reference.path()
    if path is None:
        report(what='caller x @ W', status='not measured (reference not present)')
        return
    sys.path.insert(0, path)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc import thresha, finfields
    sys.argv = argv
    from mpyc_b200 import install as inst, resident
    p = PRIMES['P128']
    F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
    r, k, c = 8, 3136, 128                # the settled object-array product takes seconds on one core
    W = np.random.default_rng(2).integers(-2**20, 2**20, size=(k, c), dtype=np.int64)
    X = DeviceArray.random(ctx, r * k, seed=3)
    plain = F(np.array(X.to_ints(), dtype=object).reshape(r, k))
    inst.install(thresha, resident=True, finfields_module=finfields, public_matmul=True)
    try:
        x = F(resident.LimbValue(ctx, X, (r, k)), check=False)
        x @ W
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(reps):
            t0 = time.perf_counter()
            y = x @ W
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
        got = y.value
    finally:
        inst.uninstall()
    t0 = time.perf_counter()
    ref = plain @ W
    settled = time.perf_counter() - t0
    report(what='caller x @ W', p='P128', shape=[r, k, c], hooked_s=best, settled_s=settled,
           equal=bool((np.asarray(got) == np.asarray(ref.value)).all()))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--shapes', type=int, default=len(SHAPES), help='first N shapes only (rehearsal)')
    args = ap.parse_args()
    report(card=card())
    rng = np.random.default_rng(1)
    for r, k, c, w_left in SHAPES[:args.shapes]:
        W = rng.integers(-2**63, 2**63 - 1, size=(r, k) if w_left else (k, c), dtype=np.int64, endpoint=True)
        for name, p in PRIMES.items():
            ctx = mpyc_b200.context_for(p)
            L = ctx.nlimbs
            t0 = time.perf_counter()
            limbs = to_limbs(W, p, L)
            conv = time.perf_counter() - t0
            X = DeviceArray.random(ctx, k * c if w_left else r * k, seed=r + k + c)
            Wl = DeviceArray.from_limbs(ctx, limbs)
            Wd = torch.from_numpy(W.reshape(-1)).cuda()
            a, b = DeviceArray.empty(ctx, r * c), DeviceArray.empty(ctx, r * c)
            wp = ctypes.c_void_p(Wd.data_ptr())
            k14 = lambda: check(lib.mpyc_b200_ff_matmul_int(ctx.handle, X.ptr, wp, 0, int(w_left), a.ptr, r, k, c,   # noqa: E731
                                                            _stream_ptr()))
            A, B = (Wl, X) if w_left else (X, Wl)
            k1c = lambda: check(lib.mpyc_b200_ff_matmul(ctx.handle, A.ptr, B.ptr, b.ptr, r, k, c, _stream_ptr()))   # noqa: E731
            k14()
            k1c()
            torch.cuda.synchronize()
            equal = torch.equal(a.t, b.t)
            t14, t1c = 1e9, 1e9
            for _ in range(args.reps):
                t14 = min(t14, event_time(k14))
                t1c = min(t1c, event_time(k1c))
            report(shape=[r, k, c], w_left=w_left, p=name, L=L, kind=ctx.kind, k14_s=t14, k1c_s=t1c,
                   speedup=t1c / t14, host_convert_s=conv, equal=equal)
            del X, Wl, Wd, A, B, a, b
            torch.cuda.empty_cache()
    caller_level(args.reps)


if __name__ == '__main__':
    main()
