"""Times K13 (csrc/prod.cuh): products, running products and all / any along an axis, at n = 10^6 and 10^7 elements for
L = 1..4 (2^64-189, 2^128-173, 2^192-237, 2^256-189), on device-resident operands; best-of CUDA-event time of the C-ABI
call after warm-up.  Shapes cover both forms and both sides of the split decision: 'full' (1, n, 1) is the rows form split
into slices, 'cols' (1, n/1000, 1000) the columns form split, 'wide' (1, 100, n/100) the columns form with many columns,
'rows8' (n/8, 8, 1) the rows form with one short reduction per warp.

  * prod against an IMAD bound: one product of N = 2L 32-bit limbs issues 2N^2 + N + 2 IMAD slots (schoolbook IMAD.WIDE
    counted twice, the pseudo-Mersenne fold; the generic Barrett product costs more), an SM retires 64 per clock at the
    max SM clock nvidia-smi reports; n products per call.
  * cumprod and all / any against HBM bytes: 2 n E (read and write) and n E (read) for E = 8L bytes per element, over
    the rate of a 2 GiB device copy measured in the same run.

Each result is checked against Python ints on a sample.  Then the reference's settled path at 10^6 elements on one host
core: the limbs turned into Python ints (codec.limbs_to_ints) and the reference's np.prod / np.cumprod / np.all of a
(10^5, 10) field array along axis 1 (needs the reference, see oracle/reference.py; reported as not measured without it).
Prints the card's name, power limit and max SM clock, then one JSON line per measurement.

    python tools/time_prod.py [--reps 5]
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
from mpyc_b200 import codec                        # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray, _stream_ptr   # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {1: 2**64 - 189, 2: 2**128 - 173, 3: 2**192 - 237, 4: 2**256 - 189}


def report(**rec):
    print(json.dumps(rec), flush=True)


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


def imad_bound(L, clock_mhz, sms):
    N = 2 * L
    return sms * 64 * clock_mhz * 1e6 / (2 * N * N + N + 2)


def shapes(n):
    return [('full', 1, n, 1), ('cols', 1, n // 1000, 1000), ('wide', 1, 100, n // 100), ('rows8', n // 8, 8, 1)]


def ints_at(a, idx):
    t = a.t[torch.as_tensor(idx, device=a.t.device)].cpu().numpy().view(np.uint64).reshape(len(idx), -1)
    return [int(v) for v in codec.limbs_to_ints(t, a.ctx)]


def check_sample(ctx, x, O, R, I, prod_out, cum_out, all_out):
    """a few outputs of each call against Python ints"""
    p = ctx.modulus
    for c in (0, O * I - 1):
        o, i = divmod(c, I)
        col = ints_at(x, [(o * R + r) * I + i for r in range(R)]) if R <= 10**6 else None
        if col is None:
            continue
        acc, run = 1, []
        for v in col:
            acc = acc * v % p
            run.append(acc)
        assert ints_at(prod_out, [c]) == [acc]
        assert ints_at(cum_out, [(o * R + R - 1) * I + i]) == [run[-1]]
        assert ints_at(all_out, [c]) == [int(all(col))]


def kernels(reps, copy):
    props = torch.cuda.get_device_properties(0)
    name = card()
    clock = int(name.split(',')[-1].strip().split()[0]) if name != 'unknown' else None
    stream = _stream_ptr()
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        E = 8 * L
        for n in (10**6, 10**7):
            x = DeviceArray.random(ctx, n, 3)
            out = DeviceArray.empty(ctx, n)
            red = DeviceArray.empty(ctx, n // 8)
            flags = DeviceArray.empty(ctx, n // 8)
            for label, O, R, I in shapes(n):
                t_prod = timed(lambda: check(lib.mpyc_b200_ff_prod_axis(ctx.handle, x.ptr, O, R, I, None, red.ptr, stream)), reps)
                t_cum = timed(lambda: check(lib.mpyc_b200_ff_cumprod_axis(ctx.handle, x.ptr, O, R, I, 0, out.ptr, stream)), reps)
                t_all = timed(lambda: check(lib.mpyc_b200_ff_all_any_axis(ctx.handle, x.ptr, O, R, I, 0, flags.ptr, stream)), reps)
                check_sample(ctx, x, O, R, I, red, out, flags)
                t_any = timed(lambda: check(lib.mpyc_b200_ff_all_any_axis(ctx.handle, x.ptr, O, R, I, 1, flags.ptr, stream)), reps)
                rec = {'L': L, 'n': n, 'shape': label, 'O': O, 'R': R, 'I': I,
                       'prod_ms': round(t_prod * 1e3, 4), 'prod_products_per_s': n / t_prod,
                       'cumprod_ms': round(t_cum * 1e3, 4), 'cumprod_of_copy': round(2 * n * E / t_cum / copy, 3),
                       'all_ms': round(t_all * 1e3, 4), 'all_of_copy': round(n * E / t_all / copy, 3),
                       'any_ms': round(t_any * 1e3, 4), 'any_of_copy': round(n * E / t_any / copy, 3)}
                if clock:
                    bound = imad_bound(L, clock, props.multi_processor_count)
                    rec.update(imad_bound_products_per_s=bound, prod_of_imad_bound=round(n / t_prod / bound, 3))
                report(**rec)
            del x, out, red, flags


def reference_settled(n=10**6):
    from oracle import reference
    ref = reference.path()
    if ref is None:
        report(what='reference settled path', note='no reference: not measured')
        return
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc import finfields
    sys.argv = argv
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        F = finfields.GF(p).array
        limbs = DeviceArray.random(ctx, n, 5).to_limbs()
        t0 = time.perf_counter()
        vals = codec.limbs_to_ints(limbs, ctx)
        t_settle = time.perf_counter() - t0
        x = F(np.asarray(vals, dtype=object).reshape(n // 10, 10), check=False)
        rec = {'what': 'reference settled path', 'L': L, 'n': n, 'shape': [n // 10, 10], 'axis': 1,
               'settle_s': round(t_settle, 4)}
        for name, fn in (('prod', np.prod), ('cumprod', np.cumprod), ('all', np.all)):
            t0 = time.perf_counter()
            fn(x, axis=1)
            rec[f'{name}_s'] = round(time.perf_counter() - t0, 4)
        report(**rec)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    print('card', card(), flush=True)
    copy = copy_rate(a.reps)
    report(what='device copy 2 GiB', GBps=round(copy / 1e9, 1))
    kernels(a.reps, copy)
    reference_settled()


if __name__ == '__main__':
    main()
