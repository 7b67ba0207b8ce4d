"""Times K12 (per-element exponents): k_powexp_fixed (one public base, comb tables in shared memory) and k_powexp_elem
(one base per element, 2-bit windows) at n = 10^6 and 10^7, for L = 1..4 (2^64-189, 2^128-173, 2^192-237, 2^256-189) and
exponent widths 64, 128 and 256 bits; best-of CUDA-event time of the C-ABI call after warm-up, on exponents already in
device memory (the fixed-base call includes building and uploading its tables).  Products per second count the products
the algorithm needs -- ceil(B / w) - 1 for the comb (w as the library picks it), 3 ceil(B / 2) + 2 for the windows, plus
the domain conversions -- against an IMAD
bound: one product of N = 2L 32-bit limbs takes N^2 IMAD.WIDE for the schoolbook product and N + 2 for the
pseudo-Mersenne fold, and an SM retires 64 32-bit IMADs per clock (two issue slots per IMAD.WIDE), at the max SM clock
nvidia-smi reports.  Each form is checked against Python's pow on a sample.  Then the reference's powmod_exp_list fallback
(a Python pow per element, mpyc/gmpy.py:288-290) at 10^5 exponents of bits(p) bits on one host core, and --caller: one
`2 ** x` of n = 10^5 SecInt(32) (1 party) with the K12 hook and without it.  Prints the card's name, power limit and max
SM clock, then one JSON line per measurement.

    python tools/time_powexp.py [--reps 5] [--caller]
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

PRIMES = {1: 2**64 - 189, 2: 2**128 - 173, 3: 2**192 - 237, 4: 2**256 - 189}
SMEM_MAX = 96 * 1024            # MPYC_PE_SMEM_MAX (csrc/launch.h)


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


def window(bits, L, ntab=1):
    """the comb window api.cu's powexp_window picks"""
    for w in range(8, 0, -1):
        nw = -(-bits // w)
        if ntab * (nw << w) * L * 8 <= SMEM_MAX:
            return w, nw
    raise AssertionError


def imad_bound(L, clock_mhz, sms):
    N = 2 * L
    per_product = 2 * N * N + N + 2            # IMAD issue slots: IMAD.WIDE counts twice
    return sms * 64 * clock_mhz * 1e6 / per_product


def sample_check(ctx, out, base, vals, p, k=200):
    idx = np.random.default_rng(1).integers(0, len(vals), size=k)
    t = out.t[torch.from_numpy(idx).to(out.t.device)].cpu().numpy().view(np.uint64).reshape(k, -1)
    got = codec.limbs_to_ints(t, ctx)
    if isinstance(base, int):
        want = [pow(base, int(vals[i]), p) for i in idx]
    else:
        b = base.t[torch.from_numpy(idx).to(base.t.device)].cpu().numpy().view(np.uint64).reshape(k, -1)
        want = [pow(int(x), int(vals[i]), p) for x, i in zip(codec.limbs_to_ints(b, ctx), idx)]
    assert [int(v) for v in got] == want


def abi(ctx, base, e, el, bits, out):
    """the C-ABI call alone, on exponents already in device memory"""
    import ctypes
    from mpyc_b200._cabi import lib, check
    null = ctypes.c_void_p(0)
    d_base, h_base = (base.ptr, null) if isinstance(base, DeviceArray) else (null, ctx.scalar_limbs(base))
    check(lib.mpyc_b200_ff_pow_exp(ctx.handle, d_base, h_base, ctypes.c_void_p(e.data_ptr()), el, bits, null, out.n, out.ptr,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


def kernels(reps):
    props = torch.cuda.get_device_properties(0)
    name = card()
    clock = int(name.split(',')[-1].strip().split()[0]) if name != 'unknown' else None
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        for n in (10**6, 10**7):
            x = DeviceArray.random(ctx, n, 3)
            out = DeviceArray.empty(ctx, n)
            g = np.random.default_rng(n + L)
            for bits in (64, 128, 256):
                el = -(-bits // 64)
                limbs = g.integers(0, 2**64 - 1, size=(n, el), dtype=np.uint64, endpoint=True)
                limbs[:, -1] |= np.uint64(1) << np.uint64((bits - 1) % 64)          # every exponent exactly `bits` wide
                e = torch.from_numpy(limbs.view(np.int64)).cuda()
                base = 3
                t_fix = timed(lambda: abi(ctx, base, e, el, bits, out), reps)
                t_elem = timed(lambda: abi(ctx, x, e, el, bits, out), reps)
                vals = [sum(int(w) << (64 * i) for i, w in enumerate(row)) for row in limbs[:200]]
                sample_check(ctx, dev.pow_exp(ctx, base, limbs[:200], None, bits), base, vals, p)
                x200 = DeviceArray(ctx, x.t[:200])
                sample_check(ctx, dev.pow_exp(ctx, x200, limbs[:200], None, bits), x200, vals, p)
                w, nw = window(bits, L)
                prod_fix = n * nw                                 # nw - 1 table products + the conversion out of the domain
                prod_elem = n * (3 * (-(-bits // 2)) + 4)         # the windows, x^2 and x^3, the two conversions
                rec = {'L': L, 'n': n, 'bits': bits, 'fixed_s': t_fix, 'elem_s': t_elem, 'window': w,
                       'fixed_products_per_s': prod_fix / t_fix, 'elem_products_per_s': prod_elem / t_elem}
                if clock:
                    bound = imad_bound(L, clock, props.multi_processor_count)
                    rec.update(imad_bound_products_per_s=bound, fixed_of_bound=prod_fix / t_fix / bound,
                               elem_of_bound=prod_elem / t_elem / bound)
                report(**rec)
                del e


def reference_fallback():
    """gmpy.powmod_exp_list without gmpy2: `list(pow(base, y, mod) for y in exp_lst)`, timed here on one core."""
    for L, p in PRIMES.items():
        g = np.random.default_rng(L)
        ex = [int.from_bytes(g.bytes(32), 'little') % p for _ in range(10**5)]
        t0 = time.perf_counter()
        r = list(pow(2, y, p) for y in ex)
        t = time.perf_counter() - t0
        ctx = mpyc_b200.context_for(p)
        dev.pow_exp(ctx, 2, *codec.exponents_to_limbs(ex))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        got = dev.pow_exp(ctx, 2, *codec.exponents_to_limbs(ex)).to_ints()
        t_dev = time.perf_counter() - t1
        assert [int(v) for v in got[:100]] == r[:100]
        report(what='powmod_exp_list', L=L, n=10**5, bits=p.bit_length(), reference_host_core_s=t,
               k12_with_packing_and_copies_s=t_dev)


def caller(n=10**5):
    from oracle import reference
    ref = reference.path()
    if ref is None:
        report(what='2 ** x', note='no reference: not measured')
        return
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc.runtime import mpc
    from mpyc import gmpy
    sys.argv = argv
    from mpyc_b200 import install
    install.install(resident=True, operators_min_size=1)
    hooked_fn = gmpy.powmod_exp_list
    secint = mpc.SecInt(32)
    mpc.run(mpc.start())
    x = mpc.input(secint.array(np.random.default_rng(2).integers(0, 31, size=n)))[0]
    mpc.run(mpc.gather(x))

    def one():
        t0 = time.perf_counter()
        out = mpc.run(mpc.output(2 ** x))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [int(v) for v in out]
    one()
    hooked, r1 = min((one() for _ in range(3)), key=lambda r: r[0])
    gmpy.powmod_exp_list = install._saved_gmpy['powmod_exp_list']         # the reference's fallback
    try:
        settled, r2 = one()
    finally:
        gmpy.powmod_exp_list = hooked_fn
    assert r1 == r2
    report(what='2 ** x', n=n, secint_bits=32, parties=1, hooked_s=round(hooked, 3), reference_powmod_exp_list_s=round(settled, 3))
    mpc.run(mpc.shutdown())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--caller', action='store_true', help='also the 2 ** x measurement')
    a = ap.parse_args()
    print('card', card(), flush=True)
    kernels(a.reps)
    reference_fallback()
    if a.caller:
        caller()


if __name__ == '__main__':
    main()
