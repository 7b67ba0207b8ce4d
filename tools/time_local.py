"""Time the protocol-local kernels (csrc/local.cuh) on one GPU: CUDA events on the launching stream, warm-up, inputs
larger than L2; achieved = algorithmic bytes / time against the measured copy peak.  One JSON line per kernel/config.

    python tools/time_local.py [--quick]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch   # noqa: E402

import mpyc_b200   # noqa: E402
from mpyc_b200 import device as dev   # noqa: E402
from mpyc_b200.device import DeviceArray   # noqa: E402

PEAK = 3350.0   # H100 SXM data sheet (HBM3), unless MEASURED_PEAKS.json gives a measured one
try:
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')) as fh:
        peaks = json.load(fh)
    PEAK = float(peaks.get('hbm_gbps', peaks.get('hbm_copy_gbps', PEAK)))
except Exception:   # noqa: BLE001
    pass


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def line(name, p, bytes_, ms, **extra):
    gbps = bytes_ / ms / 1e6
    print(json.dumps({'kernel': name, 'p_bits': p.bit_length(), 'ms': round(ms, 4), 'alg_bytes': bytes_, 'GBps': round(gbps, 1),
                      'frac_of_copy_peak': round(gbps / PEAK, 3), **extra}), flush=True)


def main():
    quick = '--quick' in sys.argv
    torch.cuda.set_device(0)
    primes = [2**64 - 189, 2**128 - 173, 2**256 - 189, 9409569905028393239, 2**69 - 93,
              0x8000000000000000000000000000000000000000000004c7]    # the last: a generic 192-bit prime (3 limbs)
    if '--only-compose' in sys.argv:      # short run for an ncu capture: k_bits_compose on the 128-bit field, f = 37 and 6
        p = 2**128 - 173
        ctx = mpyc_b200.context_for(p)
        A = DeviceArray.random(ctx, 1 << 26, seed=5, stream_id=1)
        for f in (37, 6):
            rows = A.n // f
            bits = DeviceArray(ctx, A.t[:rows * f])
            line('bits_compose', p, (f + 1) * 16 * rows, timed(lambda: dev.bits_compose(bits, rows, f), reps=3, warm=2), n=rows, f=f)
        return
    if '--ncu-all' in sys.argv:           # one pass over every K6 kernel on the 128-bit field (256 MiB operands) for ncu
        from mpyc_b200 import _cabi
        p = 2**128 - 173
        ctx = mpyc_b200.context_for(p)
        n = 1 << 24
        A, B, C = (DeviceArray.random(ctx, n, seed=5, stream_id=i) for i in (1, 2, 3))
        R, cols = 38, n // 38
        M, V = DeviceArray(ctx, A.t[:R * cols]), DeviceArray(ctx, C.t[:cols])
        for fn in (lambda: dev.fma(A, B, C), lambda: dev.fma(A, None, C), lambda: dev.axpb(A, (p + 1) >> 1, 5), lambda: dev.low_bits(A, 37),
                   lambda: dev.nonzero(A, want_mask=False), lambda: dev.bits_decompose(V, 37, descending=True),
                   lambda: dev.transpose(M, cols, R), lambda: dev.cumsum_rows(M, R, cols),
                   lambda: dev.binop_rows(M, V, _cabi.OP_SUB, R, cols, reflected=True)):
            fn()
            fn()
        torch.cuda.synchronize()
        return
    for p in primes:
        ctx = mpyc_b200.context_for(p)
        E = 8 * ctx.nlimbs
        n = (1 << 30) // E if not quick else (1 << 22)          # 1 GiB per operand
        A, B, C = (DeviceArray.random(ctx, n, seed=5, stream_id=i) for i in (1, 2, 3))
        line('fma a*b+c', p, 4 * E * n, timed(lambda: dev.fma(A, B, C)), n=n)
        line('fma a*a+c', p, 3 * E * n, timed(lambda: dev.fma(A, None, C)), n=n)
        line('axpb', p, 2 * E * n, timed(lambda: dev.axpb(A, (p + 1) >> 1, 12345)), n=n)
        line('low_bits', p, 2 * E * n, timed(lambda: dev.low_bits(A, 37)), n=n)
        line('nonzero(count)', p, E * n, timed(lambda: dev.nonzero(A, want_mask=False)), n=n)
        del B
        for f in (6, 16, 37, 64):
            rows = n // f
            bits = DeviceArray(ctx, A.t[:rows * f])
            for desc in (False, True):
                line('bits_compose', p, (f + 1) * E * rows, timed(lambda: dev.bits_compose(bits, rows, f, descending=desc)),
                     n=rows, f=f, descending=desc)
        for l in (6, 37):
            rows = n // l
            c = DeviceArray(ctx, C.t[:rows])
            line('bits_decompose', p, (l + 1) * E * rows, timed(lambda: dev.bits_decompose(c, l, descending=True)), n=rows, l=l)
        R = 38                                                  # np_sgn's matrices: (l + 1, n) with l = 37
        cols = n // R
        Mx = DeviceArray(ctx, A.t[:R * cols])
        Vx = DeviceArray(ctx, C.t[:cols])
        from mpyc_b200 import _cabi
        line('transpose', p, 2 * E * R * cols, timed(lambda: dev.transpose(Mx, cols, R)), rows=cols, cols=R)
        line('cumsum_rows', p, 2 * E * R * cols, timed(lambda: dev.cumsum_rows(Mx, R, cols)), rows=R, cols=cols)
        line('binop_rows', p, (2 * R + 1) * E * cols, timed(lambda: dev.binop_rows(Mx, Vx, _cabi.OP_SUB, R, cols, reflected=True)), rows=R, cols=cols)
        del A, C, Mx, Vx
        # np_cnnmnist's two convolution layers at batch 8 (demos/np_cnnmnist.py: 1->16 5x5 on 28x28, 16->16 5x5 on 14x14)
        for (k, r, m, nn, v, s) in ((8, 1, 28, 28, 16, 5), (8, 16, 14, 14, 16, 5)):
            X = DeviceArray.random(ctx, k * r * m * nn, seed=7, stream_id=1)
            W = DeviceArray.random(ctx, v * r * s * s, seed=7, stream_id=2)
            Bi = DeviceArray.random(ctx, v, seed=7, stream_id=3)
            ms = timed(lambda: dev.conv2d(X, W, Bi, k, r, m, nn, v, s))
            macs = k * v * m * nn * r * s * s
            print(json.dumps({'kernel': 'conv2d', 'p_bits': p.bit_length(), 'shape': [k, r, m, nn, v, s], 'ms': round(ms, 4),
                              'modular_macs_per_s': round(macs / ms * 1e3, 1)}), flush=True)
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
