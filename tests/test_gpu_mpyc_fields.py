"""K7-K12, K1c and the Shamir step (K2 / K3) on the fields MPyC's default secure types create (tests/mpyc_fields.py): the
default fixed-point field 2^80 - 65, the 2-, 3- and 4-limb shifted pseudo-Mersenne primes of secint(64), secint(128) and
secint(168), the 3-limb aligned 2^192 - 237, a 48-bit generic one-limb field and two generic fields with 1024-th roots of
unity.  Every check is bit-exact against Python integers (or the tests/oracle_* restatements of the same function);
inputs hold 0, 1, p - 1 and blocks of p - 1, which drive lazy sums to their largest values.  Shapes sit on both sides of
each launcher's form decisions: K7's rows / columns forms and split slices, K9's shared-memory tile and step forms and a
forced row swap, K10's split decision, k_inv_batch's T x B layout and K12's two forms."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import _cabi, codec, layout, device as dev   # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray, DeviceMatrix, _stream_ptr   # noqa: E402
from mpyc_fields import BY_NAME, FIELDS, field_id   # noqa: E402
import oracle_linalg                               # noqa: E402
from oracle import shamir_oracle as orc            # noqa: E402
from oracle_layout import positions                # noqa: E402

SMS = torch.cuda.get_device_properties(0).multi_processor_count


def ctx_of(f):
    ctx = mpyc_b200.context_for(f.p)
    assert (ctx.nlimbs, ctx.kind, ctx.bits) == (f.limbs, f.kind, f.bits)
    return ctx


def ints(a):
    return [int(v) for v in a.to_ints()]


def values(p, n, seed):
    """n residues: 0, 1, p - 1, p - 2 first, then random residues with every other run of 37 set to p - 1"""
    rnd = random.Random(seed)
    out = [rnd.randrange(p) if (i // 37) % 2 else p - 1 for i in range(n)]
    out[:4] = [0, 1, p - 1, p - 2][:n]
    return out


def const(ctx, n, v):
    """n copies of the residue v, made on the device (axpb of zeros)"""
    z = DeviceArray(ctx, torch.zeros((n, ctx.nlimbs), dtype=torch.int64, device='cuda'))
    return dev.axpb(z, 0, v)


def offset_copy(a):
    """a's elements in a buffer that starts one element into its allocation"""
    buf = DeviceArray.empty(a.ctx, a.n + 1)
    buf.t[1:].copy_(a.t)
    return DeviceArray(a.ctx, buf.t[1:])


# ---- K7: sums and running sums along an axis --------------------------------------------------------------------------

# 3-D shapes reduced along each axis: inner sizes 31 / 32 / 33 (rows form below 32, columns form from 32), and long axes
# with a small O * I, which axis_plan splits into slices whose last one is partial
SUM_SHAPES = [(3, 10, 31), (3, 10, 32), (3, 10, 33), (10, 1, 31), (10, 1, 32), (10, 1, 33)]
SPLIT_SHAPES = [(1, 3000, 31), (1, 3000, 32), (1, 3000, 33), (2, 1, 5001)]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_sum_and_cumsum_along_every_axis(f):
    ctx, p = ctx_of(f), f.p
    for j, shape in enumerate(SUM_SHAPES + SPLIT_SHAPES):
        n = int(np.prod(shape))
        vals = values(p, n, 100 * j + f.bits)
        x = np.array(vals, dtype=object).reshape(shape)
        a = DeviceArray.from_ints(ctx, vals)
        for axis in (0, 1, 2):
            for src in (a, offset_copy(a)):
                got, gshape = dev.sum_axis(src, shape, axis, initial=p - 2)
                want = (x.sum(axis=axis) + p - 2) % p
                assert gshape == want.shape and ints(got) == want.reshape(-1).tolist(), (shape, axis)
            for inc in (False, True):
                got, gshape = dev.cumsum_axis(offset_copy(a) if inc else a, shape, axis, include_initial=inc)
                want = np.cumulative_sum(x, axis=axis, include_initial=inc) % p
                assert gshape == want.shape and ints(got) == want.reshape(-1).tolist(), (shape, axis, inc)


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_sums_of_all_p_minus_1(f):
    """every lazy sum at its bound: the sum of R copies of p - 1 is -R mod p, the running sums -1, -2, ..."""
    ctx, p = ctx_of(f), f.p
    for O, R, I in ((1, 10**6 + 3, 1), (4, 100_003, 33), (2, 50_001, 32), (3, 4001, 31), (2, 3001, 5)):
        top = const(ctx, O * R * I, p - 1)
        out = DeviceArray.empty(ctx, O * I)
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, top.ptr, O, R, I, None, out.ptr, _stream_ptr()))
        assert set(ints(out)) == {(-R) % p}, (O, R, I)
        if O * R * I <= 400_000:
            cs = DeviceArray.empty(ctx, O * (R + 1) * I)
            check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, top.ptr, O, R, I, 1, cs.ptr, _stream_ptr()))
            want = np.broadcast_to(np.array([(-r) % p for r in range(R + 1)], dtype=object)[None, :, None], (O, R + 1, I))
            assert ints(cs) == want.reshape(-1).tolist(), (O, R, I)


# ---- K8: broadcast arithmetic, permutations and flips -----------------------------------------------------------------

BROADCASTS = [((64, 1), (64, 37)), ((40, 33), (33,)), ((33,), (40, 33)), ((5, 1, 1), (3, 5, 7, 9)), ((3, 5, 7, 9), (5, 1, 1))]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_broadcast_arithmetic(f):
    """column, row, 4-D and reflected broadcasts of + - * against object arithmetic"""
    ctx, p = ctx_of(f), f.p
    for j, (sa, sb) in enumerate(BROADCASTS):
        xa, xb = values(p, int(np.prod(sa)), j), values(p, int(np.prod(sb)), j + 50)[::-1]
        A, B = DeviceArray.from_ints(ctx, xa), DeviceArray.from_ints(ctx, xb)
        shape, va, vb = layout.broadcast_views(sa, sb)
        ca, cb = layout.collapse(va, vb)
        X, Y = np.array(xa, dtype=object).reshape(sa), np.array(xb, dtype=object).reshape(sb)
        for op, want in ((_cabi.OP_ADD, X + Y), (_cabi.OP_SUB, X - Y), (_cabi.OP_MUL, X * Y)):
            got = dev.binop_view(A, ca, B, cb, op)
            assert ints(got) == (want % p).reshape(-1).tolist(), (sa, sb, op)


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_permutation_and_flip(f):
    ctx, p = ctx_of(f), f.p
    shape = (5, 7, 33)
    vals = values(p, int(np.prod(shape)), 3)
    host = codec.ints_to_limbs(vals, ctx)
    a = offset_copy(DeviceArray.from_ints(ctx, vals))
    for view in (layout.permuted(shape, (2, 0, 1)), layout.flip_view(shape)):
        out = DeviceArray.empty(ctx, view.size)
        s, d = layout.collapse(view, layout.View.full(view.shape))
        dev.copy_view(a, s, out, d)
        assert np.array_equal(out.to_limbs(), host[positions(view).reshape(-1)]), view


# ---- K9: det / solve / inv / matrix_power ------------------------------------------------------------------------------

def matrix(p, n, seed, kind):
    """n x n random residues with every seventh entry p - 1 and a 1 beside the corner; 'swap': a zero leading pivot (the
    first nonzero entry of column 0 is in row 2, or 1 for n = 2); 'singular': row 1 = row 0 + row n - 1"""
    rnd = random.Random(seed)
    v = [p - 1 if i % 7 == 3 else rnd.randrange(p) for i in range(n * n)]
    if n > 1:
        v[1] = 1
    M = [v[i * n:(i + 1) * n] for i in range(n)]
    if kind == 'swap':
        for i in range(min(2, n - 1)):
            M[i][0] = 0
        M[min(2, n - 1)][0] = p - 1
    elif kind == 'singular':
        M[1] = [(x + y) % p for x, y in zip(M[0], M[n - 1])]
    return M


def flat(M):
    return [v for r in M for v in r]


def mat_mul(A, B, p):
    return ((np.array(A, dtype=object) @ np.array(B, dtype=object)) % p).tolist()


def mat_pow(A, e, p):
    n = len(A)
    if e < 0:
        inv = oracle_linalg.solve_ints(flat(A), n, None, n, p)
        A, e = [inv[i * n:(i + 1) * n] for i in range(n)], -e
    R = [[int(i == j) for j in range(n)] for i in range(n)]
    for _ in range(e):
        R = mat_mul(R, A, p)
    return R


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_det_solve_inv(f):
    """n = 1 .. 64 against the oracle (the tile form); n = 129 (the step form for every limb count): det against the
    oracle, solve and inv through A X == B on K1c.  A zero leading pivot forces a row swap."""
    ctx, p = ctx_of(f), f.p
    for n in (1, 2, 3, 17, 64, 129):
        for kind in ('rand', 'swap') if n > 1 else ('rand',):
            M = matrix(p, n, n + f.bits, kind)
            A = DeviceArray.from_ints(ctx, flat(M))
            rhs = values(p, n * 3, n)
            B = DeviceArray.from_ints(ctx, rhs)
            assert ints(dev.det(A, 1, n)) == [oracle_linalg.det_ints(flat(M), n, p)], (n, kind)
            X, Ai = dev.solve(A, B, n, 3), dev.inv(A, n)
            if n <= 64:
                assert ints(X) == oracle_linalg.solve_ints(flat(M), n, rhs, 3, p), (n, kind)
                assert ints(Ai) == oracle_linalg.solve_ints(flat(M), n, None, n, p), (n, kind)
            else:
                assert dev.matmul(ctx, A, X, n, n, 3).count_mismatch(B) == 0, (n, kind)
                assert dev.matmul(ctx, A, Ai, n, n, n).count_mismatch(dev.identity(ctx, n)) == 0, (n, kind)


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_matrix_power_singular_and_batched(f):
    ctx, p = ctx_of(f), f.p
    for n in (1, 2, 3, 17):
        M = matrix(p, n, 7 * n, 'swap' if n > 1 else 'rand')
        A = DeviceArray.from_ints(ctx, flat(M))
        for e in (0, 1, 2, 5, -1, -3):
            assert ints(dev.matrix_power(A, n, e)) == flat(mat_pow(M, e, p)), (n, e)
    for n in (3, 17, 129):
        M = matrix(p, n, n, 'singular')
        A = DeviceArray.from_ints(ctx, flat(M))
        assert ints(dev.det(A, 1, n)) == [0]
        with pytest.raises(ZeroDivisionError, match='no inverse exists'):
            dev.inv(A, n)
        with pytest.raises(ZeroDivisionError, match='no inverse exists'):
            dev.solve(A, DeviceArray.from_ints(ctx, values(p, n, 1)), n, 1)
        with pytest.raises(ZeroDivisionError, match='no inverse exists'):
            dev.matrix_power(A, n, -2)
        torch.cuda.synchronize()
    # a stack of 6 x 6 matrices: random ones, zero leading pivots, zero first columns and all-(p - 1) (rank 1)
    n, batch = 6, 40
    mats = []
    for b in range(batch):
        M = matrix(p, n, 1000 + b, ('rand', 'swap', 'singular')[b % 3])
        if b % 5 == 1:
            for r in M:
                r[0] = 0
        if b % 7 == 4:
            M = [[p - 1] * n for _ in range(n)]
        mats.append(M)
    got = ints(dev.det(DeviceArray.from_ints(ctx, [v for M in mats for v in flat(M)]), batch, n))
    assert got == [oracle_linalg.det_ints(flat(M), n, p) for M in mats]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_inverse_at_256(f):
    ctx, p = ctx_of(f), f.p
    n = 256
    A = DeviceArray.from_ints(ctx, values(p, n * n, f.bits))
    assert dev.matmul(ctx, A, dev.inv(A, n), n, n, n).count_mismatch(dev.identity(ctx, n)) == 0


# ---- K10: convolution ---------------------------------------------------------------------------------------------------

def window(m, n, mode):
    s, g = min(m, n), max(m, n)
    return {'full': (0, m + n - 1), 'same': ((s - 1) // 2, g), 'valid': (s - 1, g - s + 1)}[mode]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_convolve_against_object_convolution(f):
    """one chunk of taps (128, never split) and two or more (split when the window is short), in all three modes; all
    operands p - 1, where output k is its number of terms mod p"""
    ctx, p = ctx_of(f), f.p
    for m, n in ((300, 129), (129, 300), (128, 1000), (1000, 127), (700, 700), (1, 1), (2, 3)):
        a, b = values(p, m, m), values(p, n, n + 1)[::-1]
        full = [int(v) % p for v in np.convolve(np.array(a, dtype=object), np.array(b, dtype=object))]
        A, B = DeviceArray.from_ints(ctx, a), DeviceArray.from_ints(ctx, b)
        for mode in ('full', 'same', 'valid'):
            lo, count = window(m, n, mode)
            assert ints(dev.convolve(ctx, A, m, B, n, lo, count)) == full[lo:lo + count], (m, n, mode)
        top_a, top_b = const(ctx, m, p - 1), const(ctx, n, p - 1)
        ks = np.arange(m + n - 1)
        terms = np.minimum(ks, m - 1) - np.maximum(0, ks - n + 1) + 1
        assert ints(dev.convolve(ctx, top_a, m, top_b, n, 0, m + n - 1)) == [int(t) % p for t in terms], (m, n)


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_convolve_both_sides_of_the_split_decision(f):
    """valid windows of 2 * SM_COUNT runs (tiles only) and one run fewer (split) with 129 taps (two chunks), sampled"""
    ctx, p = ctx_of(f), f.p
    rnd = random.Random(f.bits)
    s = 129
    av = values(p, s, 5)
    a = DeviceArray.from_ints(ctx, av)
    for runs in (2 * SMS - 1, 2 * SMS):
        count = runs * 512
        g = count + s - 1
        b = DeviceArray.random(ctx, g, seed=runs)
        b.t[:64].copy_(const(ctx, 64, p - 1).t)
        got = dev.convolve(ctx, a, s, b, g, s - 1, count)
        idx = [0, 1, count - 1] + [rnd.randrange(count) for _ in range(20)]
        gv = codec.limbs_to_ints(got.t[torch.tensor(idx, device='cuda')].cpu().numpy().view(np.uint64), ctx)
        bv = ints(b)
        for j, v in zip(idx, gv):
            assert int(v) == sum(av[i] * bv[s - 1 + j - i] for i in range(s)) % p, (runs, j)


@pytest.mark.parametrize('f', [BY_NAME['secfxp'], BY_NAME['secint128']], ids=field_id)
def test_convolve_lazy_sums_over_2_20_taps(f):
    """a centre window of 2 * SM_COUNT runs (not split): each work item folds its lazy sums over more than 2^20 taps"""
    ctx, p = ctx_of(f), f.p
    count = 2 * SMS * 512
    m = n = 2**20 + 3 + count // 2
    lo = (m + n - 1) // 2 - count // 2
    top = const(ctx, m, p - 1)
    got = ints(dev.convolve(ctx, top, m, top, n, lo, count))
    ks = np.arange(lo, lo + count, dtype=np.int64)
    terms = np.minimum(ks, m - 1) - np.maximum(0, ks - n + 1) + 1
    assert terms.min() > 2**20
    assert got == [int(t) % p for t in terms]


# ---- K11: division and selection ----------------------------------------------------------------------------------------

def raw_divide(ctx, num, den):
    """ff_div through the C ABI: (status, out) -- out is kept when the call reports a zero divisor"""
    out = DeviceArray.empty(ctx, num.n)
    rc = lib.mpyc_b200_ff_div(ctx.handle, num.ptr, den.ptr, out.ptr, num.n, _stream_ptr())
    return rc, out


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_divide_around_the_batch_layout(f):
    ctx, p = ctx_of(f), f.p
    per_wave = SMS * 1024
    rnd = random.Random(f.bits)
    for n in (1, 2, 255, 2 * per_wave - 1, 2 * per_wave + 1, 4 * per_wave + 7):
        a, b = DeviceArray.random(ctx, n, 5), DeviceArray.random(ctx, n, 6)
        a.t[:min(n, 4)].copy_(DeviceArray.from_ints(ctx, [0, 1, p - 1, 2][:n]).t)
        b.t[:min(n, 4)].copy_(DeviceArray.from_ints(ctx, [p - 1, 1, p - 1, p - 2][:n]).t)
        if b.count_mismatch(DeviceArray(ctx, torch.zeros_like(b.t))) != n:
            continue                                          # a random zero divisor
        q = dev.divide(a, b)
        assert (q * b).count_mismatch(a) == 0, n
        idx = sorted({0, n - 1, n // 2} | {rnd.randrange(n) for _ in range(50)} | set(range(min(n, 4))))
        t = torch.tensor(idx, device='cuda')
        av, bv, qv = (codec.limbs_to_ints(x.t[t].cpu().numpy().view(np.uint64), ctx) for x in (a, b, q))
        assert [int(v) for v in qv] == [int(x) * pow(int(y), -1, p) % p for x, y in zip(av, bv)], n


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
@pytest.mark.parametrize('B', [None, 7, 32])
def test_zero_divisors_first_last_and_inside_a_batch(f, B, monkeypatch):
    """A zero divisor raises, and does not spoil the other quotients of its batch: out holds 0 at each zero divisor and
    num / den everywhere else.  MPYC_B200_INV_BATCH gives 1000 elements batches of 7 and 32 (T = 143, 32)."""
    ctx, p = ctx_of(f), f.p
    if B is not None:
        monkeypatch.setenv('MPYC_B200_INV_BATCH', str(B))
    n = 1000
    num = values(p, n, 1)
    den = [(i * 7919 + 1) % p or 1 for i in range(n)]
    den[2], den[3] = p - 1, p - 2
    T = n if B is None else -(-n // B)
    for zeros in ([0], [n - 1], [3 * T + 5], [T + 1, 4 * T + 1, 5 * T + 1], [T - 1, 2 * T - 1]):
        d = list(den)
        for z in zeros:
            d[z % n] = 0
        N, D = DeviceArray.from_ints(ctx, num), DeviceArray.from_ints(ctx, d)
        rc, out = raw_divide(ctx, N, D)
        assert rc == _cabi.EZERODIV, zeros
        assert ints(out) == [0 if y == 0 else x * pow(y, -1, p) % p for x, y in zip(num, d)], zeros
        with pytest.raises(ZeroDivisionError):
            dev.divide(N, D)
    got = dev.divide(DeviceArray.from_ints(ctx, num), DeviceArray.from_ints(ctx, den))
    assert ints(got) == [x * pow(y, -1, p) % p for x, y in zip(num, den)]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_select_with_affine_sides_both_polarities(f):
    ctx, p = ctx_of(f), f.p
    n = 1237
    xv, yv = values(p, n, 11), values(p, n, 12)[::-1]
    x, y = DeviceArray.from_ints(ctx, xv), offset_copy(DeviceArray.from_ints(ctx, yv))
    m = np.array([(i * 2654435761) >> 7 & 1 for i in range(n)], dtype=bool)
    sx, tx, sy, ty = p - 3, p - 1, 7, 1
    for invert in (False, True):
        pick = m != invert
        for xs in (x, None):
            for ys in (y, None):
                if xs is None and ys is None:
                    continue
                got = dev.select(m, xs, (sx, tx), ys, (sy, ty), n=n, invert=invert)
                want = [((u * sx + tx) % p if xs is not None else tx) if c else ((v * sy + ty) % p if ys is not None else ty)
                        for c, u, v in zip(pick, xv, yv)]
                assert ints(got) == want, (invert, xs is None, ys is None)


# ---- K12: per-element powers ------------------------------------------------------------------------------------------

def exponent_set(p):
    k = p.bit_length()
    return [0, 1, 2, p - 2, p - 1, 2**k - 1, 3, 2**64 - 1, 2**64, p + 1]


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_pow_exp_edge_exponents_and_bases(f):
    ctx, p = ctx_of(f), f.p
    es = exponent_set(p)
    bases = [0, 1, p - 1, 2, p - 2] + values(p, 7, 9)[4:]
    # per-element form: every base with every exponent
    bv = [b for b in bases for _ in es]
    ev = [e for _ in bases for e in es]
    got = ints(dev.pow_exp(ctx, DeviceArray.from_ints(ctx, bv), *codec.exponents_to_limbs(ev)))
    assert got == [pow(b, e, p) for b, e in zip(bv, ev)]
    # fixed-base comb, with negative exponents (inverses) for nonzero bases
    signed = es + [-e for e in es if e] + [-(p - 2), -(2**64 + 1)]
    for b in bases[1:]:
        got = ints(dev.pow_exp(ctx, b, *codec.exponents_to_limbs(signed)))
        assert got == [pow(b, e, p) for e in signed], b
    got = ints(dev.pow_exp(ctx, 0, *codec.exponents_to_limbs(es)))
    assert got == [pow(0, e, p) for e in es]
    with pytest.raises(ZeroDivisionError):
        dev.pow_exp(ctx, 0, *codec.exponents_to_limbs([1, -1]))


# ---- K1c matmul and the Shamir step -----------------------------------------------------------------------------------

@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_matmul_including_split_k(f):
    ctx, p = ctx_of(f), f.p
    for r, k, c in ((5, 7, 3), (33, 65, 17)):
        a, b = values(p, r * k, r), values(p, k * c, c)[::-1]
        got = ints(dev.matmul(ctx, DeviceArray.from_ints(ctx, a), DeviceArray.from_ints(ctx, b), r, k, c))
        want = (np.array(a, dtype=object).reshape(r, k) @ np.array(b, dtype=object).reshape(k, c)) % p
        assert got == want.reshape(-1).tolist(), (r, k, c)
    r, k, c = 1, 3136, 1024                                   # few output tiles: split k, slices summed by K7
    av = values(p, k, 4)
    A, B = DeviceArray.from_ints(ctx, av), DeviceArray.random(ctx, k * c, seed=f.bits)
    B.t[:37 * c].copy_(const(ctx, 37 * c, p - 1).t)
    got = ints(dev.matmul(ctx, A, B, r, k, c))
    cols = sorted({0, 1, c - 1} | set(random.Random(1).sample(range(c), 30)))
    Bc = B.t.view(k, c, ctx.nlimbs)[:, cols].contiguous().reshape(-1, ctx.nlimbs)
    bm = np.array(codec.limbs_to_ints(Bc.cpu().numpy().view(np.uint64), ctx), dtype=object).reshape(k, len(cols))
    want = (np.array(av, dtype=object) @ bm) % p
    assert [got[j] for j in cols] == [int(v) for v in want], 'split-k'
    top = const(ctx, k, p - 1)
    assert set(ints(dev.matmul(ctx, top, const(ctx, k * c, p - 1), r, k, c))) == {k % p}


@pytest.mark.parametrize('f', [BY_NAME['secint128'], BY_NAME['secint168']], ids=field_id)
@pytest.mark.parametrize('m, t', [(3, 1), (5, 2), (7, 3)])
def test_shamir_split_and_recombine(f, m, t):
    ctx, p = ctx_of(f), f.p
    F = orc.field_of(p)
    n = 4099
    s = orc.edge_block(p) + orc.synth_elements(p, n - 8, 1)
    C = [orc.synth_elements(p, n, 2 + j, stream=1) for j in range(t)]
    C[0][:37] = [p - 1] * 37
    shares = dev.shamir_split(ctx, DeviceArray.from_ints(ctx, s), DeviceMatrix.from_ints(ctx, C), t, m)
    assert [r.tolist() for r in shares.to_ints()] == orc.split_np_order(F, s, C, m)
    for xs in (list(range(1, t + 2)), list(range(m - t, m + 1))):
        rec = dev.shamir_recombine(ctx, xs, [shares.row(x - 1) for x in xs])
        assert ints(rec) == s, xs
