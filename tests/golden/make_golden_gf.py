"""Writes tests/golden/gf_local.json: what the UNMODIFIED reference computes for the GF(2^8) expressions that K15 serves,
for the AES polynomial 283 and the irreducible polynomial 285 -- np_to_bits' / np_from_bits' `np.sum(v << np.arange(l),
axis=-1)` taken into field.array (l = 1..8 and 13), stacked and broadcast matrix products (the S-box's (8, 8) @ (n, 8, 1)
among them, and a public object-array operand on either side), broadcast + - * and a NumPy integer array plus a field array
(np_to_bits' `c_bits + r_bits`).  Cases the hooks leave to the reference (partial stack broadcasts, integer matrices,
negative or wide integers, bool and float operands, mismatched shapes) are recorded too, with the reference's error where it
raises.  Usage: MPYC_REFERENCE=<reference checkout> python tests/golden/make_golden_gf.py"""
import json
import os
import sys

import numpy as np

POLYS = (283, 285)
LS = (1, 2, 3, 4, 5, 6, 7, 8, 13)


def values(shape, salt):
    n = int(np.prod(shape, dtype=np.int64))
    return [(37 * i + 11 * salt + 5) % 256 for i in range(n)]


def ints(kind, shape, salt):
    """Public integer operands: 'i8' bits (np_to_bits' c_bits), 'i64' bytes, 'neg' with a -1, 'big' with 300, 'bool', 'f64'."""
    n = int(np.prod(shape, dtype=np.int64))
    if kind == 'i8':
        return np.int8(np.array([(7 * i + salt) % 3 % 2 for i in range(n)]).reshape(shape))
    v = np.array(values(shape, salt), dtype=np.int64).reshape(shape)
    if kind == 'neg':
        v.flat[1] = -1
    elif kind == 'big':
        v.flat[0] = 300
    elif kind == 'bool':
        return v % 2 == 1
    elif kind == 'f64':
        return v.astype(np.float64)
    return v


# name -> (operands, fn, covered).  Operand: ('f', shape) a field array, ('o', shape) an object ndarray of ints (public),
# (int kind, shape).  covered: the hooks take the call on limb-backed field operands.
CASES = {}
for _l in LS:
    CASES[f'compose_l{_l}'] = ([('f', (6, _l))], 'compose', True)
CASES.update({
    'sbox': ([('f', (8, 8)), ('f', (5, 8, 1))], lambda a, b: a @ b, True),
    'sq4': ([('f', (4, 4)), ('f', (4, 4))], lambda a, b: a @ b, True),
    'stack_left': ([('f', (3, 2, 4)), ('f', (4, 5))], lambda a, b: a @ b, True),
    'stack_right': ([('f', (2, 4)), ('f', (3, 4, 5))], lambda a, b: a @ b, True),
    'stack_both': ([('f', (3, 2, 4)), ('f', (3, 4, 5))], lambda a, b: a @ b, True),
    'stack_4d': ([('f', (2, 3, 2, 4)), ('f', (4, 1))], lambda a, b: a @ b, True),
    'stack_vec_right': ([('f', (3, 2, 4)), ('f', (4,))], lambda a, b: a @ b, True),
    'stack_vec_left': ([('f', (4,)), ('f', (3, 4, 2))], lambda a, b: a @ b, True),
    'np_matmul_stack': ([('f', (2, 3, 4)), ('f', (4, 2))], lambda a, b: np.matmul(a, b), True),
    'pub_left_sbox': ([('o', (8, 8)), ('f', (5, 8, 1))], lambda a, b: a @ b, True),
    'pub_right_stack': ([('f', (5, 2, 8)), ('o', (8, 3))], lambda a, b: a @ b, True),
    'pub_left_sq4': ([('o', (4, 4)), ('f', (4, 4))], lambda a, b: a @ b, True),
    'pub_right_sq4': ([('f', (4, 4)), ('o', (4, 4))], lambda a, b: a @ b, True),
    'stack_partial': ([('f', (2, 1, 3, 4)), ('f', (1, 2, 4, 5))], lambda a, b: a @ b, False),
    'stack_bad': ([('f', (3, 2, 4)), ('f', (3, 5, 2))], lambda a, b: a @ b, False),
    'stack_int': ([('f', (3, 2, 4)), ('i64', (4, 2))], lambda a, b: a @ b, False),
    'bc_rows_add': ([('f', (4, 5)), ('f', (5,))], lambda a, b: a + b, True),
    'bc_col_mul': ([('f', (4, 1)), ('f', (4, 5))], lambda a, b: a * b, True),
    'bc_4d_add': ([('f', (3, 1, 1)), ('f', (2, 3, 4, 5))], lambda a, b: a + b, True),
    'bc_sub_r': ([('f', (5,)), ('f', (4, 5))], lambda a, b: a - b, True),
    'bc_B': ([('f', (6, 8)), ('f', (8,))], lambda a, b: a + b, True),
    'bc_mul_stack': ([('f', (3, 1, 8)), ('f', (4, 8))], lambda a, b: a * b, True),
    'bc_obj': ([('f', (4, 5)), ('o', (5,))], lambda a, b: a + b, True),
    'bc_bad': ([('f', (4, 5)), ('f', (4,))], lambda a, b: a + b, False),
    'int8_add': ([('i8', (6, 8)), ('f', (6, 8))], lambda c, r: c + r, True),
    'int64_add_r': ([('f', (6, 8)), ('i64', (6, 8))], lambda r, c: r + c, True),
    'int8_bc': ([('i8', (8,)), ('f', (6, 8))], lambda c, r: c + r, True),
    'int_neg': ([('neg', (6, 8)), ('f', (6, 8))], lambda c, r: c + r, False),
    'int_big': ([('big', (6, 8)), ('f', (6, 8))], lambda c, r: c + r, False),
    'int_mul': ([('i64', (6, 8)), ('f', (6, 8))], lambda c, r: c * r, False),
    'bool_add': ([('bool', (6, 8)), ('f', (6, 8))], lambda c, r: c + r, False),
    'float_add': ([('f64', (6, 8)), ('f', (6, 8))], lambda c, r: c + r, False),
})


def operands(F, specs, make_field=None):
    """The operands of a case; make_field(shape, salt) builds the field arrays (default: plain arrays of F)."""
    out = []
    for j, (kind, shape) in enumerate(specs):
        if kind == 'f':
            out.append(make_field(shape, j) if make_field else F(np.array(values(shape, j), dtype=object).reshape(shape)))
        elif kind == 'o':
            out.append(np.array(values(shape, j + 7), dtype=object).reshape(shape))
        else:
            out.append(ints(kind, shape, j))
    return out


def compose(F, x, l):
    """np_from_bits' expression (runtime.py:4482-4484) on the raw value v of x"""
    return F(np.sum(x.value << np.arange(l), axis=x.ndim - 1))


def outcome(r):
    """JSON form of a result: an array's shape and integer values, a field element's value, or the exception raised."""
    if isinstance(r, BaseException):
        return ['raises', type(r).__name__, str(r)]
    if hasattr(r, 'value') and isinstance(getattr(r, 'shape', None), tuple):
        v = np.asarray(r.value, dtype=object)
        return ['array', type(r).__name__, list(v.shape), [int(x) for x in v.reshape(-1)]]
    return ['element', type(r).__name__, int(r.value)]


def run_case(F, name, make_field=None):
    specs, fn, _ = CASES[name]
    try:
        ops = operands(F, specs, make_field)
        if fn == 'compose':
            return compose(F, ops[0], specs[0][1][-1])
        return fn(*ops)
    except Exception as e:    # noqa: BLE001
        return e


def main():
    ref = os.environ.get('MPYC_REFERENCE')
    if ref:
        sys.path.insert(0, ref)
    sys.argv = [sys.argv[0], '--no-log']
    from mpyc import finfields, gfpx
    out = []
    for poly in POLYS:
        F = finfields.GF(gfpx.GFpX(2)(poly)).array
        for name in CASES:
            out.append({'poly': poly, 'case': name, 'want': outcome(run_case(F, name))})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'gf_local.json')
    with open(path, 'w') as fh:
        fh.write('[\n' + ',\n'.join(json.dumps(c) for c in out) + '\n]\n')


if __name__ == '__main__':
    main()
