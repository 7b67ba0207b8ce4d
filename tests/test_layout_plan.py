"""mpyc_b200.layout (K8's host plans) against NumPy: every descriptor is applied to np.arange(n).reshape(shape) by a small
NumPy interpreter (tests/oracle_layout.positions) and must give NumPy's own result, before and after collapsing; keys and
arguments NumPy rejects are "not covered"."""
import random

import numpy as np
import pytest

from mpyc_b200 import layout
from oracle_layout import positions


def apply(flat, view):
    return flat[positions(view)]


def scatter(n, pieces, sources):
    out = np.full(n, -1, dtype=np.int64)
    for i, s, d in pieces:
        out[positions(d).reshape(-1)] = apply(sources[i], s).reshape(-1)
    return out


def check_copy(src_flat, view, want):
    got = apply(src_flat, view)
    assert got.shape == want.shape and np.array_equal(got, want)
    c = layout.collapse(view, layout.View.full(view.shape))
    assert c is not None and len(c[0].shape) <= layout.MAX_RANK
    flat = scatter(want.size, [(0,) + c], [src_flat])
    assert np.array_equal(flat, want.reshape(-1))


def random_key(rng, shape):
    items = []
    nd = len(shape)
    d = 0
    arr_at = rng.randrange(nd + 1) if nd and rng.random() < 0.5 else -1
    ell = rng.random() < 0.3
    while d < nd:
        if ell and rng.random() < 0.3:
            items.append(Ellipsis)
            break
        n = shape[d]
        if rng.random() < 0.15:
            items.append(None)
            continue
        if d == arr_at:
            k = rng.randrange(0, 5)
            idx = [rng.randrange(-n, n) for _ in range(k)] if n else []
            items.append(np.array(idx, dtype=np.int64) if rng.random() < 0.5 else idx)
        else:
            r = rng.random()
            if r < 0.25 and n:
                items.append(rng.randrange(-n, n))
            elif r < 0.3:
                items.append(n + 3)                                     # out of bounds: NumPy raises
            else:
                start = rng.choice([None, rng.randrange(-n - 2, n + 2)])
                stop = rng.choice([None, rng.randrange(-n - 2, n + 2)])
                step = rng.choice([None, 1, -1, 2, -2, 3, -3])
                items.append(slice(start, stop, step))
        d += 1
        if rng.random() < 0.2:
            break
    if rng.random() < 0.1:
        items.append(None)
    return tuple(items) if len(items) != 1 or rng.random() < 0.5 else items[0]


def test_random_keys_match_numpy():
    rng = random.Random(8)
    covered = raised = arrays = 0
    for trial in range(3000):
        nd = rng.randrange(0, 8)
        shape = tuple(rng.randrange(0, 5) if rng.random() < 0.1 else rng.randrange(1, 5) for _ in range(nd))
        key = random_key(rng, shape)
        x = np.arange(int(np.prod(shape, dtype=np.int64))).reshape(shape)
        try:
            want = x[key]
        except (IndexError, ValueError, TypeError):
            want = None
        plan = layout.getitem_plan(shape, key)
        if want is None:
            assert plan is None, (shape, key)
            raised += 1
            continue
        assert plan is not None, (shape, key)
        view, out_shape, scalar = plan
        assert scalar == (not isinstance(want, np.ndarray)), (shape, key)
        want = np.asarray(want)
        assert out_shape == want.shape, (shape, key)
        check_copy(x.reshape(-1), view, want)
        covered += 1
        arrays += view.index_axis >= 0
    assert covered > 1500 and raised > 100 and arrays > 200


def test_index_array_placement():
    x = np.arange(2 * 3 * 4 * 5).reshape(2, 3, 4, 5)
    for key in [(0, slice(None), [1, 2]), (slice(None), 0, [1, 2]), ([1, 0], slice(None), 2), (Ellipsis, [3, 0, 3]),
                (slice(None), [2, 1], 1), (1, None, [0, 2]), (None, [1], Ellipsis, None), ([1, -1],), (slice(None, None, -1), [0])]:
        view, shape, _ = layout.getitem_plan(x.shape, key)
        check_copy(x.reshape(-1), view, x[key])


@pytest.mark.parametrize('key', [np.array([True, False]), True, (np.array([0]), np.array([1])), [[0, 1]], np.array([[0]]),
                                 np.array([0.5]), (Ellipsis, Ellipsis), slice(0, 1, 0), (0, 0, 0), 1.0, 'a', [0, None]])
def test_keys_not_covered(key):
    assert layout.getitem_plan((2, 3), key) is None


def test_contiguous_selections_are_runs():
    shape = (4, 3, 2)
    for key, run in [(slice(1, 3), (6, 18)), (2, (12, 18)), ((1, 2), (10, 12)), ((slice(None), slice(None)), (0, 24)),
                     ((Ellipsis,), (0, 24)), ((None, 3), (18, 24)), ((1, slice(1, 2), None), (8, 10))]:
        view, _, _ = layout.getitem_plan(shape, key)
        assert view.run() == run, key
    for key in [slice(None, None, 2), (slice(None), 1), (Ellipsis, 0), [0, 1]]:
        view, _, _ = layout.getitem_plan(shape, key)
        assert view.run() is None, key


def test_permutations_match_numpy():
    rng = random.Random(3)
    for nd in range(0, 7):
        shape = tuple(rng.randrange(1, 5) for _ in range(nd))
        x = np.arange(int(np.prod(shape))).reshape(shape)
        perms = [None, tuple(rng.sample(range(nd), nd)), tuple(k - nd for k in rng.sample(range(nd), nd))]
        for perm in perms:
            order = layout.transpose_axes(nd, (perm,))
            check_copy(x.reshape(-1), layout.permuted(shape, order), np.transpose(x, perm))
            assert order == layout.transpose_axes(nd, perm if perm else ())
        if nd >= 2:
            for a1, a2 in [(0, -1), (1, 0), (-2, nd - 1)]:
                check_copy(x.reshape(-1), layout.permuted(shape, layout.swapaxes_axes(nd, a1, a2)), np.swapaxes(x, a1, a2))
            for s, d in [(0, -1), ((0, 1), (-1, -2)), (-1, 0)]:
                check_copy(x.reshape(-1), layout.permuted(shape, layout.moveaxis_axes(nd, s, d)), np.moveaxis(x, s, d))
    for bad in [lambda: layout.transpose_axes(2, ((0, 0),)), lambda: layout.transpose_axes(3, ((0, 1),)),
                lambda: layout.swapaxes_axes(2, 0, 2), lambda: layout.moveaxis_axes(3, (0, 1), 0),
                lambda: layout.transpose_axes(2, ((0, 1.5),))]:
        with pytest.raises((ValueError, TypeError, IndexError)):
            bad()


def test_flip_and_roll_match_numpy():
    for shape in [(5,), (3, 4), (2, 3, 4), (2, 0, 3), (1, 4, 1)]:
        x = np.arange(int(np.prod(shape))).reshape(shape)
        nd = len(shape)
        for axis in [None, 0, -1, tuple(range(nd))] + ([(0, nd - 1)] if nd > 1 else []):
            check_copy(x.reshape(-1), layout.flip_view(shape, axis), np.flip(x, axis))
        for shift in [0, 1, -2, 7, 100]:
            for axis in [None] + list(range(-nd, nd)):
                want = np.roll(x, shift, axis)
                plan = layout.pieces(layout.roll_plan(shape, shift, axis))
                assert len(plan) <= 2
                assert np.array_equal(scatter(x.size, plan, [x.reshape(-1)]), want.reshape(-1))
    with pytest.raises(ValueError):
        layout.flip_view((2, 3), 2)


def test_joins_match_numpy():
    rng = np.random.default_rng(1)
    cases = [([(2, 3), (4, 3)], 0), ([(2, 3), (2, 5)], 1), ([(2, 3), (2, 1), (2, 2)], -1), ([(2, 3, 4), (2, 3, 1)], 2),
             ([(2, 3), (5,)], None), ([(3,), (4,)], 0), ([(2, 0), (2, 3)], 1)]
    for shapes, axis in cases:
        xs = [rng.integers(0, 1000, size=s) for s in shapes]
        out_shape, items = layout.concatenate_plan(shapes, axis)
        want = np.concatenate(xs, axis=axis)
        assert out_shape == want.shape
        got = scatter(want.size, layout.pieces(items), [x.reshape(-1) for x in xs])
        assert np.array_equal(got, want.reshape(-1))
    for shapes, axis in [([(2, 3), (2, 3), (2, 3)], 0), ([(2, 3)] * 2, 1), ([(2, 3)] * 2, 2), ([(2, 3)] * 2, -1), ([(4,)] * 3, 1)]:
        xs = [rng.integers(0, 1000, size=s) for s in shapes]
        out_shape, items = layout.stack_plan(shapes, axis)
        want = np.stack(xs, axis=axis)
        assert out_shape == want.shape
        assert np.array_equal(scatter(want.size, layout.pieces(items), [x.reshape(-1) for x in xs]), want.reshape(-1))
    for shapes in [[(3,), (3,)], [(2, 3), (3,)], [(2, 3), (1, 3)], [(2, 2, 2), (1, 2, 2)]]:
        xs = [rng.integers(0, 1000, size=s) for s in shapes]
        want = np.vstack(xs)
        out_shape, items = layout.concatenate_plan(layout.vstack_shapes(shapes), 0)
        assert out_shape == want.shape
        assert np.array_equal(scatter(want.size, layout.pieces(items), [x.reshape(-1) for x in xs]), want.reshape(-1))
    for shapes in [[(3,), (2,)], [(2, 3), (2, 1)], [(2, 2, 2), (2, 1, 2)]]:
        xs = [rng.integers(0, 1000, size=s) for s in shapes]
        want = np.hstack(xs)
        out_shape, items = layout.concatenate_plan(*layout.hstack_axis(shapes))
        assert out_shape == want.shape
        assert np.array_equal(scatter(want.size, layout.pieces(items), [x.reshape(-1) for x in xs]), want.reshape(-1))
    for bad in [lambda: layout.concatenate_plan([(2, 3), (3, 3)], 1), lambda: layout.concatenate_plan([(), ()], 0),
                lambda: layout.concatenate_plan([(2,), (2, 1)], 0), lambda: layout.concatenate_plan([(2,)], 1),
                lambda: layout.stack_plan([(2,), (3,)], 0), lambda: layout.stack_plan([(2,)], 2),
                lambda: layout.concatenate_plan([], 0)]:
        with pytest.raises(ValueError):
            bad()


def test_broadcasts_match_numpy():
    cases = [((5, 1), (5, 4)), ((3, 1, 1), (2, 3, 4, 5)), ((4, 3), (3,)), ((3,), (4, 3)), ((1,), (6,)), ((), (2, 3)),
             ((2, 1, 3), (4, 1)), ((0, 3), (1, 3))]
    for sa, sb in cases:
        a = np.arange(int(np.prod(sa))).reshape(sa)
        b = 1000 + np.arange(int(np.prod(sb))).reshape(sb)
        out, va, vb = layout.broadcast_views(sa, sb)
        assert out == np.broadcast_shapes(sa, sb)
        c = layout.collapse(va, vb)
        assert np.array_equal(apply(a.reshape(-1), c[0]).reshape(out) + apply(b.reshape(-1), c[1]).reshape(out), a + b)
    with pytest.raises(ValueError):
        layout.broadcast_views((2, 3), (4,))


def test_reshapes_match_numpy():
    assert layout.reshaped((3, 4), np.expand_dims, 1) == (3, 1, 4)
    assert layout.reshaped((3, 4), np.expand_dims, (0, -1)) == (1, 3, 4, 1)
    assert layout.reshaped((1, 3, 1), np.squeeze, None) == (3,)
    assert layout.reshaped((1, 3, 1), np.squeeze, 2) == (1, 3)
    with pytest.raises(ValueError):
        layout.reshaped((1, 3), np.squeeze, 1)
    with pytest.raises(np.exceptions.AxisError):
        layout.reshaped((3,), np.expand_dims, 3)


def test_collapsing():
    # contiguous in both views: one axis
    v = layout.View.full((2, 3, 4))
    c = layout.collapse(v, layout.View.full((2, 3, 4)))
    assert c[0].shape == (24,) and c[0].strides == (1,)
    # a transpose of (2, 3, 4) -> (4, 3, 2) keeps three axes; swapping the last two of (5, 6, 7) merges nothing, and
    # (a, b, c) -> (b, c, a) merges b and c
    assert layout.collapse(layout.permuted((2, 3, 4), (2, 1, 0)), layout.View.full((4, 3, 2)))[0].shape == (4, 3, 2)
    assert layout.collapse(layout.permuted((2, 3, 4), (1, 2, 0)), layout.View.full((3, 4, 2)))[0].shape == (12, 2)
    # unit axes are dropped; an index axis is kept and never merged
    view, _, _ = layout.getitem_plan((1, 4, 5), (slice(None), [0, 2], slice(None)))
    s, d = layout.collapse(view, layout.View.full(view.shape))
    assert s.shape == (2, 5) and s.index_axis == 0
    view, _, _ = layout.getitem_plan((3, 4), (slice(None), [2]))
    s, d = layout.collapse(view, layout.View.full(view.shape))
    assert s.shape == (3,) and s.index_axis == -1 and s.offset == 2
    # rank > 6 after collapsing is not covered
    shape = (2,) * 8
    assert layout.collapse(layout.permuted(shape, tuple(reversed(range(8)))), layout.View.full(shape)) is None
    assert layout.pieces([(0, layout.permuted(shape, tuple(reversed(range(8)))), layout.View.full(shape))]) is None
    assert layout.collapse(layout.permuted(shape, (1, 0, 2, 3, 4, 5, 6, 7)), layout.View.full(shape))[0].shape == (2, 2, 64)
    # empty views collapse to one empty axis
    assert layout.collapse(layout.View.full((3, 0, 2)), layout.View.full((3, 0, 2)))[0].shape == (0,)
