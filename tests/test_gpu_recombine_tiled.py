"""Lagrange recombination of 32-byte aligned rows (the tiled K3, k_recombine_tiled) around its tile edges.

A CTA owns 8 KB of each input and output row per tile (1024 / L elements).  For k <= 4 (k <= 2 at L = 4) the rows
stay in registers for every point and the next tile is prefetched; larger k stream the rows per point.  Sizes: one
tile -1 / 0 / +1 element (partial tiles take the per-element path), and one size with more than two full persistent
waves of tiles plus an odd remainder, so that every CTA carries its prefetched rows across many tiles.  Both lambda
forms: the small one (x-coordinates 1..k at 0, lambda a signed 64-bit constant) and the full one (lambda a field
element).  Results are checked against the oracle at the tile seams and against sum_i lambda_i * row_i built from the
elementwise kernels over whole arrays.
"""
import numpy as np
import pytest

from oracle import shamir_oracle as orc

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import codec, device as dev        # noqa: E402
from mpyc_b200.device import DeviceArray, DeviceMatrix   # noqa: E402

P64, P128, P256 = 2**64 - 189, 2**128 - 173, 2**256 - 189
GEN128 = 0x800000000000000000000000000000fb
FIELDS = [P64, P128, P256, GEN128]
FIDS = ['p64', 'p128', 'p256', 'gen128']

# (xs, x_r): xs = 1..k at 0 takes the small-lambda form; [2, 5, 7] at 4 the full one
FORMS = [((1,), 0), ((1, 2), 0), ((1, 2, 3), 0), (tuple(range(1, 8)), 0), ((2, 5, 7), 4)]
FORM_IDS = ['small_k1', 'small_k2', 'small_k3', 'small_k7', 'full_k3']


def nlimbs(p):
    return (p.bit_length() + 63) // 64


def tile_elems(p):
    return 1024 // nlimbs(p)


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def many_waves(p):
    te = tile_elems(p)
    return (2 * sm_count() * 8 + 11) * te + te // 2 + 1   # > two waves at 8 CTAs per SM; odd partial tile


def random_rows(ctx, k, n, seed):
    return [DeviceArray.random(ctx, n, seed=seed + i, stream_id=3) for i in range(k)]


def lagrange_sum(ctx, xs, rows, x_r):
    """sum_i lambda_i * row_i with the elementwise kernels (K1)."""
    lam = orc.recombination_vector(orc.field_of(ctx.modulus), list(xs), x_r)
    want = rows[0] * int(lam[0])
    for r, l_i in zip(rows[1:], lam[1:]):
        want = want + r * int(l_i)
    return want


def seams(n, te):
    last = n - n % te
    return sorted({i for i in (0, 1, te - 1, te, 3 * te - 1, 3 * te, last - 1, last, n - 2, n - 1) if 0 <= i < n})


def pick(ctx, arr, idx):
    sel = torch.tensor(idx, device=arr.t.device)
    return codec.limbs_to_ints(arr.t.index_select(0, sel).cpu().numpy().view(np.uint64), ctx).tolist()


def placed(ctx, src, limb_off):
    """A copy of src that starts limb_off limbs into a buffer of its own (the buffer is returned to keep it alive)."""
    n, L = src.n, ctx.nlimbs
    buf = torch.zeros(limb_off + n * L + 8, dtype=torch.int64, device=src.t.device)
    view = buf[limb_off:limb_off + n * L].view(n, L)
    view.copy_(src.t)
    return DeviceArray(ctx, view), buf


def check_whole(ctx, xs, rows, x_r, got):
    assert got.count_mismatch(lagrange_sum(ctx, xs, rows, x_r)) == 0
    idx = seams(got.n, tile_elems(ctx.modulus))
    want = orc.recombine(orc.field_of(ctx.modulus), list(xs), [pick(ctx, r, idx) for r in rows], x_r)
    assert pick(ctx, got, idx) == want


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('xs,x_r', FORMS, ids=FORM_IDS)
@pytest.mark.parametrize('delta', [-1, 0, 1])
def test_recombine_tile_edges_vs_oracle(p, xs, x_r, delta):
    ctx = mpyc_b200.context_for(p)
    F = orc.field_of(p)
    n = tile_elems(p) + delta
    S = [(orc.edge_block(p) + orc.synth_elements(p, n - 8, 31 * i + len(xs)))[:n] for i in range(len(xs))]
    S = [s[i:] + s[:i] for i, s in enumerate(S)]   # the edge values meet different neighbours in every row
    got = dev.shamir_recombine(ctx, list(xs), [DeviceArray.from_ints(ctx, s) for s in S], x_r)
    assert got.to_ints().tolist() == orc.recombine(F, list(xs), S, x_r)


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('xs,x_r', FORMS[2:], ids=FORM_IDS[2:])
def test_recombine_many_waves(p, xs, x_r):
    ctx = mpyc_b200.context_for(p)
    rows = random_rows(ctx, len(xs), many_waves(p), seed=11)
    check_whole(ctx, xs, rows, x_r, dev.shamir_recombine(ctx, list(xs), rows, x_r))


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('x_r', [0, 40], ids=['small', 'full'])
def test_recombine_many_rows(p, x_r):
    """k = 33: the rows are streamed per point instead of held in registers."""
    ctx = mpyc_b200.context_for(p)
    xs = tuple(range(1, 34))
    rows = random_rows(ctx, len(xs), many_waves(p) // 4, seed=70)
    check_whole(ctx, xs, rows, x_r, dev.shamir_recombine(ctx, list(xs), rows, x_r))


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('xs,pts', [((1, 2, 3), [0, 9, 10, 11, 12, 13]), ((2, 5, 7), [4, 0, 1, 3, 6, 8])],
                         ids=['small', 'full'])
@pytest.mark.parametrize('width', [2, 6])
def test_recombine_width_strided(p, xs, pts, width):
    """Several points into an output matrix whose row stride exceeds n (32-byte aligned), the rows loaded once per
    tile for all of them."""
    ctx = mpyc_b200.context_for(p)
    L = ctx.nlimbs
    te = tile_elems(p)
    n = (2 * sm_count() + 3) * te + 7
    pad = {1: 4, 2: 2, 4: 1}[L] * 3
    pts = pts[:width]
    rows = random_rows(ctx, len(xs), n, seed=90)
    base = torch.zeros((width, n + pad, L), dtype=torch.int64, device='cuda')
    out = DeviceMatrix(ctx, base[:, :n])
    assert out.stride == n + pad
    dev.shamir_recombine(ctx, list(xs), rows, pts, out=out)
    for j, x_r in enumerate(pts):
        check_whole(ctx, xs, rows, x_r, out.row(j))
    assert int(torch.count_nonzero(base[:, n:])) == 0   # nothing written into the padding


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('xs,x_r', [FORMS[2], FORMS[4]], ids=['small', 'full'])
def test_recombine_rows_in_separate_buffers(p, xs, x_r):
    """Every row in a buffer of its own, each starting mid-buffer at a different 32-byte aligned offset."""
    ctx = mpyc_b200.context_for(p)
    src = random_rows(ctx, len(xs), many_waves(p) // 8, seed=120)
    held = [placed(ctx, r, 4 * (i + 1)) for i, r in enumerate(src)]
    rows = [a for a, _ in held]
    assert all(r.t.data_ptr() % 32 == 0 for r in rows)
    check_whole(ctx, xs, rows, x_r, dev.shamir_recombine(ctx, list(xs), rows, x_r))


@pytest.mark.parametrize('p', FIELDS, ids=FIDS)
@pytest.mark.parametrize('xs,x_r', [FORMS[2], FORMS[4]], ids=['small', 'full'])
def test_recombine_unaligned_row_falls_back(p, xs, x_r):
    """One row only 8-byte aligned: the per-element kernel serves the call and its result is the same."""
    ctx = mpyc_b200.context_for(p)
    src = random_rows(ctx, len(xs), 3 * tile_elems(p) + 5, seed=150)
    odd, _buf = placed(ctx, src[1], 1)
    assert odd.t.data_ptr() % 32 == 8
    rows = [src[0], odd] + src[2:]
    check_whole(ctx, xs, rows, x_r, dev.shamir_recombine(ctx, list(xs), rows, x_r))
    assert dev.shamir_recombine(ctx, list(xs), src, x_r).count_mismatch(dev.shamir_recombine(ctx, list(xs), rows, x_r)) == 0
