"""Share generation of 32-byte aligned rows (the tiled K2, k_split_tiled) around its tile edges.

A CTA owns 8 KB of every row per tile (1024 / L elements), writes the shares of the bench shapes through a
shared-memory stage with TMA bulk stores, and stores straight from registers when m x 8 KB exceeds the stage.  Sizes:
one tile -1 / 0 / +1 element (partial tiles take the per-element path), and one size with more than two full persistent
waves of tiles plus an odd remainder, so that every CTA reuses its stage: a missing fence or bulk-group wait shows up
there as wrong shares.
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

# (p, m, t): the bench shapes (L = 1, 2, 4; the generic 128-bit field) and m = 24, whose 192 KB stage does not fit
SHAPES = [(P64, 3, 1), (P128, 5, 2), (P256, 7, 3), (GEN128, 5, 2), (P128, 24, 2)]
IDS = ['ns64', 'c3', 'c5', 'c3g', 'c3_m24']


def tile_elems(p):
    return 1024 // ((p.bit_length() + 63) // 64)


@pytest.mark.parametrize('p,m,t', SHAPES, ids=IDS)
@pytest.mark.parametrize('delta', [-1, 0, 1])
def test_split_tile_edges_vs_oracle(p, m, t, delta):
    ctx = mpyc_b200.context_for(p)
    F = orc.field_of(p)
    n = tile_elems(p) + delta
    s = (orc.edge_block(p) + orc.synth_elements(p, n - 8, 7 * m + t))[:n]
    C = [orc.synth_elements(p, n, 500 + 17 * j + m, stream=2) for j in range(t)]
    sh = dev.shamir_split(ctx, DeviceArray.from_ints(ctx, s), DeviceMatrix.from_ints(ctx, C), t, m)
    assert [r.tolist() for r in sh.to_ints()] == orc.split_np_order(F, s, C, m)


@pytest.mark.parametrize('p,m,t', SHAPES, ids=IDS)
def test_split_many_waves(p, m, t):
    """Every share against the elementwise kernels (S + sum_j C_j (i+1)^j), and the oracle at the tile seams."""
    ctx = mpyc_b200.context_for(p)
    te = tile_elems(p)
    n = (2 * mpyc_b200_sm_count() * 8 + 11) * te + te // 2 + 1   # > two waves at 8 CTAs per SM; odd partial tile
    S = DeviceArray.random(ctx, n, seed=3, stream_id=1)
    C = DeviceMatrix.empty(ctx, t, n)
    for j in range(t):
        C.t[j].copy_(DeviceArray.random(ctx, n, seed=40 + j, stream_id=2).t)
    sh = dev.shamir_split(ctx, S, C, t, m)
    for i in range(m):
        want = S
        for j in range(t):
            want = want + C.row(j) * pow(i + 1, j + 1, p)
        assert sh.row(i).count_mismatch(want) == 0, f'share row {i}'
    last = n - n % te
    idx = sorted({0, 1, te - 1, te, 3 * te - 1, 3 * te, last - 1, last, n - 2, n - 1})
    sel = torch.tensor(idx, device=S.t.device)
    pick = lambda arr: codec.limbs_to_ints(arr.t.index_select(0, sel).cpu().numpy().view(np.uint64), ctx).tolist()   # noqa: E731
    want = orc.split_np_order(orc.field_of(p), pick(S), [pick(C.row(j)) for j in range(t)], m)
    assert [pick(sh.row(i)) for i in range(m)] == want


def mpyc_b200_sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
