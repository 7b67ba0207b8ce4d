"""Co-located resharing: the `_reshare` exchange of mpyc/runtime.py:603-689 as one GPU collective step.

In MPyC every one of the 2t+1 dealing parties splits its (degree-2t) share vector into m fresh degree-t
shares, pickles row i for party i and sends it over TCP; every party unpickles the 2t+1 rows it received and
recombines them (runtime.py:660-680; framing asyncoro.py:54-64).  When the m parties of a computation live on
the GPUs of one box (benchmark / simulation mode; party j on rank j % world) the same step is

    K2 on every dealer  ->  exchange of limb rows between GPUs  ->  K3s on every party

with the rows going GPU to GPU as limb buffers: no Python ints, no pickle, no host copies.  The exchange is a
grouped point-to-point batch (`torch.distributed.batch_isend_irecv`: one ncclGroupStart/End of ncclSend/ncclRecv
over NVLink on the nccl backend), posted straight on the rows of the share matrices K2 wrote -- rows that stay on
the same rank are not copied at all.  Both ends enumerate the (dealer, recipient) pairs in the same sorted
order, which is how NCCL matches sends with receives between a pair of ranks.

The arithmetic is injected as an `engine` (split / recombine on tensors) so that the routing can be exercised on
CPU tensors over gloo (tests/test_exchange_gloo.py) with the oracle standing in for the kernels; on the GPU the
engine is `DeviceEngine` below (mpyc_b200.device: K2 in generate mode, K3).

`PeerReshare` goes one step further on NVLink-connected GPUs: K2 itself stores each recipient's row into the
recipient GPU's memory, so the exchange is no separate pass at all.
"""
import torch
import torch.distributed as dist


def owner(party, world):
    """Rank that hosts a party."""
    return party % world


def local_parties(m, world, rank):
    return [j for j in range(m) if owner(j, world) == rank]


class DeviceEngine:
    """K2 (coefficients from the in-kernel ChaCha20 stream) and K3 on device-resident limb tensors."""

    def __init__(self, ctx):
        self.ctx = ctx
        self._nonce = 0

    def split(self, x, t, m):
        """x: int64 (n, L) limb tensor -> (m, n, L) tensor of shares (row i for party i)."""
        from mpyc_b200 import device as dev
        self._nonce += 1
        sh = dev.shamir_split_generate(self.ctx, dev.DeviceArray(self.ctx, x), t, m, nonce=self._nonce)
        return sh.t

    def recombine(self, xs, rows):
        from mpyc_b200 import device as dev
        return dev.shamir_recombine(self.ctx, xs, [dev.DeviceArray(self.ctx, r) for r in rows]).t

    def empty_like_row(self, x):
        return torch.empty_like(x)


def reshare(engine, shares, t, m, group=None, first_dealer=0):
    """One resharing round.

    shares: {party j: limb tensor (n, L)} for the parties hosted on this rank (their current shares, e.g. the
    degree-2t local products of a secure multiplication).  Dealers are the 2t+1 parties first_dealer,
    first_dealer+1, ... (mod m) -- runtime.py's `uci` load balancing.  Returns {party i: new degree-t share}
    for the same local parties.  Collective: every rank of the group must call it."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    mine = local_parties(m, world, rank)
    if sorted(shares) != mine:
        raise ValueError(f'rank {rank} hosts parties {mine}, got shares for {sorted(shares)}')
    dealers = [(first_dealer + a) % m for a in range(2 * t + 1)]
    if len(set(dealers)) != len(dealers):
        raise ValueError('resharing needs m >= 2t+1 parties')
    # 1. every local dealer splits its share vector: dealt[j] is (m, n, L), row i goes to party i
    dealt = {j: engine.split(shares[j], t, m) for j in dealers if j in shares}
    some = next(iter(shares.values()), None)             # None: this rank hosts no party (world > m) and only joins the group calls
    # 2. exchange: recv[i][a] = row i of dealer dealers[a]'s matrix
    recv = {i: [None] * len(dealers) for i in mine}
    ops = []
    for a, j in enumerate(dealers):                      # the same (dealer, recipient) order on every rank
        src = owner(j, world)
        for i in range(m):
            dst = owner(i, world)
            if src == rank and dst == rank:
                recv[i][a] = dealt[j][i]                 # stays on this GPU: use the row K2 wrote, no copy
            elif src == rank:
                ops.append(dist.P2POp(dist.isend, dealt[j][i].contiguous(), _global_rank(dst, group), group))
            elif dst == rank:
                buf = engine.empty_like_row(some)
                recv[i][a] = buf
                ops.append(dist.P2POp(dist.irecv, buf, _global_rank(src, group), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    # 3. every local party recombines the 2t+1 rows it now holds
    xs = [j + 1 for j in dealers]
    return {i: engine.recombine(xs, recv[i]) for i in mine}


class PeerReshare:
    """The resharing round with the exchange fused into share generation: every dealer's K2 stores row i straight
    into the receive buffer of party i's GPU (peer memory mapped through CUDA IPC, stores travel over NVLink), one
    stream-ordered all-reduce tells every rank that all rows have landed, K3s recombines.  No staging matrix, no copy
    pass: a share row crosses HBM once on the way out instead of three times (K2 write, NCCL read, NCCL write).

    Receive buffers are double-buffered by round parity; a dealer can only be one round ahead of a recipient
    (the all-reduce of round r+1 cannot complete before the recipient has issued its K3 of round r), so the rows
    of round r+2 never overwrite rows still being read.  One instance per (field, m, t, n)."""

    def __init__(self, ctx, m, t, n, group=None, first_dealer=0):
        import ctypes
        from mpyc_b200._cabi import lib, check
        self.ctx, self.m, self.t, self.n, self.group = ctx, m, t, n, group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.mine = local_parties(m, self.world, self.rank)
        self.dealers = [(first_dealer + a) % m for a in range(2 * t + 1)]
        if len(set(self.dealers)) != len(self.dealers) or m > 32:
            raise ValueError('peer resharing needs 2t+1 <= m <= 32')
        L = ctx.nlimbs
        self.row_bytes = (n * L * 8 + 31) // 32 * 32            # rows 32-byte aligned (32-byte store groups)
        self.slots = max(len(local_parties(m, self.world, r)) for r in range(self.world))
        nbytes = 2 * self.slots * len(self.dealers) * self.row_bytes
        # own receive buffer: [generation][local party slot][dealer index] rows, exported to the other ranks
        own, handle = ctypes.c_void_p(), (ctypes.c_uint8 * 64)()
        check(lib.mpyc_b200_peer_alloc(nbytes, ctypes.byref(own), handle))
        self._own = own.value
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle), group=group)
        self.base = {}
        for r, h in enumerate(handles):
            if r == self.rank:
                self.base[r] = self._own
            else:
                ptr = ctypes.c_void_p()
                check(lib.mpyc_b200_peer_open((ctypes.c_uint8 * 64).from_buffer_copy(h), ctypes.byref(ptr)))
                self.base[r] = ptr.value
        self.flag = torch.zeros(1, dtype=torch.int32, device='cuda')
        self.round = 0
        self._nonce = 0
        dist.barrier(group)                                    # nobody writes before every mapping exists

    def close(self):
        """Unmap the peers' buffers and free the own one (collective: every rank must call it)."""
        from mpyc_b200._cabi import lib, check
        if self._own is None:
            return
        torch.cuda.synchronize()
        dist.barrier(self.group)
        for r, ptr in self.base.items():
            if r != self.rank:
                check(lib.mpyc_b200_peer_close(ptr))
        dist.barrier(self.group)
        check(lib.mpyc_b200_peer_free(self._own))
        self._own = None

    def _row_ptr(self, gen, party, dealer_index):
        slot = party // self.world
        return self.base[owner(party, self.world)] + ((gen * self.slots + slot) * len(self.dealers) + dealer_index) * self.row_bytes

    def reshare(self, shares):
        """shares: {party j: limb tensor (n, L)} for the local parties; returns {party i: new share tensor (n, L)}."""
        import ctypes
        from mpyc_b200 import _cabi, device as dev
        from mpyc_b200._cabi import lib, check
        if sorted(shares) != self.mine:
            raise ValueError(f'rank {self.rank} hosts parties {self.mine}, got shares for {sorted(shares)}')
        gen = self.round & 1
        for a, j in enumerate(self.dealers):
            if j in shares:
                self._nonce += 1
                dev.shamir_split_generate_rows(self.ctx, dev.DeviceArray(self.ctx, shares[j]), self.t, self.m,
                                               [self._row_ptr(gen, i, a) for i in range(self.m)], nonce=self._nonce)
        dist.all_reduce(self.flag, group=self.group)           # stream-ordered: completes once every rank's K2s are done
        xs = _cabi.i64_array([j + 1 for j in self.dealers])
        zero = _cabi.i64_array([0])
        L, n, k = self.ctx.nlimbs, self.n, len(self.dealers)
        out = {}
        for i in self.mine:
            res = torch.empty((n, L), dtype=torch.int64, device='cuda')
            rows = _cabi.ptr_array([self._row_ptr(gen, i, a) for a in range(k)])
            check(lib.mpyc_b200_shamir_recombine(self.ctx.handle, rows, xs, k, zero, 1, ctypes.c_void_p(res.data_ptr()), n, n,
                                                 dev._stream_ptr()))
            out[i] = res
        self.round += 1
        return out


def _global_rank(group_rank, group):
    return group_rank if group is None else dist.get_global_rank(group, group_rank)
