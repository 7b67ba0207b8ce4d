"""MPyC program for K15: the AES S-box and its inverse on n secret SecFld(2^8) bytes in one batch each, then one AES-128
encryption of the FIPS-197 example block under a secret key (key schedule, SubBytes, ShiftRows, MixColumns, AddRoundKey),
then output.

    python tests/run_installed.py tests/programs/resident_aes.py [n] [-M3]

The S-box is x -> Aff(x^254): x^254 is the inverse (0 for 0), its bits (np_to_bits) go through the affine map M b + (1, 1, 0,
0, 0, 1, 1, 0) over GF(2), where row i of M has ones in columns i, i+4, i+5, i+6, i+7 mod 8, and np_from_bits makes the byte
again.  The bits are one (n, 8) array, M multiplies them as the stack M @ bits[..., None], so each S-box call is one batched
product.  Prints the opened results, then one line 'counts <name> {...}' per step with the engine's counters around it
(absent without the engine): 'c_settles' counts the limb-backed values turned into Python ints inside Runtime.np_to_bits
(its opened, public `c`), 'other_settles' all others.
"""
import json
import sys

import numpy as np
from mpyc.runtime import mpc

secfld = mpc.SecFld(2**8)
gf = secfld.field
settles = {'c': 0, 'other': 0}


def affine_rows(cols):
    return gf.array(np.array([[1 if (j - i) % 8 in cols else 0 for j in range(8)] for i in range(8)]))


M = affine_rows((0, 4, 5, 6, 7))          # the affine map of the S-box
M_INV = affine_rows((2, 5, 7))            # its inverse over GF(2)
AFFINE = gf.array(np.array([1, 1, 0, 0, 0, 1, 1, 0]))
MIX = gf.array(np.array([[(2, 3, 1, 1)[(j - i) % 4] for j in range(4)] for i in range(4)]))


def sub_bytes(x):
    b = mpc.np_to_bits(x ** 254)
    b = (M @ b[..., np.newaxis]).reshape(*b.shape) + AFFINE
    return mpc.np_from_bits(b)


def inv_sub_bytes(x):
    b = mpc.np_to_bits(x) + AFFINE
    b = (M_INV @ b[..., np.newaxis]).reshape(*b.shape)
    return mpc.np_from_bits(b) ** 254


def round_keys(key):
    """the 11 round keys (4 x 4 column-major states) of AES-128 for a secret 4 x 4 key state"""
    cols = [key[:, j] for j in range(4)]
    rcon = 1
    for i in range(4, 44):
        t = cols[-1]
        if i % 4 == 0:
            t = np.roll(sub_bytes(t), -1) + gf.array(np.array([rcon, 0, 0, 0]))
            rcon = (rcon << 1) ^ (0x11B if rcon & 0x80 else 0)
        cols.append(cols[i - 4] + t)
    return [np.stack(cols[4 * r:4 * r + 4], axis=1) for r in range(11)]


def encrypt(keys, s):
    s = s + keys[0]
    for r in range(1, 11):
        s = sub_bytes(s)
        s = np.stack([np.roll(s[i], -i) for i in range(4)])
        if r < 10:
            s = MIX @ s
        s = s + keys[r]
    return s


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls, c_settles=settles['c'], other_settles=settles['other'])


def watch_settles():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return
    orig = resident.LimbValue._materialise

    def mat(self):
        if self._ints is None:
            f = sys._getframe(1)
            while f is not None and not (f.f_code.co_name == 'np_to_bits' and f.f_code.co_filename.endswith('runtime.py')):
                f = f.f_back
            settles['c' if f is not None else 'other'] += 1
        return orig(self)
    resident.LimbValue._materialise = mat


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    watch_settles()
    n = int(sys.argv[1]) if sys.argv[1:] else 256
    await mpc.start()
    x = mpc.input(secfld.array(gf.array(np.arange(n) % 256)), senders=0)
    k = mpc.input(secfld.array(gf.array(np.arange(16).reshape(4, 4).T)), senders=0)
    p = mpc.input(secfld.array(gf.array((17 * np.arange(16)).reshape(4, 4).T)), senders=0)
    await mpc.gather(x, k, p)
    steps = [('sbox', lambda: sub_bytes(x)), ('inv_sbox', lambda: inv_sub_bytes(x)),
             ('aes128', lambda: encrypt(round_keys(k), p))]
    results, counts = [], {}
    for name, fn in steps:
        before = counters()
        r = await mpc.output(fn())
        counts[name] = delta(before, counters())
        results.append((name, r))
    for name, r in results:
        v = [int(b) for b in np.asarray(r.value).T.reshape(-1)] if name == 'aes128' else [int(b) for b in r.value]
        print(name, bytes(v).hex())
    if counts['sbox'] is not None:
        for name, cnt in counts.items():
            print('counts', name, json.dumps(cnt))
    await mpc.shutdown()

mpc.run(main())
