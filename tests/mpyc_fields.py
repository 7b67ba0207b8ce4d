"""The prime fields MPyC's secure types create with the default options (bit_length = 32, sec_param = 30).

sectypes._pfield sizes a field as finfields.find_prime_root(l + f + sec_param + 2, n=2); the two 1024-th root fields are
what find_prime_root(bits, n=1024) gives (transforms that need a large power-of-two root of unity).  The values are kept
as literals so that the GPU tests never need the reference; tests/test_mpyc_fields_host.py pins each one to the
reference's find_prime_root where the reference is present."""
from collections import namedtuple

MpycField = namedtuple('MpycField', 'name bits n p kind limbs')

# kind: 0 generic (Montgomery), 1 pseudo-Mersenne 2^(64 L) - c, 2 pseudo-Mersenne 2^k - c shifted inside L limbs
FIELDS = [
    MpycField('secint16', 48, 2, 2**48 - 65, 0, 1),
    MpycField('secfxp', 80, 2, 2**80 - 65, 2, 2),
    MpycField('secint64', 96, 2, 2**96 - 17, 2, 2),
    MpycField('secint128', 160, 2, 2**160 - 57, 2, 3),
    MpycField('secint160', 192, 2, 2**192 - 237, 1, 3),
    MpycField('secint168', 200, 2, 2**200 - 117, 2, 4),
    MpycField('root96', 96, 1024, 0x80000000000000000001dc63, 0, 2),
    MpycField('root256', 256, 1024, 0x800000000000000000000000000000000000000000000000000000000009272f, 0, 4),
]
BY_NAME = {f.name: f for f in FIELDS}
PRIMES = [f.p for f in FIELDS]


def field_id(f):
    return f.name
