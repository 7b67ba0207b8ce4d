"""ctypes binding of libmpyc_b200.so (the C ABI declared in include/mpyc_b200.h).

This is the whole Python <-> CUDA boundary: plain pointers and sizes, status codes mapped to the
exceptions the reference raises in the same situations (ZeroDivisionError from gmpy2.invert,
ValueError / TypeError for bad arguments).  There is no CPU fallback: if the shared library cannot
be loaded the import of this module raises.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_int, c_int64, c_size_t, c_uint8, c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libmpyc_b200.so')
_VARIANT = os.environ.get('MPYC_B200_LIB')   # kernel-tuning builds (mpyc_b200/_build.py -D... -o<name>)

OK, EINVAL, EUNSUPPORTED, EZERODIV, ECUDA, ENOMEM = 0, -1, -2, -3, -4, -5
KIND_GENERIC, KIND_PM_ALIGNED, KIND_PM_SHIFT, KIND_GF256 = 0, 1, 2, 3
OP_ADD, OP_SUB, OP_MUL = 0, 1, 2
MAX_LIMBS = 4
MAX_POINTS = 64


class UnsupportedFieldError(TypeError):
    """The modulus / shape is outside what the sm_90a kernels cover (MPYC_B200_EUNSUPPORTED)."""


def _load():
    # (re)build in-tree when the sources changed or the library is missing; a no-op otherwise
    import importlib.util
    spec = importlib.util.spec_from_file_location('_mpyc_b200_build', os.path.join(_HERE, '_build.py'))
    builder = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(builder)
    builder.build()   # returns at once when the library's digest stamp matches the sources; a library whose stamp does
    #                   not match is NEVER loaded (no stale-binary fallback): without nvcc this raises
    return ctypes.CDLL(os.path.join(_HERE, _VARIANT) if _VARIANT else LIB_PATH)


lib = _load()

VIEW_RANK = 6


class View(ctypes.Structure):
    """mpyc_b200_view: a strided view of an element buffer (include/mpyc_b200.h)."""
    _fields_ = [('offset', c_int64), ('rank', ctypes.c_int32), ('index_axis', ctypes.c_int32),
                ('extent', c_int64 * VIEW_RANK), ('stride', c_int64 * VIEW_RANK), ('index', POINTER(c_int64))]


_field_p = c_void_p
_view_p = POINTER(View)
_SIGNATURES = {
    'mpyc_b200_version': (c_int, []),
    'mpyc_b200_strerror': (c_char_p, [c_int]),
    'mpyc_b200_last_error': (c_char_p, []),
    'mpyc_b200_launch_count': (c_uint64, []),
    'mpyc_b200_device_count': (c_int, [POINTER(c_int)]),
    'mpyc_b200_field_create': (c_int, [POINTER(c_uint64), c_int, POINTER(_field_p)]),
    'mpyc_b200_field_create_gf256': (c_int, [c_uint32, POINTER(_field_p)]),
    'mpyc_b200_field_destroy': (None, [_field_p]),
    'mpyc_b200_field_info': (c_int, [_field_p, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_size_t)]),
    'mpyc_b200_ff_binop': (c_int, [_field_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_binop_scalar': (c_int, [_field_p, c_int, c_void_p, POINTER(c_uint64), c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_neg': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_pow': (c_int, [_field_p, c_void_p, POINTER(c_uint64), c_int, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_inv': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_sqrt': (c_int, [_field_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_is_sqr': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_matmul': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_size_t, c_void_p]),
    'mpyc_b200_ff_fma': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_axpb': (c_int, [_field_p, c_void_p, POINTER(c_uint64), POINTER(c_uint64), c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_low_bits': (c_int, [_field_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_nonzero': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_bits_compose': (c_int, [_field_p, c_void_p, c_size_t, c_int, c_int, c_void_p, c_void_p]),
    'mpyc_b200_ff_bits_decompose': (c_int, [_field_p, c_void_p, c_size_t, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_transpose': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_cumsum_rows': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_sum_axis': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_size_t, POINTER(c_uint64), c_void_p, c_void_p]),
    'mpyc_b200_ff_cumsum_axis': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_size_t, c_int, c_void_p, c_void_p]),
    'mpyc_b200_copy_view': (c_int, [c_size_t, c_void_p, c_size_t, _view_p, c_void_p, c_size_t, _view_p, c_void_p]),
    'mpyc_b200_ff_binop_view': (c_int, [_field_p, c_int, c_void_p, c_size_t, _view_p, c_void_p, c_size_t, _view_p, c_void_p,
                                        c_void_p]),
    'mpyc_b200_ff_det': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_solve': (c_int, [_field_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_convolve': (c_int, [_field_p, c_void_p, c_size_t, c_void_p, c_size_t, c_size_t, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_div': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_ff_select': (c_int, [_field_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                    c_void_p]),
    'mpyc_b200_ff_pow_exp': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_ff_prod_axis': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_size_t, POINTER(c_uint64), c_void_p, c_void_p]),
    'mpyc_b200_ff_cumprod_axis': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_size_t, c_int, c_void_p, c_void_p]),
    'mpyc_b200_ff_all_any_axis': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_size_t, c_int, c_void_p, c_void_p]),
    'mpyc_b200_ff_matmul_int': (c_int, [_field_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_size_t, c_size_t,
                                        c_void_p]),
    'mpyc_b200_gf_bits_compose': (c_int, [_field_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_gf_binop_view': (c_int, [_field_p, c_int, c_void_p, c_size_t, _view_p, c_void_p, c_size_t, _view_p, c_void_p,
                                        c_void_p]),
    'mpyc_b200_gf_matmul_batched': (c_int, [_field_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_size_t,
                                            c_size_t, c_size_t, c_void_p]),
    'mpyc_b200_ff_binop_rows': (c_int, [_field_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_void_p]),
    'mpyc_b200_ff_conv2d': (c_int, [_field_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p]),
    'mpyc_b200_shamir_split': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_size_t,
                                       c_int, c_int, c_void_p]),
    'mpyc_b200_shamir_split_generate': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_size_t, c_int, c_int,
                                                POINTER(c_uint8), c_uint64, c_void_p]),
    'mpyc_b200_shamir_split_generate_rows': (c_int, [_field_p, c_void_p, POINTER(c_void_p), c_size_t, c_int, c_int,
                                                     POINTER(c_uint8), c_uint64, c_void_p]),
    'mpyc_b200_recombination_vector': (c_int, [_field_p, POINTER(c_int64), c_int, POINTER(c_int64), c_int,
                                               POINTER(c_uint64)]),
    'mpyc_b200_shamir_recombine': (c_int, [_field_p, POINTER(c_void_p), POINTER(c_int64), c_int, POINTER(c_int64),
                                           c_int, c_void_p, c_size_t, c_size_t, c_void_p]),
    'mpyc_b200_prss_combine': (c_int, [_field_p, c_void_p, c_size_t, c_int, c_int, c_int, c_int, POINTER(c_uint64),
                                       POINTER(c_uint64), c_void_p, c_size_t, c_void_p]),
    'mpyc_b200_prss_small_form': (c_int, [_field_p, c_int, c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_int64),
                                          POINTER(c_uint64)]),
    'mpyc_b200_prss_host': (c_int, [_field_p, c_char_p, c_int, c_char_p, c_size_t, c_int, c_int, c_int, c_int,
                                    POINTER(c_uint64), POINTER(c_uint64), c_void_p, c_size_t, c_int, c_int]),
    'mpyc_b200_prss_host_bound': (c_int, [_field_p, c_char_p, c_int, c_char_p, c_size_t, c_int, c_int, c_int,
                                          POINTER(c_uint64), c_int, POINTER(c_uint64), POINTER(c_uint64), c_void_p, c_size_t,
                                          c_int, c_int]),
    'mpyc_b200_prf_reduce': (c_int, [_field_p, c_void_p, c_size_t, c_int, c_size_t, c_int, POINTER(c_uint64), c_int, c_void_p,
                                     c_size_t, POINTER(c_int), c_void_p]),
    'mpyc_b200_enable_peer_access': (c_int, [c_int, c_int]),
    'mpyc_b200_peer_alloc': (c_int, [c_size_t, POINTER(c_void_p), POINTER(c_uint8)]),
    'mpyc_b200_peer_open': (c_int, [POINTER(c_uint8), POINTER(c_void_p)]),
    'mpyc_b200_peer_close': (c_int, [c_void_p]),
    'mpyc_b200_peer_free': (c_int, [c_void_p]),
    'mpyc_b200_shake128': (c_int, [c_char_p, c_size_t, c_void_p, c_size_t]),
    'mpyc_b200_shake128_multi': (c_int, [c_char_p, c_int, c_char_p, c_size_t, c_int, c_void_p, c_size_t, c_size_t, POINTER(c_int)]),
    'mpyc_b200_fill_random': (c_int, [_field_p, c_void_p, c_size_t, c_uint64, c_uint64, c_void_p]),
    'mpyc_b200_count_mismatch': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    'mpyc_b200_shamir_split_host': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_size_t,
                                            c_int, c_int, c_int]),
    'mpyc_b200_shamir_split_generate_host': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_size_t, c_int, c_int,
                                                     POINTER(c_uint8), c_uint64, c_int]),
    'mpyc_b200_shamir_recombine_host': (c_int, [_field_p, POINTER(c_void_p), POINTER(c_int64), c_int,
                                                POINTER(c_int64), c_int, c_void_p, c_size_t, c_size_t, c_int]),
    'mpyc_b200_ff_binop_host': (c_int, [_field_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_int]),
    'mpyc_b200_shamir_reshare_step_host': (c_int, [_field_p, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_size_t, c_int, c_int,
                                                   POINTER(c_void_p), POINTER(c_int64), c_int, POINTER(c_int64), c_int, c_void_p,
                                                   c_size_t, c_size_t, c_int]),
}
for _name, (_res, _args) in _SIGNATURES.items():
    _fn = getattr(lib, _name)   # AttributeError here = library does not export the declared ABI
    _fn.restype = _res
    _fn.argtypes = _args

EXPORTED = tuple(_SIGNATURES)


def check(status):
    """Map a C-ABI status to the exception the reference raises in the same situation."""
    if status == OK:
        return
    detail = (lib.mpyc_b200_last_error() or b'').decode(errors='replace')
    text = f'{lib.mpyc_b200_strerror(status).decode()}: {detail}'
    if status == EZERODIV:
        raise ZeroDivisionError(detail or 'inverse of zero')
    if status == EINVAL:
        raise ValueError(text)
    if status == EUNSUPPORTED:
        raise UnsupportedFieldError(text)
    if status == ENOMEM:
        raise MemoryError(text)
    raise RuntimeError(text)


def u64_array(values):
    return (c_uint64 * len(values))(*values)


def i64_array(values):
    return (c_int64 * len(values))(*values)


def ptr_array(values):
    return (c_void_p * len(values))(*values)


def int_to_limbs(x, nlimbs):
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(nlimbs)]


def limbs_to_int(limbs):
    v = 0
    for i, w in enumerate(limbs):
        v |= int(w) << (64 * i)
    return v
