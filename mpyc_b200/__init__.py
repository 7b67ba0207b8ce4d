"""mpyc_b200 -- H100 (sm_90a) batched finite-field / Shamir secret-sharing engine.

A from-scratch CUDA implementation of the data-parallel hot path of lschoe/mpyc
(mpyc/thresha.py and the array half of mpyc/finfields.py), reached from Python through a thin
ctypes C ABI (include/mpyc_b200.h):

    mpyc_b200.thresha     drop-in np_random_split / np_recombine / pseudorandom_share ... (host data)
    mpyc_b200.device      DeviceArray / DeviceMatrix: limb tensors resident in HBM + shamir_split/recombine
    mpyc_b200.field       FieldContext: one handle per modulus (reduction family, cached tables)
    mpyc_b200.install     install()/uninstall(): swap the engine in behind an imported `mpyc`
    mpyc_b200.wire        limb wire format: ShareRow objects that pickle as fixed-width bytes, never Python ints
    mpyc_b200.sharding    element-axis sharding over the GPUs of one box (torch.distributed)
    mpyc_b200.exchange    co-located resharing: NCCL send/recv of limb rows, or K2 storing into the peer GPU

There is no CPU fallback: importing the package needs libmpyc_b200.so (built in-tree by
mpyc_b200._build), and every compute call needs a CUDA device.
"""
from mpyc_b200 import _cabi
from mpyc_b200._cabi import UnsupportedFieldError
from mpyc_b200.field import FieldContext, context_for, context_of_field

__version__ = '0.1.0'
__all__ = ['FieldContext', 'context_for', 'context_of_field', 'UnsupportedFieldError', 'launch_count']


def launch_count():
    """Number of kernels the library has launched in this process."""
    return int(_cabi.lib.mpyc_b200_launch_count())
