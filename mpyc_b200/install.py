"""install(): put the GPU engine behind an imported MPyC without touching MPyC's code.

mpyc/runtime.py looks the secret-sharing functions up as attributes of the `mpyc.thresha` module at
call time (runtime.py:478-485,565-572,647-656,963,982,1280,4057,4099,4219,4248); assigning the drop-in
functions of mpyc_b200.thresha over those attributes makes `_distribute`, `output`, `_reshare` and the
PRSS helpers run on the GPU while runtime.py, sectypes.py and the demos stay byte-for-byte unchanged.

Fields the engine does not cover (GF(2), GF(p^n) with n > 1, binary fields other than GF(2^8), primes
wider than 256 bits) are NOT intercepted: for those the wrapper hands the call to the reference's own
function, exactly as if install() had not been called (strict=True raises UnsupportedFieldError
instead).  The same holds per call: an argument outside the kernels' range on a covered field (e.g. a PRF bound
above 2^256) goes to the reference's function.  That hand-over is the only one: a covered call never runs on a CPU
restatement of the kernels, and without a CUDA device it raises.
"""
import functools

from mpyc_b200 import _cabi, thresha as engine
from mpyc_b200._cabi import UnsupportedFieldError
from mpyc_b200.field import context_of_field

_NAMES = ('random_split', 'recombine', 'np_random_split', 'np_recombine',
          'pseudorandom_share', 'pseudorandom_share_zero', 'np_pseudorandom_share', 'np_pseudorandom_share_0',
          '_recombination_vector', '_f_S_i')
_saved = {}


def _covered(field):
    try:
        context_of_field(field)
        return True
    except UnsupportedFieldError:
        return False


def _batch_size(name, args):
    """Number of elements a call works on (for the min_size routing of install())."""
    try:
        if name in ('random_split', 'np_random_split'):
            return len(args[0])
        if name in ('recombine', 'np_recombine'):
            return len(args[0][0][1])
        return int(args[-1])            # PRSS functions: (m, i, prfs, uci, n)
    except Exception:   # noqa: BLE001
        return None


def _wrap(name, ours, theirs, strict, min_size=0):
    @functools.wraps(theirs)
    def call(field, *args, **kwargs):
        if _covered(field):
            if min_size:
                n = _batch_size(name, args)
                if n is not None and n < min_size:
                    return theirs(field, *args, **kwargs)     # the reference's own code, as without install()
            if strict:
                return ours(field, *args, **kwargs)
            try:
                return ours(field, *args, **kwargs)
            except UnsupportedFieldError:
                # coverage is decided per CALL, not per field: a covered field with an argument outside the kernels'
                # range (a PRF bound above 2^256, more than 64 recombination points, a constant table beyond shared
                # memory ...) is computed by the reference's own function, exactly as without install() -- never
                # raise where the reference computes.  These functions are pure, so nothing is half-done.
                return theirs(field, *args, **kwargs)
        if strict:
            raise UnsupportedFieldError(f'mpyc_b200 does not cover field {getattr(field, "__name__", field)}')
        return theirs(field, *args, **kwargs)
    call.__mpyc_b200__ = True
    return call


def _install_finfields(finfields_module, min_size):
    """PrimeFieldArray._reciprocal/_pow/_sqrt/_is_sqr -> batched kernels for covered primes and arrays of
    at least `min_size` elements (below that the per-call overhead of a launch outweighs the gain)."""
    from mpyc_b200 import finfields as ours
    from mpyc_b200 import resident as _res
    cls = finfields_module.PrimeFieldArray
    orig = {name: cls.__dict__[name] for name in ('_reciprocal', '_pow', '_sqrt', '_is_sqr')}
    _saved_ff.update({'cls': cls, **orig})

    def use_gpu(klass, a):
        import numpy as np
        return np.size(a) >= min_size and klass.field.modulus % 2 == 1 and klass.field.modulus.bit_length() <= 256

    def _reciprocal(klass, a):
        return ours.reciprocal(klass, a) if use_gpu(klass, a) else orig['_reciprocal'].__func__(klass, a)

    def _pow(klass, a, b):
        theirs = lambda x, y: orig['_pow'].__func__(klass, x, y)   # noqa: E731
        return ours.power(klass, a, b, _fallback=theirs) if use_gpu(klass, a) else theirs(a, b)

    def _sqrt(klass, a, INV=False):
        theirs = lambda x, INV=False: orig['_sqrt'].__func__(klass, x, INV=INV)   # noqa: E731
        if type(a) is _res.ModValue:
            # np_random_bits: `field.array._sqrt(r2, INV=True)` on an opened value (runtime.py:4265) stays on the device
            if a.store is not None and a.exact and klass.field.modulus & 3 == 3:
                return a.sqrt(INV=INV)
            a = a._materialise()
        return ours.sqrt(klass, a, INV=INV, _fallback=theirs) if use_gpu(klass, a) else theirs(a, INV=INV)

    def _is_sqr(klass, a):
        return ours.is_sqr(klass, a) if use_gpu(klass, a) else orig['_is_sqr'].__func__(klass, a)

    cls._reciprocal = classmethod(_reciprocal)
    cls._pow = classmethod(_pow)
    cls._sqrt = classmethod(_sqrt)
    cls._is_sqr = classmethod(_is_sqr)


_saved_ff = {}
_saved_ops = {}
_saved_gmpy = {}


def _install_gmpy(thresha_module):
    """mpyc.gmpy.powmod_exp_list -> K12 (mpyc_b200.resident.powmod_exp_list).  runtime.py imports the module as
    `from mpyc import gmpy as gmpy2` and looks the function up at call time (runtime.py:24,1408,1422), so assigning over the
    module attribute reaches Runtime._np_pow_public_int_base_secret_integral_exponent -- 2 ** x, np_pow with a public int
    base and np_exp2 / np_exp -- with runtime.py unchanged.  Calls it does not cover go to the saved original."""
    import importlib
    from mpyc_b200 import resident
    package = thresha_module.__name__.rpartition('.')[0]
    try:
        gmpy = importlib.import_module(package + '.gmpy') if package else None
    except ImportError:
        gmpy = None
    if gmpy is None or not hasattr(gmpy, 'powmod_exp_list'):
        return
    theirs = gmpy.powmod_exp_list
    _saved_gmpy.update({'module': gmpy, 'powmod_exp_list': theirs})

    @functools.wraps(theirs)
    def powmod_exp_list(base, exp_lst, mod, /):
        r = resident.powmod_exp_list(base, exp_lst, mod)
        return theirs(base, exp_lst, mod) if r is resident._MISS else r
    powmod_exp_list.__mpyc_b200__ = True
    gmpy.powmod_exp_list = powmod_exp_list


# FiniteFieldArray method -> (hook in mpyc_b200.resident, fixed keyword arguments of the hook)
_HOOKS = {
    '__add__': ('binop', {'op': _cabi.OP_ADD}),
    '__radd__': ('binop', {'op': _cabi.OP_ADD}),
    '__sub__': ('binop', {'op': _cabi.OP_SUB}),
    '__rsub__': ('binop', {'op': _cabi.OP_SUB, 'reflected': True}),
    '__mul__': ('binop', {'op': _cabi.OP_MUL}),
    '__rmul__': ('binop', {'op': _cabi.OP_MUL}),
    '__neg__': ('negate', {}),
    '__matmul__': ('matmul', {}),
    '__rmatmul__': ('matmul', {'reflected': True}),
    '__lshift__': ('shift', {'right': False}),
    '__rshift__': ('shift', {'right': True}),
    '__ilshift__': ('shift', {'right': False}),
    '__irshift__': ('shift', {'right': True}),
    '__getitem__': ('getitem', {}),
    '__setitem__': ('setitem', {}),
    'transpose': ('transpose', {}),
    'swapaxes': ('swapaxes', {}),
    '__eq__': ('equals', {'negate': False}),
    '__ne__': ('equals', {'negate': True}),
    '__truediv__': ('divide', {}),
    '__rtruediv__': ('divide', {'reflected': True}),
    '__itruediv__': ('divide', {}),
    'reciprocal': ('reciprocal', {}),
    '__pow__': ('power', {}),
    '__ipow__': ('power', {}),
    'sqrt': ('sqrt', {}),
    'is_sqr': ('is_sqr', {}),
    'prod': ('prod_method', {}),
}
# in-place operators give self a new store: arrays sharing the old one keep their values
_INPLACE = ('__ilshift__', '__irshift__', '__itruediv__', '__ipow__')


def _install_operators(finfields_module, min_size):
    """FiniteFieldArray.__init__ and + - * neg @ (mpyc/finfields.py:717-725,1056-1146): limb-backed operands, and plain
    object arrays of at least `min_size` elements, are combined by the K1 / K1c kernels (mpyc_b200.resident), and so are
    np.sum / FiniteFieldArray.sum, np.cumsum, np.cumulative_sum (K7), np.outer (K1c) and np.prod / FiniteFieldArray.prod,
    np.cumprod, np.cumulative_prod, np.all, np.any (K13) of such arrays; np.matmul of field arrays runs on K1c as @ does, and
    with install(public_matmul=True) @ and np.matmul with an ndarray of a NumPy integer dtype on either side run on K14.
    Views, writes, axis permutations, joins, flips, rolls and broadcast + - * of limb-backed arrays run on K8 (mpyc_b200.layout), and
    np.linalg.det / solve / inv / matrix_power on K9 and K1c, and np.convolve on K10.  / (reflected and in place),
    reciprocal, ** and **= by an int, sqrt (Blum primes), is_sqr and np.where(cond, x, y) run on K11 and K1b, and ** and **=
    by an integer array of the same shape on K12; everything
    else -- scalars with small arrays, uncovered fields and keys -- runs the reference's own method unchanged."""
    from mpyc_b200 import resident
    import numpy as np
    resident.min_size = int(min_size)
    cls = finfields_module.FiniteFieldArray
    orig = {name: cls.__dict__[name] for name in ('__init__', *_HOOKS, '__array_function__', 'sum', '__array_ufunc__')}
    _saved_ops.update({'cls': cls, 'module': finfields_module, **orig})
    MISS = resident._MISS
    orig_hash = cls.__hash__          # assigning __eq__ on a class does not touch __hash__, kept explicit for clarity
    value_property = resident.make_value_property(finfields_module)
    slot_set = resident._slot.__set__

    def hooked(name, hook, fixed):
        # the hook is looked up in resident when called, so that rebinding it there takes effect
        inplace = name in _INPLACE

        def method(self, *args, **kwargs):
            r = getattr(resident, hook)(self, *args, **kwargs, **fixed)
            if r is MISS:
                return orig[name](self, *args, **kwargs)
            if inplace:
                slot_set(self, resident.raw_value(r))
                return self
            return r
        method.__name__ = name
        method.__doc__ = orig[name].__doc__
        return method

    def __init__(self, value, check=True, copy=False):
        lv = resident.as_limb_value(value)
        if lv is not None:
            slot_set(self, lv)         # canonical residues by construction: nothing to check, nothing to copy
            return
        if type(value) is resident.LimbValue or type(value) is resident.ModValue:
            value = value._ints        # already an object array (canonical residues)
        orig['__init__'](self, value, check=check, copy=copy)

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        # np.matmul(x, y) with two positional operands -- `int_ndarray @ field_array`, `object_ndarray @ field_array` and
        # np.matmul of field arrays, which NumPy hands to __array_ufunc__ (finfields.py:728-764) -- goes where @ goes:
        # K14 for a NumPy integer operand, K1c otherwise.  Other ufuncs, methods and keywords, and ndarray subclasses, run
        # the reference's method.
        if ufunc is np.matmul and method == '__call__' and not kwargs and len(inputs) == 2 and \
                all(isinstance(x, cls) or type(x) is np.ndarray for x in inputs):
            left = isinstance(inputs[0], cls)
            mine, other = (inputs[0], inputs[1]) if left else (inputs[1], inputs[0])
            r = resident.matmul(mine, other, reflected=not left, ufunc=True)
            if r is not MISS:
                return r
        # int_ndarray + field_array (np_to_bits' `c_bits + r_bits`) reaches np.add here: + does what the hook of __add__ does
        if ufunc is np.add and method == '__call__' and not kwargs and len(inputs) == 2 and \
                any(resident._int_matrix(x) for x in inputs) and any(isinstance(x, cls) for x in inputs) and \
                getattr(resident._ctx_of(type(self)), 'binary', False):
            left = isinstance(inputs[0], cls)
            mine, other = (inputs[0], inputs[1]) if left else (inputs[1], inputs[0])
            r = resident.binop(mine, other, op=_cabi.OP_ADD)
            if r is not MISS:
                return r
        return orig['__array_ufunc__'](self, ufunc, method, *inputs, **kwargs)

    def __array_function__(self, func, types, args, kwargs):
        r = resident.array_function(self, func, args, kwargs)
        return orig['__array_function__'](self, func, types, args, kwargs) if r is MISS else r

    def sum(self, *args, **kwargs):
        # ndarray.sum(axis=None, dtype=None, out=None, keepdims=False, initial=0, where=True)
        r = resident.reduction_function(self, np.sum, (self,) + args, kwargs) if len(args) <= 5 else MISS
        return orig['sum'](self, *args, **kwargs) if r is MISS else r

    for name, (hook, fixed) in _HOOKS.items():
        setattr(cls, name, hooked(name, hook, fixed))
    cls.__hash__ = orig_hash
    cls.__array_function__ = __array_function__
    cls.sum = sum
    cls.value = value_property
    cls.__init__ = __init__
    cls.__array_ufunc__ = __array_ufunc__


def install(thresha_module=None, strict=False, device=0, finfields_module=None, finfields_min_size=256,
            limb_wire=False, min_size=0, operators=False, operators_min_size=1024, resident=False, local_algebra=True,
            public_matmul=False):
    """Patch `mpyc.thresha` (or the module passed in); with finfields_module also the batched
    inverse/pow/sqrt/is_sqr of PrimeFieldArray.  limb_wire=True: shares travel between parties as limb
    buffers (mpyc_b200.wire; every party must run mpyc_b200).  min_size > 0: calls on fewer elements are left to
    the reference's own functions -- a GPU round trip costs ~35 us per call, which the reference beats below a few
    dozen 64-bit elements (DESIGN.md section 5); the default 0 sends every covered call to the GPU.
    operators=True: FiniteFieldArray's + - * neg @ (finfields.py:1056-1146) run on the K1 / K1c kernels for operands
    of at least operators_min_size elements (mpyc_b200.resident).  resident=True (implies operators and limb_wire):
    recombined / pseudorandom shares stay limb-backed in HBM between protocol steps; Python ints are created only
    where a value is actually looked at (input, output, raw-value arithmetic).  local_algebra (with resident): the raw-value
    arithmetic of Runtime.np_random_bits / np_trunc / np_sgn runs mod p on the device as well (resident.ModValue, K6 kernels).
    resident=True also routes mpyc.gmpy.powmod_exp_list (2 ** x, np_pow, np_exp2, np_exp of secure arrays) to K12.
    public_matmul (with operators or resident): @ and np.matmul of a field array with an ndarray of a NumPy integer dtype
    run on K14 (np_matmul with public weights, the `u @ np.arange(n)` of np_argmax / np_argmin / np_unit_vector), so the
    field operand stays limb-backed; without it those products settle the field operand and run the reference's code, as
    before K14, and the conversion counts of existing programs stay what they were.
    Returns the list of patched names."""
    if thresha_module is None:
        import mpyc.thresha as thresha_module
    if _saved:
        uninstall()
    if finfields_module is not None:
        _install_finfields(finfields_module, finfields_min_size)
    if operators or resident:
        if finfields_module is None:
            import mpyc.finfields as finfields_module
        _install_operators(finfields_module, operators_min_size)
    from mpyc_b200 import resident as res
    res.resident = bool(resident)
    res.local_algebra = bool(local_algebra and resident)
    res.public_matmul = bool(public_matmul)
    res.backend.device = device
    engine.device = device
    engine.limb_wire = bool(limb_wire or resident)
    for name in _NAMES:
        theirs = getattr(thresha_module, name)
        _saved[name] = (thresha_module, theirs)
        if name in ('_recombination_vector', '_f_S_i'):
            # keep the reference's functools.cache behaviour: results are cached per argument tuple
            ours = functools.cache(getattr(engine, name))
        else:
            ours = getattr(engine, name)
        routed = min_size if name not in ('_recombination_vector', '_f_S_i') else 0
        setattr(thresha_module, name, _wrap(name, ours, theirs, strict, routed))
    if resident:
        _install_gmpy(thresha_module)
    return list(_NAMES)


def uninstall():
    for name, (module, theirs) in list(_saved.items()):
        setattr(module, name, theirs)
    _saved.clear()
    engine.limb_wire = False
    from mpyc_b200 import resident as res
    res.resident = False
    res.public_matmul = False
    if _saved_ops:
        cls = _saved_ops.pop('cls')
        res.restore_value_slot(_saved_ops.pop('module'))
        for name, member in _saved_ops.items():
            setattr(cls, name, member)
        _saved_ops.clear()
    if _saved_gmpy:
        _saved_gmpy.pop('module').powmod_exp_list = _saved_gmpy.pop('powmod_exp_list')
    if _saved_ff:
        cls = _saved_ff.pop('cls')
        for name, member in _saved_ff.items():
            setattr(cls, name, member)
        _saved_ff.clear()
