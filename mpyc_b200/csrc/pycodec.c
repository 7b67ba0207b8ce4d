/* _pycodec: Python ints <-> fixed-width little-endian limb buffers at C speed.
 *
 * MPyC hands field arrays over as NumPy dtype=object arrays of Python ints (mpyc/finfields.py:703-725);
 * the kernels work on 8*L-byte little-endian elements.  Converting through int.to_bytes / int.from_bytes
 * in Python costs 0.2-0.4 us per element and dominated the drop-in path; these two functions do it in
 * ~30 ns per element with the CPython long API.
 *
 *   pack(seq, nbytes, modulus) -> bytearray of len(seq)*nbytes     (values reduced mod modulus if needed)
 *   unpack(buffer, nbytes)     -> list of ints
 *   unpack_into(buffer, nbytes, address) -> None; ints written into a NumPy object array's slots
 */
#define PY_SSIZE_T_CLEAN
#include <Python.h>
#include <stdint.h>
#include <string.h>

/* CPython 3.12 (30-bit digits, lv_tag = ndigits << 3 | sign): read / write the digit array directly.
 * Every other interpreter version goes through the portable _PyLong_{As,From}ByteArray calls below. */
#if PY_VERSION_HEX >= 0x030C0000 && PY_VERSION_HEX < 0x030D0000 && PyLong_SHIFT == 30 && defined(_PyLong_SIGN_MASK)
#define MPYC_FAST_LONG 1
#else
#define MPYC_FAST_LONG 0
#endif
#define MAX_LIMBS 5   /* fast paths cover elements of up to 32 bytes (+ one spill limb while shifting) */

#if MPYC_FAST_LONG
/* non-negative exact int of at most nlimbs*64 bits -> limbs; returns 0 if v does not qualify */
static int fast_digits_to_limbs(PyObject* v, uint64_t* limbs, int nlimbs) {
    if (!PyLong_CheckExact(v)) return 0;
    const PyLongObject* lv = (const PyLongObject*)v;
    const uintptr_t tag = lv->long_value.lv_tag;
    if ((tag & _PyLong_SIGN_MASK) == 2) return 0;                 /* negative */
    const Py_ssize_t nd = (Py_ssize_t)(tag >> _PyLong_NON_SIZE_BITS);
    if (nd * 30 > (Py_ssize_t)nlimbs * 64 + 29) return 0;
    for (int i = 0; i <= nlimbs; i++) limbs[i] = 0;
    for (Py_ssize_t d = 0; d < nd; d++) {
        const uint64_t dig = lv->long_value.ob_digit[d];
        const unsigned pos = (unsigned)(30 * d), w = pos >> 6, off = pos & 63;
        limbs[w] |= dig << off;
        if (off > 34) limbs[w + 1] |= dig >> (64 - off);
    }
    return limbs[nlimbs] == 0;                                    /* spill limb used: wider than the element */
}

static PyObject* fast_limbs_to_long(const uint64_t* limbs, int nlimbs) {
    int top = nlimbs - 1;
    while (top > 0 && limbs[top] == 0) top--;
    if (top == 0) return PyLong_FromUnsignedLongLong(limbs[0]);   /* also keeps the small-int singletons */
    const unsigned bits = 64u * (unsigned)top + (64u - (unsigned)__builtin_clzll(limbs[top]));
    const Py_ssize_t nd = (bits + 29) / 30;
    PyLongObject* r = _PyLong_New(nd);                            /* positive, nd digits */
    if (!r) return NULL;
    for (Py_ssize_t d = 0; d < nd; d++) {
        const unsigned pos = (unsigned)(30 * d), w = pos >> 6, off = pos & 63;
        uint64_t x = limbs[w] >> off;
        if (off > 34 && (int)w + 1 < nlimbs) x |= limbs[w + 1] << (64 - off);
        r->long_value.ob_digit[d] = (digit)(x & 0x3FFFFFFFu);
    }
    return (PyObject*)r;
}
#endif

static int as_bytes(PyObject* v, unsigned char* dst, size_t n) {
#if PY_VERSION_HEX >= 0x030D0000
    return _PyLong_AsByteArray((PyLongObject*)v, dst, n, 1, 0, 1);
#else
    return _PyLong_AsByteArray((PyLongObject*)v, dst, n, 1, 0);
#endif
}

static PyObject* pack(PyObject* self, PyObject* args) {
    PyObject *seq, *modulus;
    Py_ssize_t nbytes;
    if (!PyArg_ParseTuple(args, "OnO", &seq, &nbytes, &modulus)) return NULL;
    if (!PyLong_Check(modulus) || nbytes < 1) {
        PyErr_SetString(PyExc_TypeError, "pack(seq, nbytes, modulus:int)");
        return NULL;
    }
    PyObject* fast = PySequence_Fast(seq, "pack: expected a sequence of ints");
    if (!fast) return NULL;
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(fast);
    PyObject* out = PyByteArray_FromStringAndSize(NULL, n * nbytes);
    if (!out) {
        Py_DECREF(fast);
        return NULL;
    }
    unsigned char* dst = (unsigned char*)PyByteArray_AS_STRING(out);
    const size_t kbits = _PyLong_NumBits(modulus);
    PyObject** items = PySequence_Fast_ITEMS(fast);
#if MPYC_FAST_LONG
    uint64_t mod[MAX_LIMBS + 1];
    const int nl = (nbytes % 8 == 0 && nbytes <= 32) ? (int)(nbytes / 8) : 0;
    const int fast_ok = nl > 0 && fast_digits_to_limbs(modulus, mod, nl);
#endif
    for (Py_ssize_t i = 0; i < n; i++) {
        PyObject* v = items[i];
        PyObject* owned = NULL;
#if MPYC_FAST_LONG
        if (fast_ok) {
            uint64_t limbs[MAX_LIMBS + 1];
            if (fast_digits_to_limbs(v, limbs, nl)) {
                int lt = 0;                                        /* limbs < modulus ? */
                for (int w = nl - 1; w >= 0; w--)
                    if (limbs[w] != mod[w]) {
                        lt = limbs[w] < mod[w];
                        break;
                    }
                if (lt) {
                    memcpy(dst + i * nbytes, limbs, (size_t)nbytes);   /* little-endian host */
                    continue;
                }
            }
        }
#endif
        if (!PyLong_Check(v)) {            /* field elements / numpy ints / polynomials: go through int() */
            owned = PyNumber_Long(v);
            if (!owned) goto fail;
            v = owned;
        }
        int reduce = 0;
        if (_PyLong_Sign(v) < 0) reduce = 1;
        else {
            size_t bits = _PyLong_NumBits(v);
            if (bits > kbits) reduce = 1;
            else if (bits == kbits) {
                int lt = PyObject_RichCompareBool(v, modulus, Py_LT);
                if (lt < 0) { Py_XDECREF(owned); goto fail; }
                reduce = !lt;
            }
        }
        if (reduce) {
            PyObject* r = PyNumber_Remainder(v, modulus);
            Py_XDECREF(owned);
            if (!r) goto fail;
            owned = r;
            v = r;
        }
        int rc = as_bytes(v, dst + i * nbytes, (size_t)nbytes);
        Py_XDECREF(owned);
        if (rc < 0) goto fail;
    }
    Py_DECREF(fast);
    return out;
fail:
    Py_DECREF(fast);
    Py_DECREF(out);
    return NULL;
}

static PyObject* decode_one(const unsigned char* src, Py_ssize_t nbytes) {
#if MPYC_FAST_LONG
    if (nbytes % 8 == 0 && nbytes <= 32) {
        uint64_t limbs[MAX_LIMBS];
        memcpy(limbs, src, (size_t)nbytes);
        return fast_limbs_to_long(limbs, (int)(nbytes / 8));
    }
#endif
    return _PyLong_FromByteArray(src, (size_t)nbytes, 1, 0);
}

/* unpack_into(buffer, nbytes, address): the n decoded ints are stored straight into the n PyObject* slots at
 * `address` -- the data area of a NumPy dtype=object array owned by the caller (np.empty(n, object).ctypes.data),
 * so no intermediate list and no second pass.  The previous slot contents (None / NULL) are released. */
static PyObject* unpack_into(PyObject* self, PyObject* args) {
    Py_buffer buf;
    Py_ssize_t nbytes;
    unsigned long long addr;
    if (!PyArg_ParseTuple(args, "y*nK", &buf, &nbytes, &addr)) return NULL;
    if (nbytes < 1 || buf.len % nbytes || (!addr && buf.len)) {
        PyBuffer_Release(&buf);
        PyErr_SetString(PyExc_ValueError, "unpack_into: bad buffer length or destination");
        return NULL;
    }
    const Py_ssize_t n = buf.len / nbytes;
    PyObject** slots = (PyObject**)(uintptr_t)addr;
    const unsigned char* src = (const unsigned char*)buf.buf;
    for (Py_ssize_t i = 0; i < n; i++) {
        PyObject* v = decode_one(src + i * nbytes, nbytes);
        if (!v) {
            PyBuffer_Release(&buf);
            return NULL;
        }
        PyObject* old = slots[i];
        slots[i] = v;
        Py_XDECREF(old);
    }
    PyBuffer_Release(&buf);
    Py_RETURN_NONE;
}

static PyObject* unpack(PyObject* self, PyObject* args) {
    Py_buffer buf;
    Py_ssize_t nbytes;
    if (!PyArg_ParseTuple(args, "y*n", &buf, &nbytes)) return NULL;
    if (nbytes < 1 || buf.len % nbytes) {
        PyBuffer_Release(&buf);
        PyErr_SetString(PyExc_ValueError, "unpack: buffer length is not a multiple of nbytes");
        return NULL;
    }
    const Py_ssize_t n = buf.len / nbytes;
    PyObject* out = PyList_New(n);
    if (!out) {
        PyBuffer_Release(&buf);
        return NULL;
    }
    const unsigned char* src = (const unsigned char*)buf.buf;
    for (Py_ssize_t i = 0; i < n; i++) {
        PyObject* v = decode_one(src + i * nbytes, nbytes);
        if (!v) {
            Py_DECREF(out);
            PyBuffer_Release(&buf);
            return NULL;
        }
        PyList_SET_ITEM(out, i, v);
    }
    PyBuffer_Release(&buf);
    return out;
}

/* pack_exponents(seq, max_limbs) -> (limbs, signs, bits, el) or None: the magnitudes of a sequence of Python ints (not
 * bools) as el = max(1, ceil(bits / 64)) little-endian 64-bit limbs each, bits the largest bit length; signs a bytearray
 * with 1 for each negative entry, or None when there is none.  None when an entry is not an int or bits > 64 * max_limbs:
 * the exponents of K12 (mpyc_b200.codec.exponents_to_limbs) are not reduced, so nothing wider has a place to go. */
static PyObject* pack_exponents(PyObject* self, PyObject* args) {
    PyObject* seq;
    int max_limbs;
    if (!PyArg_ParseTuple(args, "Oi", &seq, &max_limbs)) return NULL;
    if (max_limbs < 1 || max_limbs > MAX_LIMBS - 1) {
        PyErr_SetString(PyExc_ValueError, "pack_exponents: max_limbs must be 1..4");
        return NULL;
    }
    PyObject* fast = PySequence_Fast(seq, "pack_exponents: expected a sequence of ints");
    if (!fast) return NULL;
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(fast);
    PyObject** items = PySequence_Fast_ITEMS(fast);
    size_t bits = 0;
    int negative = 0;
    for (Py_ssize_t i = 0; i < n; i++) {
        PyObject* v = items[i];
        if (!PyLong_Check(v) || PyBool_Check(v)) {
            Py_DECREF(fast);
            Py_RETURN_NONE;
        }
        const size_t b = _PyLong_NumBits(v);          /* of |v| */
        if (b == (size_t)-1 && PyErr_Occurred()) goto fail0;
        if (b > bits) bits = b;
        if (_PyLong_Sign(v) < 0) negative = 1;
    }
    if (bits > (size_t)64 * max_limbs) {
        Py_DECREF(fast);
        Py_RETURN_NONE;
    }
    const Py_ssize_t el = bits ? (Py_ssize_t)((bits + 63) / 64) : 1;
    PyObject* limbs = PyByteArray_FromStringAndSize(NULL, n * el * 8);
    PyObject* signs = negative ? PyByteArray_FromStringAndSize(NULL, n) : (Py_INCREF(Py_None), Py_None);
    if (!limbs || !signs) {
        Py_XDECREF(limbs);
        Py_XDECREF(signs);
        goto fail0;
    }
    unsigned char* dst = (unsigned char*)PyByteArray_AS_STRING(limbs);
    unsigned char* sg = negative ? (unsigned char*)PyByteArray_AS_STRING(signs) : NULL;
    for (Py_ssize_t i = 0; i < n; i++) {
        PyObject* v = items[i];
        const int neg = _PyLong_Sign(v) < 0;
        if (sg) sg[i] = (unsigned char)neg;
        PyObject* owned = neg ? PyNumber_Negative(v) : NULL;
        if (neg && !owned) goto fail;
        const int rc = as_bytes(owned ? owned : v, dst + i * el * 8, (size_t)(el * 8));
        Py_XDECREF(owned);
        if (rc < 0) goto fail;
    }
    Py_DECREF(fast);
    PyObject* r = Py_BuildValue("(NNnn)", limbs, signs, (Py_ssize_t)bits, el);
    return r;
fail:
    Py_DECREF(limbs);
    Py_DECREF(signs);
fail0:
    Py_DECREF(fast);
    return NULL;
}

static PyMethodDef methods[] = {
    {"pack", pack, METH_VARARGS, "pack(seq, nbytes, modulus) -> bytearray (little-endian, reduced mod modulus)"},
    {"pack_exponents", pack_exponents, METH_VARARGS, "pack_exponents(seq, max_limbs) -> (limbs, signs or None, bits, el) or None"},
    {"unpack", unpack, METH_VARARGS, "unpack(buffer, nbytes) -> list of ints"},
    {"unpack_into", unpack_into, METH_VARARGS, "unpack_into(buffer, nbytes, address of n object slots)"},
    {NULL, NULL, 0, NULL}};

static struct PyModuleDef moduledef = {PyModuleDef_HEAD_INIT, "_pycodec", "int <-> limb buffer codec", -1, methods};

PyMODINIT_FUNC PyInit__pycodec(void) { return PyModule_Create(&moduledef); }
