/* mpyc_b200 -- C ABI of the H100 (sm_90a) batched finite-field / Shamir engine.
 *
 * The reference (lschoe/mpyc, pure Python) has no FFI; its "plugin boundary" for this path is a
 * set of Python callables that mpyc/runtime.py looks up at call time (SURVEY.md 8b).  Each entry
 * point below is what a ctypes binding for one of those callables binds to; the reference
 * interface it replaces is cited as file:line relative to the reference checkout.
 *
 * Conventions
 *   - every function returns an int status: MPYC_B200_OK (0) or a negative MPYC_B200_E* code;
 *     nothing throws across the ABI.  mpyc_b200_strerror() names a code; the CUDA error text of
 *     the calling thread's last MPYC_B200_ECUDA is available via mpyc_b200_last_error().
 *   - field elements are canonical residues in [0, p) stored as L little-endian 64-bit limbs,
 *     L = ceil(bits(p)/64) in {1,2,3,4}, elements contiguous ("element-major").  A row of n
 *     elements is n*L uint64.  Montgomery form never crosses the ABI.
 *   - matrices (shares, coefficients) are given as a base pointer plus a row stride counted in
 *     ELEMENTS (row i starts at base + i*stride*L uint64); stride >= n.
 *   - pointers named d_* are device pointers owned by the caller; h_* are host pointers (pageable
 *     or pinned) owned by the caller.  The library owns only the mpyc_b200_field handle and the
 *     small per-field tables it caches (Vandermonde / Lagrange), freed by mpyc_b200_field_destroy.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  Device
 *     entry points enqueue work and return without synchronising unless stated otherwise.
 *   - a field handle is immutable after creation apart from its internally locked table cache;
 *     calls are safe from one host thread per stream.
 *   - there is no CPU fallback: without a CUDA device every compute entry point fails with
 *     MPYC_B200_ECUDA.
 */
#ifndef MPYC_B200_H
#define MPYC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPYC_B200_OK            0
#define MPYC_B200_EINVAL       -1   /* bad argument (shim raises ValueError)                     */
#define MPYC_B200_EUNSUPPORTED -2   /* modulus / shape outside what the kernels cover (TypeError)*/
#define MPYC_B200_EZERODIV     -3   /* inverse of zero requested (shim raises ZeroDivisionError) */
#define MPYC_B200_ECUDA        -4   /* CUDA runtime error (RuntimeError)                         */
#define MPYC_B200_ENOMEM       -5   /* host or device allocation failed (MemoryError)            */

#define MPYC_B200_MAX_LIMBS     4
#define MPYC_B200_MAX_POINTS    64  /* max shares per recombination call                         */

/* field kinds reported by mpyc_b200_field_info */
#define MPYC_B200_KIND_GENERIC     0   /* odd prime: Barrett / Montgomery (guard limb) reductions */
#define MPYC_B200_KIND_PM_ALIGNED  1   /* p = 2^(64L) - c                                        */
#define MPYC_B200_KIND_PM_SHIFT    2   /* p = 2^k - c, k % 64 != 0                               */
#define MPYC_B200_KIND_GF256       3   /* GF(2^8) = GF(2)[X]/(modulus), one byte per element     */

/* elementwise binary ops for mpyc_b200_ff_binop* */
#define MPYC_B200_OP_ADD 0
#define MPYC_B200_OP_SUB 1
#define MPYC_B200_OP_MUL 2

typedef struct mpyc_b200_field mpyc_b200_field;

int         mpyc_b200_version(void);
const char* mpyc_b200_strerror(int status);
const char* mpyc_b200_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py's gpu_launches) */
uint64_t    mpyc_b200_launch_count(void);
int         mpyc_b200_device_count(int* count);

/* ---- field context ------------------------------------------------------------------------
 * Replaces finfields.GF(p) / pGF (mpyc/finfields.py:23-42,347-363) as the carrier of the modulus.
 * modulus: nlimbs little-endian limbs of an odd prime p >= 3 (primality is the caller's business,
 * as pGF checks it with gmpy2.is_prime before this is reached). */
int  mpyc_b200_field_create(const uint64_t* modulus, int nlimbs, mpyc_b200_field** out);
/* GF(2^8) with the given degree-8 modulus polynomial (e.g. 283 = x^8+x^4+x^3+x+1, the AES field
 * of demos/np_aes.py); replaces finfields.GF(gfpx.GFpX(2)(283)) (mpyc/finfields.py:1542-1563). */
int  mpyc_b200_field_create_gf256(uint32_t modulus_poly, mpyc_b200_field** out);
void mpyc_b200_field_destroy(mpyc_b200_field* f);
int  mpyc_b200_field_info(const mpyc_b200_field* f, int* nlimbs, int* kind, int* bits,
                          size_t* elem_bytes);

/* ---- elementwise field arithmetic on device-resident arrays ------------------------------
 * FiniteFieldArray.__add__/__sub__/__mul__ (mpyc/finfields.py:1056-1124): out[h] = a[h] op b[h]. */
int mpyc_b200_ff_binop(const mpyc_b200_field* f, int op, const void* d_a, const void* d_b,
                       void* d_out, size_t n, void* stream);
/* same with a broadcast scalar b (host limbs, canonical) -- a op scalar (finfields.py:1045-1054) */
int mpyc_b200_ff_binop_scalar(const mpyc_b200_field* f, int op, const void* d_a,
                              const uint64_t* h_scalar, void* d_out, size_t n, void* stream);
/* __neg__ (mpyc/finfields.py:1189-1192) */
int mpyc_b200_ff_neg(const mpyc_b200_field* f, const void* d_a, void* d_out, size_t n, void* stream);
/* PrimeFieldArray._pow with one public exponent e >= 0 (mpyc/finfields.py:1408-1414):
 * out[h] = a[h]^e.  exponent: exp_nlimbs little-endian limbs. */
int mpyc_b200_ff_pow(const mpyc_b200_field* f, const void* d_a, const uint64_t* h_exponent,
                     int exp_nlimbs, void* d_out, size_t n, void* stream);
/* PrimeFieldArray._reciprocal (mpyc/finfields.py:1416-1422): out[h] = a[h]^-1.  SYNCHRONISES the
 * stream; returns MPYC_B200_EZERODIV if any a[h] == 0 (gmpy2.invert raises, mpyc/gmpy.py:192-213);
 * d_out is then unspecified. */
int mpyc_b200_ff_inv(const mpyc_b200_field* f, const void* d_a, void* d_out, size_t n, void* stream);
/* PrimeFieldArray._sqrt for Blum primes p % 4 == 3 (mpyc/finfields.py:1424-1438):
 * inverse == 0: a^((p+1)/4); inverse != 0: a^((3p-5)/4) and EZERODIV if any a[h] == 0
 * (synchronises in that case).  EUNSUPPORTED for p % 4 == 1. */
int mpyc_b200_ff_sqrt(const mpyc_b200_field* f, const void* d_a, int inverse, void* d_out, size_t n,
                      void* stream);
/* PrimeFieldArray._is_sqr (mpyc/finfields.py:1463-1470): d_out_u8[h] = legendre(a[h], p) != -1 */
int mpyc_b200_ff_is_sqr(const mpyc_b200_field* f, const void* d_a, uint8_t* d_out_u8, size_t n,
                        void* stream);

/* FiniteFieldArray.__matmul__ (mpyc/finfields.py:1126-1146; np_matmul's local step, runtime.py:2531):
 * C[r x c] = A[r x k] @ B[k x c] mod p, all row-major and contiguous.  Exact big-int semantics: the k
 * products are accumulated unreduced and reduced once, like `(a @ b) % p`. */
int mpyc_b200_ff_matmul(const mpyc_b200_field* f, const void* d_a, const void* d_b, void* d_c,
                        size_t r, size_t k, size_t c, void* stream);

/* ---- protocol-local algebra on raw share values (SURVEY 8f N3 / N4; prime fields) -------------
 * Between two openings MPyC's protocols compute on the RAW share values in NumPy object loops and reduce when
 * the result enters a field array (finfields.py:717-725).  These entry points are those steps mod p (reduction is
 * a ring homomorphism, so the field array that results is the same bit for bit); `&` and `>>` are applied to
 * canonical residues, as the reference applies them to the canonical result of Runtime.output. */

/* out = a*b + c; d_b == NULL: a*a + c -- np_random_bits' `_r.value**2 + z.value` (runtime.py:4252) */
int mpyc_b200_ff_fma(const mpyc_b200_field* f, const void* d_a, const void* d_b, const void* d_c, void* d_out,
                     size_t n, void* stream);
/* out = a*s + t for canonical host scalars s, t (L limbs each) -- np_random_bits' tail `bits += 1; bits *= (p+1)>>1;
 * bits <<= f` (runtime.py:4267-4271) is one call with s = 2^f (p+1)/2, t = s; `x << l`, `(x << 1) - 1`, `x + (1 << l)` alike */
int mpyc_b200_ff_axpb(const mpyc_b200_field* f, const void* d_a, const uint64_t* h_s, const uint64_t* h_t,
                      void* d_out, size_t n, void* stream);
/* out = a & (2^nbits - 1) -- `c.value & ((1<<f) - 1)` on an opened value (runtime.py:870,3657) */
int mpyc_b200_ff_low_bits(const mpyc_b200_field* f, const void* d_a, int nbits, void* d_out, size_t n, void* stream);
/* d_out_u8[h] = a[h] != 0 (d_out_u8 may be NULL), *d_count = number of non-zero elements --
 * `mask = _r2.value != 0; np.count_nonzero(mask)` (runtime.py:4254-4255) */
int mpyc_b200_ff_nonzero(const mpyc_b200_field* f, const void* d_a, uint8_t* d_out_u8, uint64_t* d_count, size_t n,
                         void* stream);
/* out[i] = sum_j bits[i*nbits + j] * 2^e(j) mod p over the (n, nbits) row-major matrix d_bits of arbitrary residues
 * (shares of bits); e(j) = j (descending == 0) or nbits-1-j --
 * `np.sum(r_bits.value.reshape((n, f)) << np.arange(f), axis=1)` (runtime.py:860, 4415) and np_sgn's
 * `np.sum(r_bits << np.arange(l-1, -1, -1), axis=1)` (runtime.py:3650-3651).  d_bits / d_out 16-byte aligned. */
int mpyc_b200_ff_bits_compose(const mpyc_b200_field* f, const void* d_bits, size_t n, int nbits, int descending,
                              void* d_out, void* stream);
/* out[j*out_stride + i] = bit e(j) of the canonical residue c[i], as a field element 0 / 1 (out_stride in elements) --
 * `np.right_shift.outer(c, shifts).T & 1` (runtime.py:3660, 4423) */
int mpyc_b200_ff_bits_decompose(const mpyc_b200_field* f, const void* d_c, size_t n, int nbits, int descending,
                                void* d_out, size_t out_stride, void* stream);
/* (rows, cols) matrices of elements, row-major and contiguous -- the (l, n) bit-matrix algebra of np_sgn:
 * out (cols, rows) = in^T (`r_bits.T`, runtime.py:3661; not in place);
 * out[j][i] = sum_{j' <= j} in[j'][i] (`np.cumsum(..., axis=0)`, runtime.py:3667);
 * out[j][i] = a[j][i] (op) b[i], reflected: b[i] (op) a[j][i] (`s_sign - <matrix>`, NumPy row broadcast, runtime.py:3670). */
int mpyc_b200_ff_transpose(const mpyc_b200_field* f, const void* d_in, size_t rows, size_t cols, void* d_out, void* stream);
int mpyc_b200_ff_cumsum_rows(const mpyc_b200_field* f, const void* d_in, size_t rows, size_t cols, void* d_out, void* stream);
int mpyc_b200_ff_binop_rows(const mpyc_b200_field* f, int op, int reflected, const void* d_a, const void* d_b, void* d_out,
                            size_t rows, size_t cols, void* stream);
/* ---- sums along an axis (K7; prime fields) ----------------------------------------------------
 * d_in is a C-ordered array viewed as (outer, len, inner): len is the length of the axis, outer the product of the axes
 * before it, inner the product of the axes after it.  Any 8-byte aligned d_in works (a slice may start at any element).
 *
 * np.sum(a, axis, initial=...) / FiniteFieldArray.sum (mpyc/finfields.py:1332-1337, 766-819; Runtime.np_sum,
 * runtime.py:3476-3506): out[o][i] = (initial + sum_r in[o][r][i]) mod p, out (outer, inner).  initial: L canonical host
 * limbs, or NULL for 0.  len == 0 writes initial. */
int mpyc_b200_ff_sum_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                          const uint64_t* initial, void* d_out, void* stream);
/* np.cumsum(a, axis) / np.cumulative_sum(a, axis, include_initial) (Runtime.np_cumsum / np_cumulative_sum,
 * runtime.py:3510-3549): out[o][inc + r][i] = sum_{r' <= r} in[o][r'][i] mod p, out (outer, len + inc, inner) with
 * inc = include_initial != 0 and a zero row first when inc.  d_in and d_out must not overlap. */
int mpyc_b200_ff_cumsum_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                             int include_initial, void* d_out, void* stream);

/* ---- strided views, joins and broadcasts (K8) --------------------------------------------------
 * A view of a buffer of `len` elements: element (c_0, .., c_{rank-1}) is at
 *   offset + sum_k o_k * stride[k],  o_k = index[c_k] on index_axis, else c_k
 * Strides are signed element counts (negative: a flip, 0: a broadcast axis).  index (host memory, extent[index_axis]
 * int64 entries) is uploaded by the call; index_axis = -1 for none.  Every element of a non-empty view must lie in
 * [0, len); rank <= MPYC_B200_VIEW_RANK (the caller collapses adjacent axes first). */
#define MPYC_B200_VIEW_RANK 6
typedef struct {
    int64_t offset;
    int32_t rank;
    int32_t index_axis;
    int64_t extent[MPYC_B200_VIEW_RANK];
    int64_t stride[MPYC_B200_VIEW_RANK];
    const int64_t* index;
} mpyc_b200_view;
/* dst view <- src view, elements of elem_bytes in {1 (GF(2^8)), 8, 16, 24, 32} (any field: layout does not depend on it).
 * Both views have the same rank and extents; the buffers must not overlap.  Replaces the copies behind NumPy's views of
 * field arrays: FiniteFieldArray.__getitem__ / __setitem__ (mpyc/finfields.py:1004-1029), transpose / swapaxes / T
 * (:1358-1368) and np.concatenate / stack / flip / roll / moveaxis through __array_function__ (:766-819); used by
 * Runtime.np_getitem / np_update / np_transpose / np_concatenate / np_stack / np_flip / np_roll, np_sort, np_argmax and
 * np_add_bits (mpyc/runtime.py:1758-1773, 2657-2679, 3741-3820, 4310-4325). */
int mpyc_b200_copy_view(size_t elem_bytes, const void* d_src, size_t src_len, const mpyc_b200_view* src, void* d_dst,
                        size_t dst_len, const mpyc_b200_view* dst, void* stream);
/* out = a (op) b mod p on prime fields, op ADD / SUB / MUL: a and b are views (no index axis) whose extents are the
 * broadcast shape, out is contiguous in C order of it; a broadcast operand is read in place (stride 0).  out must not
 * overlap a or b.  NumPy's broadcasting of FiniteFieldArray + - * (mpyc/finfields.py:1056-1124), e.g. np_add_bits'
 * `c1[..., -1, np.newaxis] * d2` (mpyc/runtime.py:4310-4325). */
int mpyc_b200_ff_binop_view(const mpyc_b200_field* f, int op, const void* d_a, size_t a_len, const mpyc_b200_view* a,
                            const void* d_b, size_t b_len, const mpyc_b200_view* b, void* d_out, void* stream);

/* ---- determinants, linear solves and inverses (K9) ----------------------------------------------
 * Prime fields; matrices are dense, row-major, elements contiguous.  Inputs are never modified (the elimination runs on
 * a stream-ordered workspace copy).  Both entry points reject sizes whose byte counts overflow, n == 0 and an output that
 * overlaps an input with MPYC_B200_EINVAL before any CUDA call.
 *
 * d_out[b] = det of the n x n matrix b of d_a (batch x n x n), as FiniteFieldArray.gauss_det computes it
 * (mpyc/finfields.py:916-955): Gaussian elimination that swaps row k with the first row below it with a nonzero entry
 * in column k when a[k][k] == 0, and does NOT negate the result for a swap; 0 for a singular matrix.  np.linalg.det and
 * Runtime.np_det (mpyc/runtime.py:3951-3982). */
int mpyc_b200_ff_det(const mpyc_b200_field* f, const void* d_a, size_t batch, size_t n, void* d_out, void* stream);
/* d_x (n x nrhs) = d_a^-1 d_b for d_a n x n and d_b n x nrhs; d_b == NULL means the identity (nrhs must be n), which gives
 * the inverse.  gauss_solve / gauss_inv (mpyc/finfields.py:872-914): np.linalg.solve / inv.  Synchronises the stream;
 * MPYC_B200_EZERODIV ("no inverse exists") when d_a is singular, d_x is then undefined. */
int mpyc_b200_ff_solve(const mpyc_b200_field* f, const void* d_a, size_t n, const void* d_b, size_t nrhs, void* d_x,
                       void* stream);

/* ---- 1-D convolution (K10) ----------------------------------------------------------------------
 * d_c[j] = sum_{i + l = lo + j} a[i] * b[l] mod p for j < count (np.convolve, finfields.py:766-819; Runtime.np_convolve,
 * runtime.py:2580-2634; the secret-shift branch of Runtime.np_roll, runtime.py:3300-3314).  Prime fields.  The window
 * [lo, lo + count) of the full result (m + n - 1 elements) is computed alone: np.convolve's 'full' is lo = 0,
 * count = m + n - 1; with s = min(m, n), g = max(m, n), 'same' is lo = (s - 1) / 2, count = g and 'valid' is lo = s - 1,
 * count = g - s + 1.  Any 8-byte aligned buffers work.  MPYC_B200_EINVAL before any CUDA call for m == 0 or n == 0,
 * lo + count > m + n - 1, byte counts that overflow and an output that overlaps an input; count == 0 does nothing. */
int mpyc_b200_ff_convolve(const mpyc_b200_field* f, const void* d_a, size_t m, const void* d_b, size_t n,
                          size_t lo, size_t count, void* d_c, void* stream);

/* ---- division and selection (K11) ---------------------------------------------------------------
 * d_out[h] = d_num[h] * d_den[h]^-1 mod p in one Montgomery-trick pass (FiniteFieldArray.__truediv__ / __itruediv__,
 * finfields.py:1199-1225, whose `self.value * cls._reciprocal(other)` it replaces; Runtime.np_reciprocal's `r / ar`,
 * runtime.py:1290).  Prime fields.  MPYC_B200_EZERODIV if any d_den[h] == 0 (synchronises the stream, as ff_inv); d_out
 * then holds 0 where d_den[h] == 0 and the quotient everywhere else: a zero does not spoil its batch.  MPYC_B200_EINVAL
 * before any CUDA call for null buffers, byte counts that overflow and an output that overlaps either input (the forward
 * pass keeps prefix products in d_out); num and den may be the same buffer. */
int mpyc_b200_ff_div(const mpyc_b200_field* f, const void* d_num, const void* d_den, void* d_out, size_t n, void* stream);

/* d_out[h] = ((d_mask[h] != 0) != invert) ? X(h) : Y(h) mod p: np.where(cond, x, y) of field arrays and raw share values
 * (finfields.py:766-819; Runtime._np_is_zero, runtime.py:3614-3615; Runtime.np_lsb, runtime.py:1819).  A side is
 * d_x[h] * s + t with h_x_st = {s (L limbs), t (L limbs)}, canonical residues, or the constant t when d_x is null (likewise
 * Y).  d_mask: n bytes in device memory.  Element buffers need 8-byte alignment only.  Prime fields; MPYC_B200_EINVAL
 * before any CUDA call for null buffers or maps, non-canonical scalars, byte counts that overflow and an output that
 * overlaps an input. */
int mpyc_b200_ff_select(const mpyc_b200_field* f, const uint8_t* d_mask, int invert, const void* d_x, const uint64_t* h_x_st,
                        const void* d_y, const uint64_t* h_y_st, void* d_out, size_t n, void* stream);

/* ---- per-element exponents (K12) ----------------------------------------------------------------
 * d_out[h] = base(h)^e[h] mod p (PrimeFieldArray._pow with an exponent array, finfields.py:1409-1414; gmpy.powmod_exp_list,
 * gmpy.py:288-290, which Runtime._np_pow_public_int_base_secret_integral_exponent calls twice, runtime.py:1408,1422).
 * d_exps: n exponents of exp_limbs (1..4) little-endian 64-bit limbs each, none wider than exp_bits <= 64 * exp_limbs bits
 * (the loop bound); not reduced.  Exactly one base:
 *   h_base (L canonical limbs on the host): a public base for every element (fixed-base comb).  d_signs (n bytes, may be
 *     null): a nonzero byte makes that exponent negative, base^-e[h]; MPYC_B200_EZERODIV for a zero base with d_signs.
 *   d_base (n elements): one base per element; exponents are non-negative (d_signs must be null).
 * Buffers need 8-byte alignment only.  Prime fields (MPYC_B200_EUNSUPPORTED otherwise); MPYC_B200_EINVAL before any CUDA
 * call for null buffers, both or neither base, d_signs with d_base, a non-canonical h_base, exp_limbs outside 1..4,
 * exp_bits > 64 * exp_limbs, byte counts that overflow and an output that overlaps an input. */
int mpyc_b200_ff_pow_exp(const mpyc_b200_field* f, const void* d_base, const uint64_t* h_base, const uint64_t* d_exps,
                         int exp_limbs, int exp_bits, const uint8_t* d_signs, size_t n, void* d_out, void* stream);

/* Y[k][v][m][n] = B[v] + 'same' 2-D correlation of X[k][r][m][n] with W[v][r][s][s] summed over the r input channels,
 * mod p, s odd -- demos/np_cnnmnist.py:69-81 (convolvetensor's np.correlate loops followed by field.array(Y)).
 * All arrays contiguous, row-major. */
int mpyc_b200_ff_conv2d(const mpyc_b200_field* f, const void* d_x, const void* d_w, const void* d_b, void* d_y,
                        int k, int r, int m, int n, int v, int s, void* stream);

/* ---- Shamir share generation ---------------------------------------------------------------
 * thresha.np_random_split (mpyc/thresha.py:47-64) with the coefficient matrix C given explicitly:
 *   shares[i][h] = sum_{j=0..t} (i+1)^j * M[j][h] mod p,   M[0] = secrets, M[j] = coeffs row j-1
 * i.e. coeffs row j-1 holds the coefficient of X^j for every secret (the (t, n) row-major layout of
 * thresha.py:60).  shares: m rows.  0 <= t < m.  For GF(2^8) the points are the field elements with
 * integer encoding i+1 (thresha.py:54,61). */
int mpyc_b200_shamir_split(const mpyc_b200_field* f, const void* d_secrets, const void* d_coeffs,
                           size_t coeff_stride, void* d_shares, size_t share_stride, size_t n,
                           int t, int m, void* stream);
/* Same, coefficients generated on the device and never written to memory ("generate mode"):
 * a ChaCha20 keystream keyed by key32/nonce (caller supplies fresh CSPRNG bytes, the role of
 * secrets.randbelow in thresha.py:58-60), reduced to [0, p) from 64 extra bits.  Not bit-exact
 * with anything (neither is the reference: its randomness is unseeded); shares are a valid
 * degree-t sharing and recombine to the secrets. */
int mpyc_b200_shamir_split_generate(const mpyc_b200_field* f, const void* d_secrets, void* d_shares,
                                    size_t share_stride, size_t n, int t, int m,
                                    const uint8_t key32[32], uint64_t nonce, void* stream);

/* Same, every share row written to its own destination: d_share_rows is a HOST array of m device pointers (m <= 32),
 * row i of n elements.  The pointers may refer to another GPU's memory mapped into this process (CUDA IPC / peer
 * access): a dealer then writes each recipient's row straight into the recipient GPU over NVLink -- the exchange
 * step of runtime.py:660-669 fused into share generation (mpyc_b200.exchange.PeerReshare). */
int mpyc_b200_shamir_split_generate_rows(const mpyc_b200_field* f, const void* d_secrets, void* const* d_share_rows,
                                         size_t n, int t, int m, const uint8_t key32[32], uint64_t nonce, void* stream);

/* ---- Lagrange recombination ----------------------------------------------------------------
 * thresha._recombination_vector (mpyc/thresha.py:67-85): lambda[r][i] for x-coordinates xs[0..k)
 * and recombination points x_rs[0..width); written as width*k*L host limbs, canonical. */
int mpyc_b200_recombination_vector(const mpyc_b200_field* f, const int64_t* xs, int k,
                                   const int64_t* x_rs, int width, uint64_t* h_lambda);
/* thresha.np_recombine (mpyc/thresha.py:119-132): out[r][h] = sum_i lambda[r][i] * shares_i[h] mod p.
 * d_share_rows: host array of k device pointers (one row of n elements each; rows may come from
 * different buffers, as the k received messages do in runtime.py:582-586,672-680). */
int mpyc_b200_shamir_recombine(const mpyc_b200_field* f, const void* const* d_share_rows,
                               const int64_t* xs, int k, const int64_t* x_rs, int width,
                               void* d_out, size_t out_stride, size_t n, void* stream);

/* ---- PRSS linear step ------------------------------------------------------------------------
 * thresha.np_pseudorandom_share / np_pseudorandom_share_0 (mpyc/thresha.py:163-173,201-217) after
 * the PRF: for each of nsub key subsets S the caller provides the raw SHAKE128 output stream
 * (thresha.py:257) as n*d chunks of chunk_bytes little-endian bytes.  out[h] =
 *   sum_S  f_S(i) * sum_{j<d} (chunk_{S,h,j} mod p) * w[j]   mod p
 * with h_coef[S] = f_S(i) (thresha.py:135-141) and h_weights[j] = 1 (d = 1, share) or (i+1)^(j+1)
 * (share_0), both canonical host limbs.  bound_bits == 0: the PRF bound is the field order (chunks are
 * reduced mod p); bound_bits = b > 0: the bound is 2^b <= p (runtime.py:4076, chunks are masked to b
 * bits, chunk_bytes == ceil(b/8)).  GF(2^8): one byte per chunk, bound_bits = b in 1..8 masks it to b bits (bound 2^b;
 * b = 1 is runtime.random_bits on a characteristic-2 field, runtime.py:4138,4218), 0 = the whole byte.  Any other bound:
 * mpyc_b200_prf_reduce first. */
int mpyc_b200_prss_combine(const mpyc_b200_field* f, const uint8_t* d_prf_bytes, size_t subset_stride_bytes,
                           int nsub, int d, int chunk_bytes, int bound_bits, const uint64_t* h_coef,
                           const uint64_t* h_weights, void* d_out, size_t n, void* stream);

/* Host-only: the small-integer form K4 uses when it exists.  f_S(i) (thresha.py:135-141) is a ratio of small integers, so
 * for some k <= 20 every h_coef[S] * k! mod p is a small signed integer num_S (|num_S| < 2^57): h_num[S] receives it and
 * h_scale_inv (L limbs, may be NULL) receives (k!)^-1 mod p, i.e. coef_S = num_S * scale_inv mod p.  EUNSUPPORTED if the
 * coefficients (or the weights, which must be plain integers < 2^58) have no such form; the kernel then uses full products. */
int mpyc_b200_prss_small_form(const mpyc_b200_field* f, int nsub, int d, const uint64_t* h_coef,
                              const uint64_t* h_weights, int64_t* h_num, uint64_t* h_scale_inv);
/* The same with the PRF evaluated inside the library (thresha.PRF.__call__, mpyc/thresha.py:240-266, and the
 * callers thresha.py:163-217): subset S's stream is SHAKE128(key_S || uci) squeezed to n*d*chunk_bytes bytes.
 * h_keys: nsub keys of key_bytes bytes each (PRF.key), h_uci: the unique call identifier bytes.  One sponge is
 * sequential, so the nsub sponges run on up to max_threads host threads (0 = all hardware threads), squeezed
 * chunk by chunk into pinned staging buffers and overlapped with the H2D copy and the combine kernel of the
 * previous chunk.  h_out: host buffer of n elements (limb layout).  device = CUDA device ordinal. */
int mpyc_b200_prss_host(const mpyc_b200_field* f, const uint8_t* h_keys, int key_bytes, const uint8_t* h_uci,
                        size_t uci_bytes, int nsub, int d, int chunk_bytes, int bound_bits, const uint64_t* h_coef,
                        const uint64_t* h_weights, void* h_out, size_t n, int device, int max_threads);
/* PRF values for an ARBITRARY bound (thresha.PRF.__call__, mpyc/thresha.py:257-261: int.from_bytes(chunk, 'little') % bound).
 * The two bounds of the secure-randomness protocols (the field order, 2^b <= p) are folded into prss_combine; every other
 * bound -- runtime._convert's (1 << (k+l)) // comb(m,t) + 1 (mpyc/runtime.py:735-739), the source field's order used on a
 * smaller target field (runtime.py:758-760), a power of two above p -- is reduced by this kernel first.  h_bound:
 * bound_nlimbs (<= 5) little-endian host limbs, 2 <= bound <= 2^256.  For each of nsub streams, `count` chunks of
 * chunk_bytes (<= 8 * (limbs(bound) + 2)) bytes are read from d_prf_bytes + S * subset_stride_bytes and
 * d_values + S * value_stride_bytes receives `count` values of *value_bytes bytes each: 8 * limbs(bound - 1)
 * little-endian bytes, or, when f is a GF(2^8) handle, ONE byte -- the GF(2)[X] polynomial whose integer encoding is the
 * reduced chunk (gfpx's int coercion, mpyc/gfpx.py:73-81) modulo the field polynomial.  f may be NULL (plain integers).
 * Feed the values to mpyc_b200_prss_combine with chunk_bytes = *value_bytes, bound_bits = 0. */
int mpyc_b200_prf_reduce(const mpyc_b200_field* f, const uint8_t* d_prf_bytes, size_t subset_stride_bytes, int nsub,
                         size_t count, int chunk_bytes, const uint64_t* h_bound, int bound_nlimbs, void* d_values,
                         size_t value_stride_bytes, int* value_bytes, void* stream);
/* mpyc_b200_prss_host for an arbitrary PRF bound (see mpyc_b200_prf_reduce): per pipeline chunk the library runs
 * the reduction kernel and then the combine kernel on the reduced values. */
int mpyc_b200_prss_host_bound(const mpyc_b200_field* f, const uint8_t* h_keys, int key_bytes, const uint8_t* h_uci,
                              size_t uci_bytes, int nsub, int d, int chunk_bytes, const uint64_t* h_bound, int bound_nlimbs,
                              const uint64_t* h_coef, const uint64_t* h_weights, void* h_out, size_t n, int device,
                              int max_threads);
/* SHAKE128 (FIPS 202) of `in`, squeezed to outlen bytes: hashlib.shake_128(in).digest(outlen), the XOF of
 * thresha.PRF (mpyc/thresha.py:257).  Host only; no GPU involved. */
int mpyc_b200_shake128(const uint8_t* in, size_t inlen, uint8_t* out, size_t outlen);

/* The XOF streams of one PRSS call: `count` sponges SHAKE128(key_i || suffix) (thresha.py:257: key_i of each key subset,
 * suffix = the unique call identifier), each squeezed to outlen bytes at out + i * out_stride.  On hosts with AVX-512F the
 * sponges advance eight at a time in lock step on one core (csrc/shake128_x8.h; *used_wide = 1), which is what a PRSS
 * worker thread that owns several key subsets does inside mpyc_b200_prss_host.  Host only; no GPU involved. */
int mpyc_b200_shake128_multi(const uint8_t* keys, int key_bytes, const uint8_t* suffix, size_t suffix_len, int count,
                             uint8_t* out, size_t out_stride, size_t outlen, int* used_wide);

/* Lets kernels launched on `device` load/store memory of `peer_device` (cudaDeviceEnablePeerAccess; idempotent).
 * Needed once per pair before mpyc_b200_shamir_split_generate_rows is given rows on another GPU. */
int mpyc_b200_enable_peer_access(int device, int peer_device);

/* Device buffers that kernels of ANOTHER process (one process per GPU) can store into: peer_alloc = cudaMalloc (zeroed)
 * + cudaIpcGetMemHandle; peer_open maps an exported buffer into the calling process in the current device's context
 * with peer access to the exporting GPU enabled (cudaIpcOpenMemHandle, cudaIpcMemLazyEnablePeerAccess).  The owner
 * frees with peer_free after every importer has called peer_close. */
int mpyc_b200_peer_alloc(size_t bytes, void** d_ptr, uint8_t handle[64]);
int mpyc_b200_peer_open(const uint8_t handle[64], void** d_ptr);
int mpyc_b200_peer_close(void* d_ptr);
int mpyc_b200_peer_free(void* d_ptr);

/* ---- utilities -------------------------------------------------------------------------------
 * deterministic synthetic residues (tests, bench): element h = (L+1 SplitMix64 words of counter
 * seed + (stream_id << 56) + h*(L+1) + w, truncated to bits(p)+64 bits) mod p -- same recipe as
 * oracle/shamir_oracle.py:synth_elements. */
int mpyc_b200_fill_random(const mpyc_b200_field* f, void* d_out, size_t n, uint64_t seed,
                          uint64_t stream_id, void* stream);
/* out[0] = number of positions where a and b differ (device-side compare for full-size parity) */
int mpyc_b200_count_mismatch(const mpyc_b200_field* f, const void* d_a, const void* d_b, size_t n,
                             uint64_t* d_count, void* stream);

/* ---- host-buffer entry points (what a drop-in caller with host data uses) ---------------------
 * Inputs and outputs are HOST buffers in the same limb layout; the library stages them through
 * pinned buffers, overlapping H2D copy, kernel and D2H copy chunk by chunk on its own streams, and
 * returns when the output is complete.  device = CUDA device ordinal. */
int mpyc_b200_shamir_split_host(const mpyc_b200_field* f, const void* h_secrets, const void* h_coeffs,
                                size_t coeff_stride, void* h_shares, size_t share_stride, size_t n,
                                int t, int m, int device);
/* np_random_split as the reference defines it -- secrets in, shares out, randomness drawn inside (thresha.py:47-64):
 * generate mode through the same chunk pipeline.  Chunk c uses nonce + c with the caller's key: pass a fresh key per
 * call (t <= 4). */
int mpyc_b200_shamir_split_generate_host(const mpyc_b200_field* f, const void* h_secrets, void* h_shares,
                                         size_t share_stride, size_t n, int t, int m, const uint8_t key32[32],
                                         uint64_t nonce, int device);
int mpyc_b200_shamir_recombine_host(const mpyc_b200_field* f, const void* const* h_share_rows,
                                    const int64_t* xs, int k, const int64_t* x_rs, int width,
                                    void* h_out, size_t out_stride, size_t n, int device);
/* A party's steady state in a stream of resharing rounds (mpyc/runtime.py:660-680): recombine the rows received for batch
 * j (mpyc_b200_shamir_recombine_host's arguments, n_rec elements) WHILE dealing the shares of batch j+1
 * (mpyc_b200_shamir_split_host's arguments, n_split elements).  One host thread issues the pipeline chunks of both jobs
 * alternately on two independent stream sets, so the D2H-heavy split and the H2D-heavy recombination keep both PCIe
 * directions busy.  Either job may be empty.  Results are identical to the two separate calls. */
int mpyc_b200_shamir_reshare_step_host(const mpyc_b200_field* f, const void* h_secrets, const void* h_coeffs,
                                       size_t coeff_stride, void* h_shares, size_t share_stride, size_t n_split, int t, int m,
                                       const void* const* h_share_rows, const int64_t* xs, int k, const int64_t* x_rs,
                                       int width, void* h_out, size_t out_stride, size_t n_rec, int device);
int mpyc_b200_ff_binop_host(const mpyc_b200_field* f, int op, const void* h_a, const void* h_b,
                            void* h_out, size_t n, int device);

#ifdef __cplusplus
}
#endif
#endif /* MPYC_B200_H */
