// Host-side launch interface between the C-ABI translation unit (api.cu) and the per-limb-count
// kernel instantiation units (inst_L{1,2,3,4}.cu), which are compiled in parallel.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include "kernels.cuh"

extern std::atomic<unsigned long long> g_mpyc_launches;

// host-side description of where K2 (generate mode) puts its m share rows
struct ShareDst {
    u64* base = nullptr;
    size_t stride = 0;
    int use_rows = 0;
    u64* rows[MPYC_MAX_SHARE_ROWS] = {};
};

// persistent-grid sizing: enough CTAs to cover the items, capped at one full wave
int mpyc_grid_size(const void* kernel, size_t items, size_t dyn_smem);

// stream-ordered scratch for split partials from the library's per-device pool, which keeps its memory between calls
// (api.cu); release with cudaFreeAsync on the same stream
cudaError_t mpyc_scratch_alloc(u64** p, size_t bytes, cudaStream_t st);

template <int L>
struct Launch {
    // op in {OP_ADD, OP_SUB, OP_MUL, OP_NEG}; scal != nullptr -> broadcast second operand (host limbs)
    static cudaError_t binop(const FieldParams& fp, int op, const u64* a, const u64* b, const u64* scal, u64* out,
                             size_t n, cudaStream_t st);
    // mode 0: out = a^e; mode 1: out8 = (a^e != p-1)
    static cudaError_t pow(const FieldParams& fp, const ExpParams& ex, int mode, const u64* a, u64* out,
                           unsigned char* out8, int* zero_flag, size_t n, cudaStream_t st);
    // out[h] = a[h]^-1 (0 for a[h] == 0, reported in zero_flag); ex = p - 2; a and out must not alias.
    // num (K11): out[h] = num[h] * a[h]^-1 in the same pass; num must not alias out
    static cudaError_t inv_batch(const FieldParams& fp, const ExpParams& ex, const u64* a, u64* out, int* zero_flag,
                                 size_t n, cudaStream_t st, const u64* num = nullptr);
    static cudaError_t split(const FieldParams& fp, bool full, const u64* secrets, const u64* coeffs, size_t cstride,
                             u64* shares, size_t sstride, size_t n, int t, int m, const u64* gtab, u32 tab_bytes,
                             cudaStream_t st);
    // dst: strided matrix (base, stride in limbs) or explicit row pointers (use_rows; small-form tables only)
    static cudaError_t split_gen(const FieldParams& fp, bool full, const ChaChaKey& key, const u64* secrets,
                                 const ShareDst& dst, size_t n, int t, int m, const u64* gtab, u32 tab_bytes, cudaStream_t st);
    // small: 64-bit signed-magnitude lambda table
    static cudaError_t recombine(const FieldParams& fp, bool small, const RowPtrs& rows, int k, int width, const u64* gtab,
                                 u32 tab_bytes, u64* out, size_t ostride, size_t n, cudaStream_t st);
    // small: subset coefficients as 64-bit signed-magnitude constants + D^-1 (api.cu: prss_small_table)
    // simple (with small): d == 1 and the weight is 1
    static cudaError_t prss(const FieldParams& fp, bool small, bool simple, const unsigned char* bytes, size_t subset_stride, int nsub, int d,
                            int chunk_bytes, int bound_bits, const u64* gtab, u32 tab_bytes, u64* out, size_t n,
                            cudaStream_t st);
    static cudaError_t matmul(const FieldParams& fp, const u64* A, const u64* B, u64* C, size_t r, size_t k, size_t c,
                              cudaStream_t st);
    static cudaError_t fill_random(const FieldParams& fp, u64* out, size_t n, u64 base, cudaStream_t st);
    // ---- K6: protocol-local algebra on raw share values (local.cuh) ----
    // out = a*b + c (square: a*a + c, b ignored)
    static cudaError_t fma(const FieldParams& fp, bool square, const u64* a, const u64* b, const u64* c, u64* out, size_t n,
                           cudaStream_t st);
    // out = a*s + t for canonical host scalars s, t
    static cudaError_t axpb(const FieldParams& fp, const u64* a, const u64* s, const u64* t, u64* out, size_t n, cudaStream_t st);
    // out = a & (2^nbits - 1)
    static cudaError_t low_bits(const FieldParams& fp, const u64* a, int nbits, u64* out, size_t n, cudaStream_t st);
    // out8[h] = a[h] != 0 (out8 may be null); *count (device, zeroed by the caller) += non-zero elements
    static cudaError_t nonzero(const FieldParams& fp, const u64* a, unsigned char* out8, unsigned long long* count, size_t n,
                               cudaStream_t st);
    // out[i] = sum_j bits[i*f + j] 2^e(j), e(j) = j or f-1-j
    static cudaError_t bits_compose(const FieldParams& fp, const u64* bits, u64* out, size_t n, int f, bool descending, cudaStream_t st);
    // out[j*ostride + i] = bit e(j) of c[i]   (ostride in elements)
    static cudaError_t bits_decompose(const FieldParams& fp, const u64* c, u64* out, size_t ostride, size_t n, int l, bool descending,
                                      cudaStream_t st);
    // out (C, R) = in (R, C) transposed; out = a (R, C) (op) b (C) broadcast over the rows (reflected: b (op) a)
    static cudaError_t transpose(const FieldParams& fp, const u64* in, u64* out, size_t R, size_t C, cudaStream_t st);
    static cudaError_t binop_rows(const FieldParams& fp, int op, bool reflected, const u64* a, const u64* b, u64* out, size_t R,
                                  size_t C, cudaStream_t st);
    // Y (k, v, m, n) = 'same' correlation of X (k, r, m, n) with W (v, r, s, s) over the r input channels + B (v); s odd
    static cudaError_t conv2d(const FieldParams& fp, const u64* X, const u64* W, const u64* B, u64* Y, int k, int r, int m, int n,
                              int v, int s, cudaStream_t st);
    // ---- K7: along the middle axis of a C-ordered (O, R, I) array (reduce.cuh) ----
    // out (O, I) = init + sum_r in (O, R, I); init: L canonical host limbs, or null for 0
    static cudaError_t sum_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, const u64* init,
                                cudaStream_t st);
    // out (O, R + inc, I) = running sums of in (O, R, I) along R, after a zero row when inc; in and out must not overlap
    static cudaError_t scan_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool inc,
                                 cudaStream_t st);
    // ---- K8: broadcast arithmetic on views (layout.cuh) ----
    // out (C order over pl.ext) = a_view (op) b_view, op in {OP_ADD, OP_SUB, OP_MUL}
    static cudaError_t binop_view(const FieldParams& fp, int op, const BinopPlan& pl, const u64* a, const u64* b, u64* out,
                                  cudaStream_t st);
};

// K8 (inst_layout.cu): dst_view <- src_view for elements of elem_bytes in {1, 8, 16, 24, 32}; the views are validated and
// their index tables (if any) are in device memory
cudaError_t launch_copy_view(const CopyPlan& pl, size_t elem_bytes, const void* src, void* dst, cudaStream_t st);

// K9 (inst_linalg.cu): out[b] = det of the n x n matrix b of a (batch x n x n; the reference's determinant, which ignores
// the sign of its row swaps).  Prime fields; sizes validated by the caller.
cudaError_t launch_det(const FieldParams& fp, const u64* a, size_t batch, size_t n, u64* out, cudaStream_t st);
// x (n x nrhs) = a^-1 b, b null: the identity (nrhs = n).  Synchronises st; *singular = 1 when a has no inverse (x is
// then undefined).
cudaError_t launch_solve(const FieldParams& fp, const u64* a, size_t n, const u64* b, size_t nrhs, u64* x, int* singular,
                         cudaStream_t st);

// K10 (inst_conv.cu): c[j] = sum_{i + l = lo + j} a[i] b[l] mod p for j < count (a of m, b of n elements).  Prime fields;
// sizes validated by the caller.
cudaError_t launch_convolve(const FieldParams& fp, const u64* a, size_t m, const u64* b, size_t n, size_t lo, size_t count,
                            u64* c, cudaStream_t st);

// K11 (inst_select.cu): out[h] = (mask[h] != 0) != invert ? X(h) : Y(h), a side being x[h] * xs + xt, or the constant xt
// when x is null (xs, xt: L canonical limbs each).  Prime fields; sizes validated by the caller.
cudaError_t launch_select(const FieldParams& fp, const unsigned char* mask, bool invert, const u64* x, const u64* xs,
                          const u64* xt, const u64* y, const u64* ys, const u64* yt, u64* out, size_t n, cudaStream_t st);

// K12 (inst_powexp.cu): out[h] = base(h)^e[h], e[h] = el little-endian limbs of at most ebits bits.  tab non-null: the
// fixed-base form, tab = comb tables of tab_bytes (<= MPYC_PE_SMEM_MAX) in the domain, window w, nwin windows, sgn (may be
// null) picking the second table; else the per-element form on a.  Prime fields; sizes validated by the caller.
#define MPYC_PE_SMEM_MAX (96u * 1024u)
cudaError_t launch_powexp(const FieldParams& fp, const u64* a, const u64* tab, u32 tab_bytes, int w, int nwin, const u64* e,
                          int el, int ebits, const unsigned char* sgn, u64* out, size_t n, cudaStream_t st);

// K13 (inst_prod.cu), on a C-ordered (O, R, I) array as K7: out (O, I) = init * prod_r in (O, R, I) (init: L canonical host
// limbs, or null for 1); out (O, R + inc, I) = running products along R after a row of ones when inc; out (O, I) = 0 / 1
// for all (any == false) or any element along R being nonzero.  in and out must not overlap.  Prime fields; sizes
// validated by the caller.
cudaError_t launch_prod_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, const u64* init,
                             cudaStream_t st);
cudaError_t launch_cumprod_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool inc,
                                cudaStream_t st);
cudaError_t launch_all_any_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool any,
                                cudaStream_t st);

// K14 (inst_matmul_int.cu): C (r x c) = X (r x k) @ W (k x c), or with w_left W (r x k) @ X (k x c), mod p; X canonical
// field elements, W 64-bit integers (int64, or uint64 when w_unsigned).  Prime fields; sizes validated by the caller.
cudaError_t launch_matmul_int(const FieldParams& fp, const u64* X, const u64* W, bool w_unsigned, bool w_left, u64* C, size_t r,
                              size_t k, size_t c, cudaStream_t st);

// K15 (inst_gf.cu), GF(2^8) bytes: out[i] = sum_j x[i l + j] X^j mod poly (l >= 1); out = a_view (op) b_view, op OP_ADD / OP_SUB
// (both XOR) or OP_MUL; C[b] (r x c) = A + b as (r x k) @ B + b bs (k x c), a batch stride 0 broadcasting its side.  Sizes
// validated by the caller.
cudaError_t launch_gf_bits_compose(unsigned poly, const unsigned char* x, size_t n, size_t l, unsigned char* out, cudaStream_t st);
cudaError_t launch_gf_binop_view(unsigned poly, int op, const BinopPlan& pl, const unsigned char* a, const unsigned char* b,
                                 unsigned char* out, cudaStream_t st);
cudaError_t launch_gf_matmul_batched(unsigned poly, const unsigned char* A, size_t as, const unsigned char* B, size_t bs,
                                     unsigned char* C, size_t batch, size_t r, size_t k, size_t c, cudaStream_t st);

extern template struct Launch<1>;
extern template struct Launch<2>;
extern template struct Launch<3>;
extern template struct Launch<4>;
