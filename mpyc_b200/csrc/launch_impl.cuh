// Definitions of Launch<L>: picks the kernel instantiation (reduction kind, vector/scalar memory
// path, compile-time t+1) and launches it on a persistent grid.
#pragma once
#include <stdlib.h>
#include <algorithm>
#include "launch.h"

static inline bool aligned32(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31u) == 0; }
// every share row starts 32-byte aligned (stride in limbs)
static inline bool dst_aligned32(const ShareDst& dst, int m) {
    if (!dst.use_rows) return aligned32(dst.base) && (dst.stride % 4 == 0 || m <= 1);
    for (int i = 0; i < m; i++)
        if (!aligned32(dst.rows[i])) return false;
    return true;
}

template <class... KArgs, class... Args>
static cudaError_t launch_kernel(void (*kernel)(KArgs...), size_t items, size_t smem, cudaStream_t st, Args... args) {
    if (items == 0) return cudaSuccess;
    int grid = mpyc_grid_size(reinterpret_cast<const void*>(kernel), items, smem);
    if (grid <= 0) return cudaErrorLaunchFailure;
    kernel<<<grid, MPYC_THREADS, smem, st>>>(args...);
    g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

#define KIND_SWITCH(kind, MACRO)                       \
    switch (kind) {                                    \
        case KIND_GENERIC: MACRO(KIND_GENERIC); break; \
        case KIND_PM_ALIGNED: MACRO(KIND_PM_ALIGNED); break; \
        case KIND_PM_SHIFT: MACRO(KIND_PM_SHIFT); break; \
        default: return cudaErrorInvalidValue;         \
    }

// ---- elementwise ---------------------------------------------------------------------------

template <int L, int KIND, bool VEC>
static cudaError_t binop_k(const FieldParams& fp, int op, const u64* a, const u64* b, const u64* scal, u64* out,
                           size_t n, cudaStream_t st) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    ScalarParam sp = {};
    if (scal)
        for (int i = 0; i < L; i++) sp.v[i] = scal[i];
    size_t items = (n + E - 1) / E;
#define BINOP_CASE(OPC, SC) return launch_kernel(k_binop<L, KIND, OPC, SC, VEC>, items, 0, st, fp, a, b, sp, out, n)
    if (scal) {
        switch (op) {
            case OP_ADD: BINOP_CASE(OP_ADD, true);
            case OP_SUB: BINOP_CASE(OP_SUB, true);
            case OP_MUL: BINOP_CASE(OP_MUL, true);
            default: return cudaErrorInvalidValue;
        }
    }
    switch (op) {
        case OP_ADD: BINOP_CASE(OP_ADD, false);
        case OP_SUB: BINOP_CASE(OP_SUB, false);
        case OP_MUL: BINOP_CASE(OP_MUL, false);
        case OP_NEG: BINOP_CASE(OP_NEG, false);
        default: return cudaErrorInvalidValue;
    }
#undef BINOP_CASE
}

template <int L>
cudaError_t Launch<L>::binop(const FieldParams& fp, int op, const u64* a, const u64* b, const u64* scal, u64* out,
                             size_t n, cudaStream_t st) {
    const bool vec = L != 3 && aligned32(a) && aligned32(out) && (scal || op == OP_NEG || aligned32(b));
    if constexpr (L != 3) {
        if (vec) {
#define M(K) return binop_k<L, K, true>(fp, op, a, b, scal, out, n, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return binop_k<L, K, false>(fp, op, a, b, scal, out, n, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

// ---- pow family ----------------------------------------------------------------------------

template <int L>
cudaError_t Launch<L>::pow(const FieldParams& fp, const ExpParams& ex, int mode, const u64* a, u64* out,
                           unsigned char* out8, int* zero_flag, size_t n, cudaStream_t st) {
#define M(K)                                                                                              \
    if (mode == 0) return launch_kernel(k_pow<L, K, 0>, n, 0, st, fp, ex, a, out, out8, zero_flag, n);    \
    return launch_kernel(k_pow<L, K, 1>, n, 0, st, fp, ex, a, out, out8, zero_flag, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

int mpyc_sm_count();

template <int L>
cudaError_t Launch<L>::inv_batch(const FieldParams& fp, const ExpParams& ex, const u64* a, u64* out, int* zero_flag,
                                 size_t n, cudaStream_t st, const u64* num) {
    // batch length: as long as possible while every SM still gets >= 1024 threads; <= 32
    int B = 1;
    const size_t per_wave = (size_t)mpyc_sm_count() * 1024;
    while (B < 32 && n / (2 * (size_t)B) >= per_wave) B *= 2;
    if (const char* forced = getenv("MPYC_B200_INV_BATCH")) {   // tests: exercise long batches on small arrays
        const int v = atoi(forced);
        if (v >= 1 && v <= 1024) B = v;
    }
    const size_t T = (n + B - 1) / B;
#define M(K)                                                                                                      \
    if (num) return launch_kernel(k_inv_batch<L, K, true>, T, 0, st, fp, ex, a, out, zero_flag, n, T, B, num);     \
    return launch_kernel(k_inv_batch<L, K, false>, T, 0, st, fp, ex, a, out, zero_flag, n, T, B, (const u64*)nullptr)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

// ---- split ----------------------------------------------------------------------------------

// Small-table share generation sums M[0] + sum_{j>=1} M[j] (i+1)^j < (1 + m + ... + m^t) p.  When that factor is
// at most 2^31 every value handed to the per-share reduction is < 2^(k+31): generic fields may use the one-limb
// quotient (Fp::barrett_small32) and 2^64 - c the single-multiply fold (Fp::reduce_small_q32).  Returns fp with q32
// set accordingly (the copy travels as the kernel parameter).
static inline FieldParams split_q32(const FieldParams& fp, bool full, int t, int m) {
    FieldParams f = fp;
    f.q32 = 0;
    if (!full && (fp.kind == KIND_GENERIC || (fp.kind == KIND_PM_ALIGNED && fp.L == 1)) && m >= 1 && t >= 0 && t <= 16 && getenv("MPYC_B200_NO_Q32") == nullptr) {
        unsigned __int128 sum = 0, pw = 1;             // m <= 255, t <= 16: m^t < 2^128
        for (int j = 0; j <= t; j++) {
            sum += pw;
            pw *= (unsigned)m;
        }
        f.q32 = sum <= ((unsigned __int128)1 << 31) ? 1u : 0u;
    }
    return f;
}

#ifndef MPYC_SPLIT_STAGE_MAX
// the tiled K2 writes through a shared-memory stage while two CTAs per SM still fit (228 KB of shared memory per SM,
// 1 KB of it reserved per CTA); larger m store straight from registers (-DMPYC_SPLIT_STAGE_MAX=0: always; experiments)
#define MPYC_SPLIT_STAGE_MAX (113u * 1024u)
#endif

template <int L, int KIND, int TP1, bool FULL>
static cudaError_t split_tiled_k(const FieldParams& fp, const u64* secrets, const u64* coeffs, size_t cstride,
                                 u64* shares, size_t sstride, size_t n, int m, const u64* gtab, u32 tab_bytes,
                                 cudaStream_t st) {
    const size_t ntiles = n / (MPYC_TILE_LIMBS / L);
    const size_t items = std::max<size_t>(ntiles, 1) * MPYC_THREADS;
    const size_t smem = ((tab_bytes + 127u) & ~127u) + (size_t)m * MPYC_TILE_LIMBS * sizeof(u64);
    if (smem <= MPYC_SPLIT_STAGE_MAX) {
        auto kernel = k_split_tiled<L, KIND, TP1, FULL, true>;
        if (smem > 48u * 1024u) {
            cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        return launch_kernel(kernel, items, smem, st, fp, secrets, coeffs, cstride, shares, sstride, n, m, gtab, tab_bytes);
    }
    return launch_kernel(k_split_tiled<L, KIND, TP1, FULL, false>, items, tab_bytes, st, fp, secrets, coeffs, cstride,
                         shares, sstride, n, m, gtab, tab_bytes);
}

template <int L, int KIND, bool FULL, bool VEC>
static cudaError_t split_k(const FieldParams& fp, const u64* secrets, const u64* coeffs, size_t cstride, u64* shares,
                           size_t sstride, size_t n, int t, int m, const u64* gtab, u32 tab_bytes, cudaStream_t st) {
    constexpr int MAXT = FULL ? 5 : 9;
#define SPLIT_CASE(T)                                                                                            \
    case T:                                                                                                      \
        if constexpr (T <= MAXT) {                                                                               \
            if constexpr (VEC)                                                                                   \
                return split_tiled_k<L, KIND, T, FULL>(fp, secrets, coeffs, cstride, shares, sstride, n, m, gtab, \
                                                       tab_bytes, st);                                           \
            return launch_kernel(k_split<L, KIND, T, FULL>, n, tab_bytes, st, fp, secrets, coeffs, cstride, shares, \
                                 sstride, n, m, gtab, tab_bytes);                                                \
        }                                                                                                        \
        break
    switch (t + 1) {
        SPLIT_CASE(1);
        SPLIT_CASE(2);
        SPLIT_CASE(3);
        SPLIT_CASE(4);
        SPLIT_CASE(5);
        SPLIT_CASE(6);
        SPLIT_CASE(7);
        SPLIT_CASE(8);
        SPLIT_CASE(9);
        default: break;
    }
#undef SPLIT_CASE
    return cudaErrorNotSupported;   // caller falls back to k_split_dyn
}

template <int L, bool FULL, bool VEC>
static cudaError_t split_kind(const FieldParams& fp, const u64* secrets, const u64* coeffs, size_t cstride, u64* shares,
                              size_t sstride, size_t n, int t, int m, const u64* gtab, u32 tab_bytes, cudaStream_t st) {
    if constexpr (FULL) {
#define M(K) return split_k<L, K, true, VEC>(fp, secrets, coeffs, cstride, shares, sstride, n, t, m, gtab, tab_bytes, st)
        KIND_SWITCH(fp.kind, M)
#undef M
    } else {
#define M(K) return split_k<L, K, false, VEC>(fp, secrets, coeffs, cstride, shares, sstride, n, t, m, gtab, tab_bytes, st)
        KIND_SWITCH(fp.kind, M)
#undef M
    }
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::split(const FieldParams& fp0, bool full, const u64* secrets, const u64* coeffs, size_t cstride,
                             u64* shares, size_t sstride, size_t n, int t, int m, const u64* gtab, u32 tab_bytes,
                             cudaStream_t st) {
    const FieldParams fp = split_q32(fp0, full, t, m);
    const bool vec = L != 3 && aligned32(secrets) && aligned32(shares) && (t == 0 || aligned32(coeffs)) &&
                     (cstride % 4 == 0 || t <= 1) && (sstride % 4 == 0 || m <= 1);   // strides in limbs
    const int maxt = full ? 5 : 9;
    if (t + 1 > maxt) {
        if (!full) return cudaErrorInvalidValue;   // api.cu asks for full tables whenever t > 8
#define M(K) return launch_kernel(k_split_dyn<L, K>, n, 0, st, fp, secrets, coeffs, cstride, shares, sstride, n, m, t + 1, gtab)
        KIND_SWITCH(fp.kind, M)
#undef M
    }
#define GO(VECF)                                                                                                   \
    return full ? split_kind<L, true, VECF>(fp, secrets, coeffs, cstride, shares, sstride, n, t, m, gtab, tab_bytes, st) \
                : split_kind<L, false, VECF>(fp, secrets, coeffs, cstride, shares, sstride, n, t, m, gtab, tab_bytes, st)
    if constexpr (L != 3) {
        if (vec) {
            GO(true);
        }
    }
    GO(false);
#undef GO
}

// ---- split, generate mode (t <= 4) -----------------------------------------------------------------

template <int L, int KIND, bool FULL, bool VEC>
static cudaError_t split_gen_k(const FieldParams& fp, const ChaChaKey& key, const u64* secrets, const ShareDst& dst,
                               size_t n, int t, int m, const u64* gtab, u32 tab_bytes, cudaStream_t st) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    size_t items = (n + E - 1) / E;
#define GEN_CASE(T)                                                                                                 \
    case T:                                                                                                         \
        if constexpr (!FULL) {                                                                                      \
            if (dst.use_rows) {                                                                                     \
                RowsDst rd;                                                                                         \
                for (int i = 0; i < MPYC_MAX_SHARE_ROWS; i++) rd.rows[i] = dst.rows[i];                             \
                return launch_kernel(k_split_gen<L, KIND, T, FULL, VEC, RowsDst>, items, tab_bytes, st, fp, key,    \
                                     secrets, rd, n, m, gtab, tab_bytes);                                           \
            }                                                                                                       \
        }                                                                                                           \
        if (dst.use_rows) return cudaErrorNotSupported;                                                             \
        return launch_kernel(k_split_gen<L, KIND, T, FULL, VEC, StridedDst>, items, tab_bytes, st, fp, key, secrets, \
                             StridedDst{dst.base, dst.stride}, n, m, gtab, tab_bytes)
    switch (t + 1) {
        GEN_CASE(1);
        GEN_CASE(2);
        GEN_CASE(3);
        GEN_CASE(4);
        GEN_CASE(5);
        default: break;
    }
#undef GEN_CASE
    return cudaErrorNotSupported;
}

template <int L>
cudaError_t Launch<L>::split_gen(const FieldParams& fp0, bool full, const ChaChaKey& key, const u64* secrets,
                                 const ShareDst& dst, size_t n, int t, int m, const u64* gtab, u32 tab_bytes, cudaStream_t st) {
    const FieldParams fp = split_q32(fp0, full, t, m);
    const bool vec = L != 3 && aligned32(secrets) && dst_aligned32(dst, m);
#define GEN_GO(V)                                                                                                  \
    do {                                                                                                           \
        if (full) {                                                                                                \
            switch (fp.kind) {                                                                                     \
                case KIND_GENERIC: return split_gen_k<L, KIND_GENERIC, true, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
                case KIND_PM_ALIGNED: return split_gen_k<L, KIND_PM_ALIGNED, true, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
                case KIND_PM_SHIFT: return split_gen_k<L, KIND_PM_SHIFT, true, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
            }                                                                                                      \
            return cudaErrorInvalidValue;                                                                          \
        }                                                                                                          \
        switch (fp.kind) {                                                                                         \
            case KIND_GENERIC: return split_gen_k<L, KIND_GENERIC, false, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
            case KIND_PM_ALIGNED: return split_gen_k<L, KIND_PM_ALIGNED, false, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
            case KIND_PM_SHIFT: return split_gen_k<L, KIND_PM_SHIFT, false, V>(fp, key, secrets, dst, n, t, m, gtab, tab_bytes, st); \
        }                                                                                                          \
        return cudaErrorInvalidValue;                                                                              \
    } while (0)
    if constexpr (L != 3) {
        if (vec) GEN_GO(true);
    }
    GEN_GO(false);
#undef GEN_GO
}

// ---- recombine ------------------------------------------------------------------------------

template <int L, int KIND, bool SMALL, int KB>
static cudaError_t recombine_tiled_k(const FieldParams& fp, const RowPtrs& rows, int k, int width, const u64* gtab,
                                     u32 tab_bytes, u64* out, size_t ostride, size_t n, cudaStream_t st) {
    const size_t ntiles = n / (MPYC_TILE_LIMBS / L);
    return launch_kernel(k_recombine_tiled<L, KIND, SMALL, KB>, std::max<size_t>(ntiles, 1) * MPYC_THREADS, tab_bytes,
                         st, fp, rows, k, width, gtab, tab_bytes, out, ostride, n);
}

// The rows stay in registers (and the next tile's are prefetched) while that leaves room for two CTAs per SM: k <= 4
// for L <= 2 (106-128 registers at k = 3, 4), k <= 2 for L = 4 (74).  Larger k stream their rows: k = 8 in registers
// takes 166-192 registers, one CTA per SM, and C5's K3 (L = 4, k = 7) 2.19 ms instead of 1.82.
template <int L, int KIND, bool SMALL>
static cudaError_t recombine_tiled(const FieldParams& fp, const RowPtrs& rows, int k, int width, const u64* gtab,
                                   u32 tab_bytes, u64* out, size_t ostride, size_t n, cudaStream_t st) {
#define GO(KB) return recombine_tiled_k<L, KIND, SMALL, KB>(fp, rows, k, width, gtab, tab_bytes, out, ostride, n, st)
    if (k <= 2) GO(2);
    if constexpr (L <= 2) {
        if (k == 3) GO(3);
        if (k == 4) GO(4);
    }
    GO(0);
#undef GO
}

template <int L>
cudaError_t Launch<L>::recombine(const FieldParams& fp, bool small, const RowPtrs& rows, int k, int width,
                                 const u64* gtab, u32 tab_bytes, u64* out, size_t ostride, size_t n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    bool tiled = L != 3 && aligned32(out) && (ostride % 4 == 0 || width <= 1);   // stride in limbs
    for (int i = 0; i < k; i++) tiled = tiled && aligned32(rows.p[i]);
    if constexpr (L != 3) {
        if (tiled) {
#define M(K)                                                                                                       \
    return small ? recombine_tiled<L, K, true>(fp, rows, k, width, gtab, tab_bytes, out, ostride, n, st)           \
                 : recombine_tiled<L, K, false>(fp, rows, k, width, gtab, tab_bytes, out, ostride, n, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K)                                                                                                           \
    return small ? launch_kernel(k_recombine<L, K, true>, n, tab_bytes, st, fp, rows, k, width, gtab, tab_bytes, out,  \
                                 ostride, n)                                                                           \
                 : launch_kernel(k_recombine<L, K, false>, n, tab_bytes, st, fp, rows, k, width, gtab, tab_bytes, out, \
                                 ostride, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

// ---- PRSS / utilities ---------------------------------------------------------------------------

template <int L, int KIND, bool SMALL, bool A8, bool SIMPLE>
static cudaError_t prss_tiles_k(const FieldParams& fp, const unsigned char* bytes, size_t subset_stride, int nsub, int d,
                                int chunk_bytes, int bound_bits, const u64* gtab, u32 tab_bytes, u64* out, size_t n,
                                u32 tile_bytes, size_t smem, cudaStream_t st) {
    auto kernel = k_prss_tiles<L, KIND, SMALL, A8, SIMPLE>;
    if (smem > 48u * 1024u) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    const size_t ntiles = (n + MPYC_THREADS - 1) / MPYC_THREADS;
    return launch_kernel(kernel, ntiles * MPYC_THREADS, smem, st, fp, bytes, subset_stride, nsub, d, chunk_bytes, bound_bits,
                         gtab, tab_bytes, out, n, tile_bytes);
}

template <int L>
cudaError_t Launch<L>::prss(const FieldParams& fp, bool small, bool simple, const unsigned char* bytes, size_t subset_stride, int nsub, int d,
                            int chunk_bytes, int bound_bits, const u64* gtab, u32 tab_bytes, u64* out, size_t n,
                            cudaStream_t st) {
    // tiled form (TMA-staged PRF bytes) when the byte streams are 16-byte aligned and two tiles fit in shared memory
    const size_t tile_bytes = ((size_t)MPYC_THREADS * d * chunk_bytes + 15) & ~(size_t)15;
    const size_t smem = ((tab_bytes + 127u) & ~127u) + 2 * tile_bytes;
    const bool aligned = ((reinterpret_cast<uintptr_t>(bytes) | subset_stride) & 15u) == 0;
    const bool padded = subset_stride >= (((size_t)n * d * chunk_bytes + 15) & ~(size_t)15);   // last tile reads whole 16-byte groups
    if (aligned && padded && smem <= 160u * 1024u && n >= MPYC_THREADS && getenv("MPYC_B200_PRSS_UNTILED") == nullptr) {
#define TILES(K, SM, A8, SI) \
    return prss_tiles_k<L, K, SM, A8, SI>(fp, bytes, subset_stride, nsub, d, chunk_bytes, bound_bits, gtab, tab_bytes, out, n, (u32)tile_bytes, smem, st)
#define M(K)                                   \
    if (small && simple) {                     \
        if (chunk_bytes % 8 == 0) TILES(K, true, true, true);   \
        TILES(K, true, false, true);           \
    }                                          \
    if (small) {                               \
        if (chunk_bytes % 8 == 0) TILES(K, true, true, false);  \
        TILES(K, true, false, false);          \
    }                                          \
    if (chunk_bytes % 8 == 0) TILES(K, false, true, false);     \
    TILES(K, false, false, false)
        KIND_SWITCH(fp.kind, M)
#undef M
#undef TILES
    }
#define M(K)                                                                                                            \
    if (small)                                                                                                          \
        return launch_kernel(k_prss_combine<L, K, true>, n, tab_bytes, st, fp, bytes, subset_stride, nsub, d, chunk_bytes, \
                             bound_bits, gtab, tab_bytes, out, n);                                                      \
    return launch_kernel(k_prss_combine<L, K, false>, n, tab_bytes, st, fp, bytes, subset_stride, nsub, d, chunk_bytes,  \
                         bound_bits, gtab, tab_bytes, out, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::fill_random(const FieldParams& fp, u64* out, size_t n, u64 base, cudaStream_t st) {
#define M(K) return launch_kernel(k_fill_random<L, K>, n, 0, st, fp, out, n, base)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::matmul(const FieldParams& fp, const u64* A, const u64* B, u64* C, size_t r, size_t k, size_t c,
                              cudaStream_t st) {
    const size_t col_tiles = (c + MPYC_THREADS - 1) / MPYC_THREADS;
    const int tm = r >= 4 ? 4 : 1;      // rows per thread: 4 when there are enough rows, else 1 (vector-matrix products)
    const size_t tiles = col_tiles * ((r + tm - 1) / tm);
    // split-k when the output alone cannot fill the machine: aim at ~4 CTAs per SM, slices of >= 64 terms
    size_t ksplit = 1;
    const size_t want = (size_t)mpyc_sm_count() * 4;
    if (tiles < want && k >= 256) ksplit = std::min((want + tiles - 1) / tiles, k / 64);
    if (ksplit < 2) ksplit = 1;
    const size_t kslice = std::max<size_t>(((k + ksplit - 1) / ksplit + MPYC_MM_KT - 1) / MPYC_MM_KT * MPYC_MM_KT, MPYC_MM_KT);   // whole shared-memory chunks (k may be 0)
    ksplit = std::max<size_t>((k + kslice - 1) / kslice, 1);
    u64* dst = C;
    u64* part = nullptr;
    if (ksplit > 1) {
        cudaError_t e = cudaMallocAsync(&part, ksplit * r * c * L * sizeof(u64), st);
        if (e != cudaSuccess) return e;
        dst = part;
    }
    cudaError_t e = cudaErrorInvalidValue;
#define M(K)                                                                                                              \
    e = tm == 4 ? launch_kernel(k_matmul<L, K, 4>, tiles * ksplit * MPYC_THREADS, 0, st, fp, A, B, dst, r, k, c, kslice, ksplit) \
                : launch_kernel(k_matmul<L, K, 1>, tiles * ksplit * MPYC_THREADS, 0, st, fp, A, B, dst, r, k, c, kslice, ksplit); \
    break
    switch (fp.kind) {
        case KIND_GENERIC: M(KIND_GENERIC);
        case KIND_PM_ALIGNED: M(KIND_PM_ALIGNED);
        case KIND_PM_SHIFT: M(KIND_PM_SHIFT);
        default: break;
    }
#undef M
    if (e == cudaSuccess && ksplit > 1) e = sum_axis(fp, part, C, 1, ksplit, r * c, nullptr, st);   // the slices' sum
    if (part) cudaFreeAsync(part, st);
    return e;
}

// ---- K6: protocol-local algebra (local.cuh) ---------------------------------------------------

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <int L>
cudaError_t Launch<L>::fma(const FieldParams& fp, bool square, const u64* a, const u64* b, const u64* c, u64* out, size_t n,
                           cudaStream_t st) {
    const bool vec = L != 3 && aligned32(a) && aligned32(c) && aligned32(out) && (square || aligned32(b));
    constexpr int E = VecItem<L>::E;
#define M(K)                                                                                                             \
    if constexpr (L != 3) {                                                                                              \
        if (vec) {                                                                                                       \
            if (square) return launch_kernel(k_fma<L, K, true, true>, (n + E - 1) / E, 0, st, fp, a, b, c, out, n);      \
            return launch_kernel(k_fma<L, K, false, true>, (n + E - 1) / E, 0, st, fp, a, b, c, out, n);                 \
        }                                                                                                                \
    }                                                                                                                    \
    if (square) return launch_kernel(k_fma<L, K, true, false>, n, 0, st, fp, a, b, c, out, n);                           \
    return launch_kernel(k_fma<L, K, false, false>, n, 0, st, fp, a, b, c, out, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::axpb(const FieldParams& fp, const u64* a, const u64* s, const u64* t, u64* out, size_t n, cudaStream_t st) {
    AffineParams ap = {};
    bool unit = s[0] == 1;
    for (int i = 0; i < L; i++) {
        ap.s[i] = s[i];
        ap.t[i] = t[i];
        if (i && s[i]) unit = false;
    }
    const bool vec = L != 3 && aligned32(a) && aligned32(out);
    constexpr int E = VecItem<L>::E;
#define M(K)                                                                                                             \
    if constexpr (L != 3) {                                                                                              \
        if (vec) return launch_kernel(k_axpb<L, K, true>, (n + E - 1) / E, 0, st, fp, ap, (int)unit, a, out, n);         \
    }                                                                                                                    \
    return launch_kernel(k_axpb<L, K, false>, n, 0, st, fp, ap, (int)unit, a, out, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::low_bits(const FieldParams& fp, const u64* a, int nbits, u64* out, size_t n, cudaStream_t st) {
    ScalarParam mask = {};
    for (int i = 0; i < L; i++) {
        const int lo = 64 * i;
        mask.v[i] = nbits >= lo + 64 ? ~0ull : (nbits > lo ? ((1ull << (nbits - lo)) - 1) : 0ull);
    }
    constexpr int E = VecItem<L>::E;
    if constexpr (L != 3) {
        if (aligned32(a) && aligned32(out)) return launch_kernel(k_low_bits<L, true>, (n + E - 1) / E, 0, st, mask, a, out, n);
    }
    return launch_kernel(k_low_bits<L, false>, n, 0, st, mask, a, out, n);
}

template <int L>
cudaError_t Launch<L>::nonzero(const FieldParams& fp, const u64* a, unsigned char* out8, unsigned long long* count, size_t n,
                               cudaStream_t st) {
    constexpr int E = VecItem<L>::E;
    if constexpr (L != 3) {
        if (aligned32(a)) return launch_kernel(k_nonzero<L, true>, (n + E - 1) / E, 0, st, a, out8, count, n);
    }
    return launch_kernel(k_nonzero<L, false>, n, 0, st, a, out8, count, n);
}

template <int L>
cudaError_t Launch<L>::bits_compose(const FieldParams& fp, const u64* bits, u64* out, size_t n, int f, bool descending,
                                    cudaStream_t st) {
    if (L % 2 == 0 && (!aligned16(bits) || !aligned16(out))) return cudaErrorMisalignedAddress;
    if (n == 0) return cudaSuccess;
    const size_t smem = (size_t)ComposeCfg<L>::smem(f);
    // the shared-memory footprint depends on f, so the wave size is computed per launch (not cached per kernel)
#define M(K)                                                                                                        \
    {                                                                                                               \
        auto kernel = k_bits_compose<L, K>;                                                                         \
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ComposeCfg<L>::smem(1 << 20)); \
        if (e != cudaSuccess) return e;                                                                             \
        int occ = 0;                                                                                                \
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, MPYC_THREADS, smem);                        \
        if (e != cudaSuccess) return e;                                                                             \
        const size_t tiles = (n + MPYC_THREADS - 1) / MPYC_THREADS;                                                 \
        const int grid = (int)std::min<size_t>(tiles, (size_t)mpyc_sm_count() * (size_t)std::max(occ, 1));          \
        kernel<<<grid, MPYC_THREADS, smem, st>>>(fp, bits, out, n, f, (int)descending);                             \
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);                                                    \
        return cudaGetLastError();                                                                                  \
    }
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::bits_decompose(const FieldParams& fp, const u64* c, u64* out, size_t ostride, size_t n, int l,
                                      bool descending, cudaStream_t st) {
    constexpr int E = VecItem<L>::E;
    if constexpr (L != 3) {
        if (aligned32(c) && aligned32(out) && (ostride * L) % 4 == 0)
            return launch_kernel(k_bits_decompose<L, true>, (n + E - 1) / E, 0, st, c, out, ostride, n, l, (int)descending);
    }
    return launch_kernel(k_bits_decompose<L, false>, n, 0, st, c, out, ostride, n, l, (int)descending);
}

template <int L>
cudaError_t Launch<L>::conv2d(const FieldParams& fp, const u64* X, const u64* W, const u64* B, u64* Y, int k, int r, int m,
                              int n, int v, int s, cudaStream_t st) {
    const size_t smem = (size_t)r * s * s * 2 * L * sizeof(u32);
    const size_t ptiles = ((size_t)m * n + MPYC_THREADS - 1) / MPYC_THREADS;
    const size_t items = (size_t)k * v * ptiles;
#define M(K)                                                                                                      \
    {                                                                                                             \
        auto kernel = k_conv2d<L, K>;                                                                             \
        if (smem > 48u * 1024u) {                                                                                 \
            cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            if (e != cudaSuccess) return e;                                                                       \
        }                                                                                                         \
        return launch_kernel(kernel, items * MPYC_THREADS, smem, st, fp, X, W, B, Y, k, r, m, n, v, s);           \
    }
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t Launch<L>::transpose(const FieldParams& fp, const u64* in, u64* out, size_t R, size_t C, cudaStream_t st) {
    const size_t tiles = ((R + 31) / 32) * ((C + 31) / 32);
    return launch_kernel(k_transpose<L>, tiles * MPYC_THREADS, 0, st, in, out, R, C);
}


template <int L>
cudaError_t Launch<L>::binop_rows(const FieldParams& fp, int op, bool reflected, const u64* a, const u64* b, u64* out, size_t R,
                                  size_t C, cudaStream_t st) {
    if (L % 2 == 0 && (!aligned16(a) || !aligned16(b) || !aligned16(out))) return cudaErrorMisalignedAddress;
    const size_t total = C;            // a thread per column
#define ROWS_CASE(K, OPC)                                                                                   \
    return reflected ? launch_kernel(k_binop_rows<L, K, OPC, true>, total, 0, st, fp, a, b, out, R, C)      \
                     : launch_kernel(k_binop_rows<L, K, OPC, false>, total, 0, st, fp, a, b, out, R, C)
#define M(K)                                   \
    switch (op) {                              \
        case OP_ADD: ROWS_CASE(K, OP_ADD);     \
        case OP_SUB: ROWS_CASE(K, OP_SUB);     \
        case OP_MUL: ROWS_CASE(K, OP_MUL);     \
        default: return cudaErrorInvalidValue; \
    }
    KIND_SWITCH(fp.kind, M)
#undef M
#undef ROWS_CASE
    return cudaErrorInvalidValue;
}

// ---- K7: sums and running sums along an axis (reduce.cuh) ---------------------------------------

// Split R into S slices of rs rows when the work items of the shape (columns: O*I threads; rows form: O warps) cannot
// fill the machine.  Slices keep >= 64 rows (columns) / >= 1024 elements (rows form), so that each item still has
// enough loads in flight.  The partial sums (S, O, I) are then summed (or scanned) along S by the same launcher.
struct AxisPlan {
    size_t S, rs;
};
static inline AxisPlan axis_plan(size_t O, size_t R, size_t I) {
    const bool cols = I >= 32;
    const size_t sms = (size_t)mpyc_sm_count();
    const size_t items = cols ? O * I : O;
    const size_t want = cols ? sms * 1024 : sms * 16;
    const size_t most = cols ? R / 64 : R * I / 1024;
    size_t S = items < want ? std::min((want + items - 1) / items, most) : 1;
    if (S < 2) return AxisPlan{1, R};
    const size_t rs = (R + S - 1) / S;
    return AxisPlan{(R + rs - 1) / rs, rs};
}

template <int L, int KIND, bool VEC>
static cudaError_t sum_pass(const FieldParams& fp0, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                            const ScalarParam& init, int add_init, cudaStream_t st) {
    FieldParams fp = fp0;
    fp.q32 = rs <= ((size_t)1 << 31) ? 1u : 0u;          // every lazy sum < rs * p <= 2^(k+31)
    if (I >= 32) return launch_kernel(k_sum_cols<L, KIND, VEC>, S * O * I, 0, st, fp, in, out, O, R, I, rs, S, init, add_init);
    return launch_kernel(k_sum_rows<L, KIND, VEC>, S * O * 32, 0, st, fp, in, out, O, R, I, rs, S, init, add_init);
}

template <int L, int KIND, bool VEC>
static cudaError_t scan_pass(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                             const u64* carry, int inc, cudaStream_t st) {
    if (I >= 32) return launch_kernel(k_scan_cols<L, KIND, VEC>, S * O * I, 0, st, fp, in, out, O, R, I, rs, S, carry, inc);
    return launch_kernel(k_scan_rows<L, KIND, VEC>, S * O * 32, 0, st, fp, in, out, O, R, I, rs, S, carry, inc);
}

// the VEC forms (16-byte accesses) need even L and 16-byte aligned arrays; a DeviceArray slice may start at any element
template <int L>
static cudaError_t sum_pass_any(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                                const ScalarParam& init, int add_init, cudaStream_t st) {
    if constexpr (L % 2 == 0) {
        if (aligned16(in) && aligned16(out)) {
#define M(K) return sum_pass<L, K, true>(fp, in, out, O, R, I, S, rs, init, add_init, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return sum_pass<L, K, false>(fp, in, out, O, R, I, S, rs, init, add_init, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
static cudaError_t scan_pass_any(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                                 const u64* carry, int inc, cudaStream_t st) {
    if constexpr (L % 2 == 0) {
        if (aligned16(in) && aligned16(out)) {
#define M(K) return scan_pass<L, K, true>(fp, in, out, O, R, I, S, rs, carry, inc, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return scan_pass<L, K, false>(fp, in, out, O, R, I, S, rs, carry, inc, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
static cudaError_t sum_axis_impl(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I,
                                 const ScalarParam& init, int add_init, cudaStream_t st) {
    if (O * I == 0) return cudaSuccess;
    const AxisPlan pl = axis_plan(O, R, I);
    if (pl.S == 1) return sum_pass_any<L>(fp, in, out, O, R, I, 1, R, init, add_init, st);
    u64* part = nullptr;                                 // (S, O, I) slice sums, stream-ordered scratch
    cudaError_t e = cudaMallocAsync(&part, pl.S * O * I * L * sizeof(u64), st);
    if (e != cudaSuccess) return e;
    e = sum_pass_any<L>(fp, in, part, O, R, I, pl.S, pl.rs, init, 0, st);
    if (e == cudaSuccess) e = sum_axis_impl<L>(fp, part, out, 1, pl.S, O * I, init, add_init, st);
    cudaFreeAsync(part, st);
    return e;
}

// Reduce-then-scan when R is split: slice sums (S, O, I), their inclusive scan along S, then every slice is scanned
// again from its carry-in.  No CTA waits on another (three launches in stream order); the input is read twice.
template <int L>
static cudaError_t scan_axis_impl(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, int inc,
                                  cudaStream_t st) {
    if (O * I == 0) return cudaSuccess;
    const AxisPlan pl = axis_plan(O, R, I);
    if (pl.S == 1) return scan_pass_any<L>(fp, in, out, O, R, I, 1, R, nullptr, inc, st);
    const size_t count = pl.S * O * I;
    u64* part = nullptr;                                 // slice sums, then their running sums
    cudaError_t e = cudaMallocAsync(&part, 2 * count * L * sizeof(u64), st);
    if (e != cudaSuccess) return e;
    const ScalarParam zero = {};
    e = sum_pass_any<L>(fp, in, part, O, R, I, pl.S, pl.rs, zero, 0, st);
    if (e == cudaSuccess) e = scan_axis_impl<L>(fp, part, part + count * L, 1, pl.S, O * I, 0, st);
    if (e == cudaSuccess) e = scan_pass_any<L>(fp, in, out, O, R, I, pl.S, pl.rs, part + count * L, inc, st);
    cudaFreeAsync(part, st);
    return e;
}

template <int L>
cudaError_t Launch<L>::sum_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, const u64* init,
                                cudaStream_t st) {
    ScalarParam sp = {};
    if (init)
        for (int i = 0; i < L; i++) sp.v[i] = init[i];
    return sum_axis_impl<L>(fp, in, out, O, R, I, sp, init ? 1 : 0, st);
}

template <int L>
cudaError_t Launch<L>::scan_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool inc,
                                 cudaStream_t st) {
    return scan_axis_impl<L>(fp, in, out, O, R, I, inc ? 1 : 0, st);
}

// ---- K8: broadcast arithmetic on views (layout.cuh) ---------------------------------------------

template <int L>
cudaError_t Launch<L>::binop_view(const FieldParams& fp, int op, const BinopPlan& pl, const u64* a, const u64* b, u64* out,
                                  cudaStream_t st) {
    size_t n = 1;
    for (int k = 0; k < pl.rank; k++) n *= (size_t)pl.ext[k];
#define VIEW_CASE(K, OPC) return launch_kernel(k_binop_view<L, K, OPC>, n, 0, st, fp, pl, a, b, out, n)
#define M(K)                                   \
    switch (op) {                              \
        case OP_ADD: VIEW_CASE(K, OP_ADD);     \
        case OP_SUB: VIEW_CASE(K, OP_SUB);     \
        case OP_MUL: VIEW_CASE(K, OP_MUL);     \
        default: return cudaErrorInvalidValue; \
    }
    KIND_SWITCH(fp.kind, M)
#undef M
#undef VIEW_CASE
    return cudaErrorInvalidValue;
}
