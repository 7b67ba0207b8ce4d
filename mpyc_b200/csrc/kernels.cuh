// sm_90a kernels for the GF(p) Shamir hot path.  All kernels are persistent grid-stride
// streamers: one CTA wave sized from the SM count, 128-bit global loads/stores on the limb
// arrays (LDG.E.128 / STG.E.128; read-once data bypasses L1 allocation), per-call constant tables
// (Vandermonde / Lagrange, a few hundred bytes) staged global -> shared memory once per CTA with a
// TMA bulk copy (cp.async.bulk + mbarrier; UBLKCP in SASS); K4 also stages its PRF byte tiles that
// way, double-buffered.  Integer modular work: no tensor cores.
//
//   K1   k_binop                                finfields.py:1056-1124,1189-1192
//   K1b  k_pow (pow / sqrt / is_sqr), k_inv_batch (Montgomery-trick inverse)   finfields.py:1408-1470
//   K1c  k_matmul                               finfields.py:1126-1146
//   K2   k_split_tiled (aligned rows; shares leave through shared memory as TMA bulk stores), k_split (small / full
//        tables; unaligned rows and 3-limb fields), k_split_gen (ChaCha20 coefficients, strided or per-row destinations),
//        k_split_dyn (any t)                    thresha.py:47-64
//   K3   k_recombine_tiled (aligned rows; small / full lambda), k_recombine (unaligned rows and 3-limb fields)
//                                               thresha.py:119-132
//   K4   k_prss_tiles, k_prss_combine           thresha.py:163-173,201-217
//   K7   k_sum_cols / k_sum_rows, k_scan_cols / k_scan_rows (reduce.cuh)   np.sum / np.cumsum along any axis
//   K8   k_copy_gather, k_copy_permute, k_binop_view (layout.cuh)   strided views, joins, broadcast arithmetic
//   K11  k_inv_batch<NUM> (ff_div), k_select (select.cuh)   division and np.where       finfields.py:1199-1225
//   K12  k_powexp_fixed, k_powexp_elem (powexp.cuh)   per-element exponents   finfields.py:1409-1414, gmpy.py:288-290
//   K13  k_prod_*, k_cumprod_*, k_allany_* (prod.cuh)   np.prod / np.cumprod / np.all / np.any along any axis
#pragma once
#include "ff_arith.cuh"

#define MPYC_MAX_POINTS 64
#define MPYC_THREADS 256
// launch bounds: asking ptxas for >= 1 resident CTA lets it use the registers it wants (fewer moves,
// measured +1..8 % on K2); -DMPYC_LB_PLAIN restores the default heuristic (experiments)
#ifdef MPYC_LB_PLAIN
#define MPYC_LB __launch_bounds__(MPYC_THREADS)
#else
#define MPYC_LB __launch_bounds__(MPYC_THREADS, 1)
#endif

struct RowPtrs {
    const u64* p[MPYC_MAX_POINTS];
};

// Destination of the m share rows of K2 (a template parameter of the split kernels, so that the strided form costs
// nothing): StridedDst = base + i*stride (limbs); RowsDst = one explicit pointer per party -- how a dealer writes each
// recipient's row straight into that recipient GPU's memory (peer pointers over NVLink,
// mpyc_b200.exchange.PeerReshare) instead of into a local matrix that is copied afterwards.
#define MPYC_MAX_SHARE_ROWS 32
struct StridedDst {
    u64* base;
    size_t stride;
    __device__ __forceinline__ u64* row(int i) const { return base + (size_t)i * stride; }
};
struct RowsDst {
    u64* rows[MPYC_MAX_SHARE_ROWS];
    __device__ __forceinline__ u64* row(int i) const { return rows[i]; }
};

struct ScalarParam {
    u64 v[4];
};

struct ExpParams {
    u64 e[8];
    int ebits;
};

// ---------------------------------------------------------------------------------------
// memory helpers
// ---------------------------------------------------------------------------------------

__device__ __forceinline__ void ldg_v4(u32* v, const u64* p) {   // 16 bytes = two 64-bit limbs
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
        : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p));
}
__device__ __forceinline__ void ldg_v2(u32* v, const u64* p) {   // one 64-bit limb
    asm("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(v[0]), "=r"(v[1]) : "l"(p));
}
__device__ __forceinline__ void stg_v4(u64* p, const u32* v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}
__device__ __forceinline__ void stg_v2(u64* p, const u32* v) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v[0]), "r"(v[1]) : "memory");
}

// load / store NL 64-bit limbs starting at p, as 2*NL 32-bit registers.  VEC: 128-bit accesses, the widest
// global access sm_90 has (LDG.E.128 / STG.E.128), in pairs covering 32-byte groups (p 32-byte aligned, NL a
// multiple of 4); else one limb at a time.
template <int NL, bool VEC>
__device__ __forceinline__ void load_limbs(u32* v, const u64* p) {
    if constexpr (VEC) {
        static_assert(NL % 4 == 0, "vector path moves 32-byte groups");
#pragma unroll
        for (int q = 0; q < NL / 2; q++) ldg_v4(v + 4 * q, p + 2 * q);
    } else {
#pragma unroll
        for (int q = 0; q < NL; q++) ldg_v2(v + 2 * q, p + q);
    }
}
template <int NL, bool VEC>
__device__ __forceinline__ void store_limbs(u64* p, const u32* v) {
    if constexpr (VEC) {
#pragma unroll
        for (int q = 0; q < NL / 2; q++) stg_v4(p + 2 * q, v + 4 * q);
    } else {
#pragma unroll
        for (int q = 0; q < NL; q++) stg_v2(p + q, v + 2 * q);
    }
}

// elements per vector item: the smallest E with E*L a multiple of 4 limbs (32 bytes)
template <int L>
struct VecItem {
    static constexpr int E = (L == 4) ? 1 : (L == 2 ? 2 : 4);
};

// ---------------------------------------------------------------------------------------
// TMA bulk copy of a small table into shared memory (whole CTA waits on the mbarrier)
// ---------------------------------------------------------------------------------------

__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }

// bytes must be a multiple of 16; src and dst 16-byte aligned.  Call from all threads.
__device__ __forceinline__ void tma_stage_table(void* smem_dst, const void* gmem_src, u32 bytes, u64* mbar) {
    if (bytes == 0) return;
    const u32 bar = smem_u32(mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(smem_dst)),
            "l"(gmem_src), "r"(bytes), "r"(bar)
            : "memory");
    }
    u32 done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar)
            : "memory");
    }
}

// ---------------------------------------------------------------------------------------
// K1: elementwise
// ---------------------------------------------------------------------------------------

enum { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_NEG = 3 };

template <int L, int KIND, int OP>
__device__ __forceinline__ void apply_op(u32* r, const u32* a, const u32* b, const FieldParams& f) {
    if constexpr (OP == OP_ADD) Fp<L, KIND>::add(r, a, b, f);
    else if constexpr (OP == OP_SUB) Fp<L, KIND>::sub(r, a, b, f);
    else if constexpr (OP == OP_MUL) Fp<L, KIND>::mul(r, a, b, f);
    else Fp<L, KIND>::neg(r, a, f);
}

// SCALAR: b is one broadcast element (canonical) in sc; NEG ignores b.
// U items are processed together: all loads are issued before the first multiply.
template <int L, int KIND, int OP, bool SCALAR, int E, bool VEC, int U>
__device__ __forceinline__ void binop_items(const FieldParams& f, const u64* a, const u64* b, const u32* sc,
                                            u64* out, size_t item0, size_t item_step) {
    constexpr int N = 2 * L;
    u32 x[U][E * N], y[U][E * N];
#pragma unroll
    for (int u = 0; u < U; u++) {
        const size_t off = (item0 + u * item_step) * (size_t)(E * L);
        load_limbs<E * L, VEC>(x[u], a + off);
        if constexpr (!SCALAR && OP != OP_NEG) load_limbs<E * L, VEC>(y[u], b + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
        u32 r[E * N];
#pragma unroll
        for (int e = 0; e < E; e++) {
            if constexpr (SCALAR) apply_op<L, KIND, OP>(r + e * N, x[u] + e * N, sc, f);
            else apply_op<L, KIND, OP>(r + e * N, x[u] + e * N, y[u] + e * N, f);
        }
        store_limbs<E * L, VEC>(out + (item0 + u * item_step) * (size_t)(E * L), r);
    }
}

template <int L, int KIND, int OP, bool SCALAR, bool VEC>
__global__ void MPYC_LB
k_binop(FieldParams f, const u64* __restrict__ a, const u64* __restrict__ b, ScalarParam scal,
        u64* __restrict__ out, size_t n) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
#ifndef MPYC_BINOP_U
#define MPYC_BINOP_U 1
#endif
    constexpr int U = MPYC_BINOP_U;   // items in flight per thread
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    u32 sc[2 * L];
#pragma unroll
    for (int i = 0; i < 2 * L; i++) sc[i] = as32(scal.v)[i];
    size_t it = tid;
    for (; it + (U - 1) * nth < n_items; it += U * nth)
        binop_items<L, KIND, OP, SCALAR, E, VEC, U>(f, a, b, sc, out, it, nth);
    for (; it < n_items; it += nth) binop_items<L, KIND, OP, SCALAR, E, VEC, 1>(f, a, b, sc, out, it, nth);
    if constexpr (E > 1) {   // leftover elements
        for (size_t h = n_items * E + tid; h < n; h += nth)
            binop_items<L, KIND, OP, SCALAR, 1, false, 1>(f, a, b, sc, out, h, nth);
    }
}

// ---------------------------------------------------------------------------------------
// K1b: out = a^e (uniform public exponent).  MODE 0: pow; 1: is_sqr (u8 out, e = (p-1)/2);
// zero_flag (may be null): set to 1 if any input element is zero (inverse / inverse sqrt).
// ---------------------------------------------------------------------------------------

template <int L, int KIND, int MODE>
__global__ void MPYC_LB
k_pow(FieldParams f, ExpParams ex, const u64* __restrict__ a, u64* __restrict__ out, unsigned char* __restrict__ out_u8,
      int* zero_flag, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        constexpr int N = 2 * L;
        u32 x[N], r[N];
        load_limbs<L, false>(x, a + h * L);
        if (zero_flag != nullptr && is_zero_n<N>(x)) *zero_flag = 1;
        Fp<L, KIND>::to_dom(x, x, f);
        Fp<L, KIND>::dpow_uniform(r, x, ex.e, ex.ebits, f);
        Fp<L, KIND>::from_dom(r, r, f);
        if constexpr (MODE == 0) {
            store_limbs<L, false>(out + h * L, r);
        } else {
            // legendre(a, p) == -1  <=>  a^((p-1)/2) == p - 1
            u32 pm1[N];
            copy_n<N>(pm1, as32(f.p));
            pm1[0] -= 1;   // p odd
            u32 d = 0;
#pragma unroll
            for (int i = 0; i < N; i++) d |= r[i] ^ pm1[i];
            out_u8[h] = d != 0;
        }
    }
}

// ---------------------------------------------------------------------------------------
// K1b': batched inverse (PrimeFieldArray._reciprocal, finfields.py:1416-1422) with Montgomery's trick:
// thread `tid` of T owns the B elements tid, tid+T, ..., tid+(B-1)T (coalesced across the warp), writes
// their running products into `out`, inverts the last one with ONE Fermat exponentiation and walks back:
//   inv(x_b) = inv(x_0..x_b) * (x_0..x_{b-1}),   inv(x_0..x_{b-1}) = inv(x_0..x_b) * x_b
// i.e. 3 multiplications per element + 1/B of an exponentiation (~1.5 bits(p) multiplications) instead of
// a whole one.  Zeros are skipped in the products (the result for them is 0) and reported through
// zero_flag (the reference raises ZeroDivisionError, gmpy.py:192-213).  a and out must not alias.
// NUM (K11, ff_div): the backward walk multiplies each inverse by num[h] before storing it, so that
// out[h] = num[h] * a[h]^-1 in the same pass -- one more load and one more multiplication per element.  num may
// alias a but not out (the forward pass leaves prefix products in out).  Without NUM, num is unused.
// ---------------------------------------------------------------------------------------

template <int L>
__device__ __forceinline__ void load_plain(u32* v, const u64* p) {   // coherent loads: `out` is re-read
#pragma unroll
    for (int q = 0; q < L; q++) {
        const u64 w = p[q];
        v[2 * q] = (u32)w;
        v[2 * q + 1] = (u32)(w >> 32);
    }
}

template <int L, int KIND, bool NUM = false>
__global__ void MPYC_LB
k_inv_batch(FieldParams f, ExpParams ex, const u64* __restrict__ a, u64* out, int* zero_flag, size_t n, size_t T, int B,
            const u64* __restrict__ num) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x; tid < T; tid += nth) {
        u32 acc[N], x[N];
        zero_n<N>(acc);
        acc[0] = 1;
        int cnt = 0;
        bool saw_zero = false;
        for (int b = 0; b < B; b++) {
            const size_t h = tid + (size_t)b * T;
            if (h >= n) break;
            load_limbs<L, false>(x, a + h * L);
            if (is_zero_n<N>(x)) {
                saw_zero = true;
                x[0] = 1;
            }
            F::mul(acc, acc, x, f);
            store_limbs<L, false>(out + h * L, acc);
            cnt = b + 1;
        }
        if (saw_zero) *zero_flag = 1;
        u32 inv[N];
        F::to_dom(inv, acc, f);
        F::dpow_uniform(inv, inv, ex.e, ex.ebits, f);
        F::from_dom(inv, inv, f);
        for (int b = cnt - 1; b >= 0; b--) {
            const size_t h = tid + (size_t)b * T;
            u32 prev[N], r[N];
            load_limbs<L, false>(x, a + h * L);
            const bool z = is_zero_n<N>(x);
            if (z) x[0] = 1;
            if (b > 0) {
                load_plain<L>(prev, out + (h - T) * L);
                F::mul(r, inv, prev, f);
            } else {
                copy_n<N>(r, inv);
            }
            F::mul(inv, inv, x, f);
            if constexpr (NUM) {
                u32 y[N];
                load_limbs<L, false>(y, num + h * L);
                F::mul(r, r, y, f);
            }
            if (z) zero_n<N>(r);
            store_limbs<L, false>(out + h * L, r);
        }
    }
}

// ---------------------------------------------------------------------------------------
// K2: Shamir share generation.  M[0] = secrets, M[j] = coefficient row j-1.
//   small: table entry (i, j) is the plain integer (i+1)^j < 2^59:
//          acc (L+1 limbs) = M[0] + sum_j M[j] * v  -> one fold (pseudo-Mersenne) or one 64-bit-quotient
//          Barrett step (generic fields) per share
//   full : table entry is a full field element in table form; acc (2L+1 limbs), one reduction
// ---------------------------------------------------------------------------------------

// items in flight per thread (split is fastest without unrolling); override with -D for experiments
#ifndef MPYC_SPLIT_U
#define MPYC_SPLIT_U 1
#endif
// shares computed per trip of the party loop of split_compute: two independent share evaluations in flight, one
// share's carry chains issuing while the other's wait.  Neutral on an H100 SXM at 400 W (DESIGN.md section 5)
#ifndef MPYC_SPLIT_MU
#define MPYC_SPLIT_MU ((L == 1 || KIND == KIND_GENERIC) ? 1 : 2)
#endif

// Tiled K2 and K3 (k_split_tiled, k_recombine_tiled): a CTA owns a tile of MPYC_THREADS x 32 bytes of every row (8 KB).  A thread's item is two
// 16-byte chunks at tile limb offsets o and o + H: for L <= 2 the chunks tid and tid + MPYC_THREADS, so that a warp
// load covers 512 contiguous bytes; for L = 4 the two halves of element tid.
#define MPYC_TILE_LIMBS (MPYC_THREADS * 4)
template <int L>
struct TileItem {
    static constexpr int STEP = (L == 4) ? 4 : 2;                      // o = STEP * tid
    static constexpr int H = (L == 4) ? 2 : 2 * MPYC_THREADS;          // limbs from the first chunk to the second
};
// share rows written a tile item at a time; SMEM: the tile's stage in shared memory (stride MPYC_TILE_LIMBS), each row
// at the same offsets as in its global row
template <int L, bool SMEM>
struct TileDst {
    u64* base;
    size_t stride;
    __device__ __forceinline__ u64* row(int i) const { return base + (size_t)i * stride; }
};

template <int L>
__device__ __forceinline__ void load_tile_item(u32* v, const u64* p) {
    ldg_v4(v, p);
    ldg_v4(v + 4, p + TileItem<L>::H);
}

template <int NL, bool VEC, class DST>
__device__ __forceinline__ void store_share(const DST& dst, int i, size_t limb_off, const u32* r) {
    store_limbs<NL, VEC>(dst.row(i) + limb_off, r);
}
template <int NL, bool VEC, int L, bool SMEM>
__device__ __forceinline__ void store_share(const TileDst<L, SMEM>& dst, int i, size_t limb_off, const u32* r) {
    static_assert(NL == 4, "a tile item is two 16-byte chunks");
    u64* p = dst.row(i) + limb_off;
    if constexpr (SMEM) {
        *reinterpret_cast<uint4*>(p) = make_uint4(r[0], r[1], r[2], r[3]);
        *reinterpret_cast<uint4*>(p + TileItem<L>::H) = make_uint4(r[4], r[5], r[6], r[7]);
    } else {
        stg_v4(p, r);
        stg_v4(p + TileItem<L>::H, r + 4);
    }
}

// shares of one item (E elements) from its t+1 polynomial coefficient rows held in registers
template <int L, int KIND, int TP1, bool FULL, int E, bool VEC, class DST>
__device__ __forceinline__ void split_compute(const FieldParams& f, const u32 (*M)[E * 2 * L], const DST& dst,
                                              int m, const u64* tab, size_t limb_off) {
    constexpr int N = 2 * L;
    typedef Fp<L, KIND> F;
    constexpr int MU = MPYC_SPLIT_MU;   // shares computed per trip of the party loop
#pragma unroll MU
    for (int i = 0; i < m; i++) {
        u32 r[E * N];
#pragma unroll
        for (int e = 0; e < E; e++) {
            if constexpr (FULL) {
                u32 acc[F::WACC];
                zero_n<F::WACC>(acc);
#pragma unroll
                for (int j = 0; j < TP1; j++) F::mac(acc, M[j] + e * N, as32(tab + (size_t)(i * TP1 + j) * L));
                F::finish(r + e * N, acc, f);
            } else {
                u32 acc[F::WSM];
                copy_n<N>(acc, M[0] + e * N);
                acc[N] = acc[N + 1] = 0;
#pragma unroll
                for (int j = 1; j < TP1; j++) F::mac_const(acc, M[j] + e * N, tab[i * TP1 + j]);
                if constexpr (TP1 > 1) F::reduce_small_q32(r + e * N, acc, f);
                else copy_n<N>(r + e * N, acc);
            }
        }
        store_share<E * L, VEC>(dst, i, limb_off, r);
    }
}

// U items (item u at limb offset limb_off + u*limb_step) are processed together: every load is
// issued before the first multiply so that U*(t+1) 16-byte requests per thread are in flight.
template <int L, int KIND, int TP1, bool FULL, int E, bool VEC, int U>
__device__ __forceinline__ void split_items(const FieldParams& f, const u64* secrets, const u64* coeffs,
                                            size_t cstride, const StridedDst& dst, int m, const u64* tab,
                                            size_t limb_off, size_t limb_step) {
    constexpr int N = 2 * L;
    u32 M[U][TP1][E * N];
#pragma unroll
    for (int u = 0; u < U; u++) {
        const size_t off = limb_off + u * limb_step;
        load_limbs<E * L, VEC>(M[u][0], secrets + off);
#pragma unroll
        for (int j = 1; j < TP1; j++) load_limbs<E * L, VEC>(M[u][j], coeffs + (size_t)(j - 1) * cstride + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++)
        split_compute<L, KIND, TP1, FULL, E, VEC>(f, M[u], dst, m, tab, limb_off + u * limb_step);
}

#ifndef MPYC_SPLIT_PREFETCH
// software-pipelined main loop of k_split for fields of at most this many limbs (0 = off; neutral on an H100 SXM)
#define MPYC_SPLIT_PREFETCH 1
#endif
#ifndef MPYC_SPLIT_MINB
#define MPYC_SPLIT_MINB 1   // min resident CTAs per SM requested from ptxas for k_split (register cap)
#endif
#ifndef MPYC_SPLIT_MINB1
#define MPYC_SPLIT_MINB1 1  // the same for 1-limb fields with t+1 <= 2 (ns64: 52 registers miss the 5th CTA per SM by one)
#endif
template <int L, int KIND, int TP1, bool FULL>
__global__ void __launch_bounds__(MPYC_THREADS, (L == 1 && TP1 <= 2 && !FULL) ? MPYC_SPLIT_MINB1 : MPYC_SPLIT_MINB)
k_split(FieldParams f, const u64* __restrict__ secrets, const u64* __restrict__ coeffs, size_t cstride,
        u64* __restrict__ shares, size_t sstride, size_t n, int m, const u64* __restrict__ gtab, u32 tab_bytes) {
    const StridedDst dst = {shares, sstride};
    extern __shared__ __align__(16) u64 stab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(stab, gtab, tab_bytes, &mbar);
    constexpr int U = (TP1 * L <= 8) ? MPYC_SPLIT_U : 1;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (L <= MPYC_SPLIT_PREFETCH && !FULL && TP1 <= 3) {
        // software pipeline for the narrow fields (few bytes per item, latency-bound at one item per trip): the t+1
        // input vectors of item it+nth are requested before the shares of item it are computed and stored
        constexpr int N = 2 * L;
        u32 cur[TP1][N], nxt[TP1][N];
        auto fetch = [&](u32 (*M)[N], size_t item) {
            const size_t off = item * (size_t)L;
            load_limbs<L, false>(M[0], secrets + off);
#pragma unroll
            for (int j = 1; j < TP1; j++) load_limbs<L, false>(M[j], coeffs + (size_t)(j - 1) * cstride + off);
        };
        if (it < n) fetch(cur, it);
        for (; it < n; it += nth) {
            const bool more = it + nth < n;
            if (more) fetch(nxt, it + nth);
            split_compute<L, KIND, TP1, FULL, 1, false>(f, cur, dst, m, stab, it * (size_t)L);
            if (more) {
#pragma unroll
                for (int j = 0; j < TP1; j++)
#pragma unroll
                    for (int q = 0; q < N; q++) cur[j][q] = nxt[j][q];
            }
        }
    } else {
        for (; it + (U - 1) * nth < n; it += U * nth)
            split_items<L, KIND, TP1, FULL, 1, false, U>(f, secrets, coeffs, cstride, dst, m, stab, it * (size_t)L,
                                                         nth * (size_t)L);
        for (; it < n; it += nth)
            split_items<L, KIND, TP1, FULL, 1, false, 1>(f, secrets, coeffs, cstride, dst, m, stab, it * (size_t)L, 0);
    }
}

// K2 for 32-byte aligned rows of 1-, 2- and 4-limb fields, one tile (TileItem) per CTA and trip.  STAGE: the shares are
// written to a stage of m x 8 KB in shared memory at their tile offsets and leave as one TMA bulk store per row
// (cp.async.bulk, UBLKCP in SASS); otherwise (m too large for the stage) every thread stores its two chunks itself
// (coalesced for L <= 2).  Whole sectors instead of a 32-byte item per thread, which used half of every sector a warp
// access touched (a 3 in / 5 out stream probe: 2235 -> 2822 GB/s on an H100 SXM at 400 W, DESIGN.md section 5).
// For t+1 <= 4 the input chunks of the thread's next tile are requested before the current tile's shares are computed.
// smem layout: [table (tab_bytes rounded up to 128)] [stage: m x MPYC_TILE_LIMBS limbs]
template <int L, int KIND, int TP1, bool FULL, bool STAGE>
__global__ void MPYC_LB
k_split_tiled(FieldParams f, const u64* __restrict__ secrets, const u64* __restrict__ coeffs, size_t cstride,
              u64* __restrict__ shares, size_t sstride, size_t n, int m, const u64* __restrict__ gtab, u32 tab_bytes) {
    extern __shared__ __align__(128) u64 smem[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(smem, gtab, tab_bytes, &mbar);
    constexpr int E = VecItem<L>::E, N = 2 * L;
    constexpr int TE = MPYC_TILE_LIMBS / L;   // elements per tile
    const size_t ntiles = n / TE;
    const u32 o = threadIdx.x * TileItem<L>::STEP;
    u64* const stage = smem + ((tab_bytes + 127u) & ~127u) / sizeof(u64);
    u32 cur[TP1][E * N], nxt[TP1][E * N];
    auto fetch = [&](u32 (*M)[E * N], size_t tile) {
        const size_t off = tile * MPYC_TILE_LIMBS + o;
        load_tile_item<L>(M[0], secrets + off);
#pragma unroll
        for (int j = 1; j < TP1; j++) load_tile_item<L>(M[j], coeffs + (size_t)(j - 1) * cstride + off);
    };
    // more coefficient rows held for the next tile cost more occupancy than they hide (64-bit m = 17, t = 8: 172 registers)
    constexpr bool PREFETCH = TP1 <= 4;
    size_t tile = blockIdx.x;
    if (PREFETCH && tile < ntiles) fetch(cur, tile);
    for (; tile < ntiles; tile += gridDim.x) {
        const bool more = PREFETCH && tile + gridDim.x < ntiles;
        if constexpr (PREFETCH) {
            if (more) fetch(nxt, tile + gridDim.x);
        } else {
            fetch(cur, tile);
        }
        if constexpr (STAGE) {
            // the bulk stores of the previous tile have finished reading the stage (bulk groups belong to thread 0)
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            __syncthreads();
            split_compute<L, KIND, TP1, FULL, E, true>(f, cur, TileDst<L, true>{stage, MPYC_TILE_LIMBS}, m, smem, o);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // make the stage visible to the async proxy
            __syncthreads();
            if (threadIdx.x == 0) {
                // evict-first: the share rows are not read again by this step, and leaving them in L2 as the most
                // recent lines slowed the recombination (K3) that follows by up to 10 % (DESIGN.md section 5)
                u64 pol;
                asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
                for (int i = 0; i < m; i++)
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(
                                     shares + (size_t)i * sstride + tile * MPYC_TILE_LIMBS),
                                 "r"(smem_u32(stage + (size_t)i * MPYC_TILE_LIMBS)), "n"(MPYC_TILE_LIMBS * 8), "l"(pol)
                                 : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        } else {
            split_compute<L, KIND, TP1, FULL, E, true>(f, cur, TileDst<L, false>{shares, sstride}, m, smem,
                                                       tile * MPYC_TILE_LIMBS + o);
        }
        if (more) {
#pragma unroll
            for (int j = 0; j < TP1; j++)
#pragma unroll
                for (int q = 0; q < E * N; q++) cur[j][q] = nxt[j][q];
        }
    }
    if constexpr (STAGE) {
        if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // before the stage goes away
    }
    // partial last tile: one element per thread, stored directly
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = ntiles * TE + (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth)
        split_items<L, KIND, TP1, FULL, 1, false, 1>(f, secrets, coeffs, cstride, StridedDst{shares, sstride}, m, smem,
                                                     h * (size_t)L, 0);
}

// ---- generate mode: coefficients come from a ChaCha20 keystream and never touch memory ----------
// (the role of secrets.randbelow in thresha.py:58-60; 64 bits wider than p, then reduced: bias < 2^-64)

struct ChaChaKey {
    u32 k[8];
    u32 nonce[2];
};

#ifndef MPYC_CHACHA_ROUNDS
#define MPYC_CHACHA_ROUNDS 20
#endif

__device__ __forceinline__ void chacha_qr(u32& a, u32& b, u32& c, u32& d) {
    a += b; d ^= a; d = __funnelshift_l(d, d, 16);
    c += d; b ^= c; b = __funnelshift_l(b, b, 12);
    a += b; d ^= a; d = __funnelshift_l(d, d, 8);
    c += d; b ^= c; b = __funnelshift_l(b, b, 7);
}

__device__ __forceinline__ void chacha_block(u32* out, const ChaChaKey& key, u64 counter) {
    u32 x[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u,
                 key.k[0], key.k[1], key.k[2], key.k[3], key.k[4], key.k[5], key.k[6], key.k[7],
                 (u32)counter, (u32)(counter >> 32), key.nonce[0], key.nonce[1]};
    u32 w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = x[i];
#pragma unroll
    for (int r = 0; r < MPYC_CHACHA_ROUNDS; r += 2) {
        chacha_qr(w[0], w[4], w[8], w[12]);
        chacha_qr(w[1], w[5], w[9], w[13]);
        chacha_qr(w[2], w[6], w[10], w[14]);
        chacha_qr(w[3], w[7], w[11], w[15]);
        chacha_qr(w[0], w[5], w[10], w[15]);
        chacha_qr(w[1], w[6], w[11], w[12]);
        chacha_qr(w[2], w[7], w[8], w[13]);
        chacha_qr(w[3], w[4], w[9], w[14]);
    }
#pragma unroll
    for (int i = 0; i < 16; i++) out[i] = w[i] + x[i];
}

// coefficient slots per 16-word block: each coefficient takes N+2 words (rounded up to a power of two)
template <int L>
struct GenLayout {
    static constexpr int SLOT = (2 * L + 2 <= 4) ? 4 : (2 * L + 2 <= 8 ? 8 : 16);
    static constexpr int PER_BLOCK = 16 / SLOT;
};

template <int L, int KIND, int TP1, bool FULL, int E, bool VEC, class DST>
__device__ __forceinline__ void split_gen_item(const FieldParams& f, const ChaChaKey& key, u64 counter0,
                                               const u64* secrets, const DST& dst, int m,
                                               const u64* tab, size_t limb_off) {
    constexpr int N = 2 * L;
    constexpr int NC = (TP1 - 1) * E;   // coefficients of this item
    u32 M[TP1][E * N];
    load_limbs<E * L, VEC>(M[0], secrets + limb_off);
    u32 blk[16];
#pragma unroll
    for (int c = 0; c < NC; c++) {
        if (c % GenLayout<L>::PER_BLOCK == 0) chacha_block(blk, key, counter0 + c / GenLayout<L>::PER_BLOCK);
        u32 x[N + 2];
#pragma unroll
        for (int w = 0; w < N + 2; w++) x[w] = blk[(c % GenLayout<L>::PER_BLOCK) * GenLayout<L>::SLOT + w];
        // keep bits(p)+64 bits so that x < 2^64 p (precondition of reduce_small)
        const u32 keep = f.k + 64;
#pragma unroll
        for (int w = 0; w < N + 2; w++) {
            const u32 lo = 32u * w;
            if (lo >= keep) x[w] = 0;
            else if (lo + 32 > keep) x[w] &= (1u << (keep - lo)) - 1;
        }
        const int j = 1 + c / E, e = c % E;
        Fp<L, KIND>::reduce_small(M[j] + e * N, x, f);
    }
    split_compute<L, KIND, TP1, FULL, E, VEC>(f, M, dst, m, tab, limb_off);
}

template <int L, int KIND, int TP1, bool FULL, bool VEC, class DST>
__global__ void MPYC_LB
k_split_gen(FieldParams f, ChaChaKey key, const u64* __restrict__ secrets, DST dst,
            size_t n, int m, const u64* __restrict__ gtab, u32 tab_bytes) {
    extern __shared__ __align__(16) u64 stab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(stab, gtab, tab_bytes, &mbar);
    constexpr int E = VEC ? VecItem<L>::E : 1;
    constexpr int BPI = ((TP1 - 1) * E + GenLayout<L>::PER_BLOCK - 1) / GenLayout<L>::PER_BLOCK;   // blocks per item
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    for (size_t it = tid; it < n_items; it += nth)
        split_gen_item<L, KIND, TP1, FULL, E, VEC>(f, key, (u64)it * BPI, secrets, dst, m, stab,
                                                   it * (size_t)(E * L));
    if constexpr (E > 1) {
        ChaChaKey tail = key;
        tail.nonce[1] ^= 0x80000000u;   // disjoint keystream for the scalar tail
        for (size_t h = n_items * E + tid; h < n; h += nth)
            split_gen_item<L, KIND, TP1, FULL, 1, false>(f, tail, (u64)h * BPI, secrets, dst, m, stab,
                                                         h * (size_t)L);
    }
}

// any t: streams the t+1 input rows per output row (re-reads hit L1/L2); full tables
template <int L, int KIND>
__global__ void MPYC_LB
k_split_dyn(FieldParams f, const u64* __restrict__ secrets, const u64* __restrict__ coeffs, size_t cstride,
            u64* __restrict__ shares, size_t sstride, size_t n, int m, int tp1, const u64* __restrict__ gtab) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        for (int i = 0; i < m; i++) {
            typedef Fp<L, KIND> F;
            u32 acc[F::WACC];
            zero_n<F::WACC>(acc);
            for (int j = 0; j < tp1; j++) {
                u32 x[2 * L], w[2 * L];
                const u64* src = j == 0 ? secrets + h * L : coeffs + (size_t)(j - 1) * cstride + h * L;
#pragma unroll
                for (int l = 0; l < L; l++) {
                    set64(x, l, src[l]);
                    set64(w, l, gtab[(size_t)(i * tp1 + j) * L + l]);
                }
                F::mac(acc, x, w);
            }
            u32 r[2 * L];
            F::finish(r, acc, f);
            store_limbs<L, false>(shares + (size_t)i * sstride + h * L, r);
        }
    }
}

// ---------------------------------------------------------------------------------------
// K3: Lagrange recombination, out[r] = sum_i lambda[r][i] * row_i for each of the `width` points r.
//   full : tab[(r*k + i)*L ..] = lambda[r][i] in table form; k full products, lazy sum, one reduction.
//   small: when every lambda has a signed representative of magnitude < 2^58 -- always the case for
//          x-coordinates 1..k at 0, where lambda_i = (-1)^(i-1) C(k,i), e.g. the 2t+1 = m shares of a resharing
//          (runtime.py:672-680) -- the k full-width products become multiplications by 64-bit constants into ONE
//          (L+1)-limb sum.  tab[2*(r*k+i)] = |lambda|, tab[2*(r*k+i)+1] = sign.
// ---------------------------------------------------------------------------------------

template <int L, int KIND, bool SMALL>
struct RecSum {
    typedef Fp<L, KIND> F;
    static constexpr int N = 2 * L;
    static constexpr int W = SMALL ? F::WSM : F::WACC;   // accumulator words
    // acc += lambda[idx] * x, idx = r*k + i (warp-uniform)
    static __device__ __forceinline__ void add(u32* acc, const u32* x, const FieldParams& f, const u64* tab, int idx) {
        if constexpr (SMALL) {
            const u64 mag = tab[2 * idx];
            const bool minus = tab[2 * idx + 1] != 0;
            // -|lambda| * share = |lambda| * (p - share): one accumulator, one reduction
            // (p - 0 = p is a fine representative of 0: the sum stays below k 2^58 p)
            u32 y[N];
            if (minus) sub_n<N>(y, as32(f.p), x);
            else copy_n<N>(y, x);
            F::mac_const(acc, y, mag);
        } else {
            u32 lam[N];
            copy_n<N>(lam, as32(tab + (size_t)idx * L));
            F::mac(acc, x, lam);
        }
    }
    static __device__ __forceinline__ void reduce(u32* r, u32* acc, const FieldParams& f) {
        if constexpr (SMALL) F::reduce_small_q32(r, acc, f);
        else F::finish(r, acc, f);
    }
};

// one element (limb offset limb_off in every row) for every point; rows loaded RB at a time, the loads of a batch
// issued before its multiplies
template <int L, int KIND, bool SMALL>
__device__ __forceinline__ void recombine_element(const FieldParams& f, const RowPtrs& rows, int k, int width,
                                                  const u64* tab, u64* out, size_t ostride, size_t limb_off) {
    typedef RecSum<L, KIND, SMALL> S;
    constexpr int RB = 4;
    for (int r = 0; r < width; r++) {
        u32 acc[S::W];
        zero_n<S::W>(acc);
        for (int i0 = 0; i0 < k; i0 += RB) {
            u32 x[RB][2 * L];
#pragma unroll
            for (int b = 0; b < RB; b++)
                if (i0 + b < k) load_limbs<L, false>(x[b], rows.p[i0 + b] + limb_off);
#pragma unroll
            for (int b = 0; b < RB; b++)
                if (i0 + b < k) S::add(acc, x[b], f, tab, r * k + i0 + b);
        }
        u32 res[2 * L];
        S::reduce(res, acc, f);
        store_limbs<L, false>(out + (size_t)r * ostride + limb_off, res);
    }
}

// K3 for rows that are not all 32-byte aligned, and for 3-limb fields: one element per thread and trip
template <int L, int KIND, bool SMALL>
__global__ void MPYC_LB
k_recombine(FieldParams f, RowPtrs rows, int k, int width, const u64* __restrict__ gtab, u32 tab_bytes,
            u64* __restrict__ out, size_t ostride, size_t n) {
    extern __shared__ __align__(16) u64 stab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(stab, gtab, tab_bytes, &mbar);
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth)
        recombine_element<L, KIND, SMALL>(f, rows, k, width, stab, out, ostride, h * (size_t)L);
}

// K3 for 32-byte aligned rows of 1-, 2- and 4-limb fields, in K2's tile layout (TileItem): a CTA owns 8 KB of each of
// the k input rows and of each output row per trip, so that a warp load (and for L <= 2 a warp store) covers 512
// contiguous bytes.  A 32-byte item per thread, as K3 had before, uses half of every sector a warp access touches.
// KB > 0 (k <= KB): the thread's chunks of all k rows stay in registers while every point is computed, so each row is
// read once per tile whatever the width, and the next tile's chunks are requested before the current tile is
// computed.  KB = 0 (any k): rows are streamed RB at a time for each point, no prefetch.
// L = 4: a thread's item is one 32-byte element, so its accesses are the half-sector pattern again.  The loads are 7/8
// of C5's K3 traffic, and the card moves that mix at 98 % of the coalesced rate in that form (stream probe, DESIGN.md
// section 5).  Results stored through a shared-memory stage with TMA bulk stores measured slower (C5 K3 1.73 vs
// 1.71 ms), so they are stored from registers.
template <int L, int KIND, bool SMALL, int KB>
__global__ void MPYC_LB
k_recombine_tiled(FieldParams f, RowPtrs rows, int k, int width, const u64* __restrict__ gtab, u32 tab_bytes,
                  u64* __restrict__ out, size_t ostride, size_t n) {
    extern __shared__ __align__(16) u64 stab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(stab, gtab, tab_bytes, &mbar);
    typedef RecSum<L, KIND, SMALL> S;
    constexpr int E = VecItem<L>::E, N = 2 * L;
    constexpr int TE = MPYC_TILE_LIMBS / L;   // elements per tile
    constexpr int RB = 4;                      // KB = 0: rows per load batch
    constexpr int KR = KB > 0 ? KB : 1;
    const size_t ntiles = n / TE;
    const u32 o = threadIdx.x * TileItem<L>::STEP;
    u32 cur[KR][E * N], nxt[KR][E * N];
    auto fetch = [&](u32 (*X)[E * N], size_t tile) {
        const size_t off = tile * MPYC_TILE_LIMBS + o;
#pragma unroll
        for (int i = 0; i < KR; i++)
            if (i < k) load_tile_item<L>(X[i], rows.p[i] + off);
    };
    // point r of the thread's item (E elements) of this tile
    auto point = [&](u32* res, int r, size_t tile) {
        u32 acc[E][S::W];
#pragma unroll
        for (int e = 0; e < E; e++) zero_n<S::W>(acc[e]);
        if constexpr (KB > 0) {
#pragma unroll
            for (int i = 0; i < KB; i++)
                if (i < k) {
#pragma unroll
                    for (int e = 0; e < E; e++) S::add(acc[e], cur[i] + e * N, f, stab, r * k + i);
                }
        } else {
            const size_t off = tile * MPYC_TILE_LIMBS + o;
            for (int i0 = 0; i0 < k; i0 += RB) {
                u32 x[RB][E * N];
#pragma unroll
                for (int b = 0; b < RB; b++)
                    if (i0 + b < k) load_tile_item<L>(x[b], rows.p[i0 + b] + off);
#pragma unroll
                for (int b = 0; b < RB; b++)
                    if (i0 + b < k) {
#pragma unroll
                        for (int e = 0; e < E; e++) S::add(acc[e], x[b] + e * N, f, stab, r * k + i0 + b);
                    }
            }
        }
#pragma unroll
        for (int e = 0; e < E; e++) S::reduce(res + e * N, acc[e], f);
    };
    size_t tile = blockIdx.x;
    if constexpr (KB > 0) {
        if (tile < ntiles) fetch(cur, tile);
    }
    for (; tile < ntiles; tile += gridDim.x) {
        const bool more = KB > 0 && tile + gridDim.x < ntiles;
        if constexpr (KB > 0) {
            if (more) fetch(nxt, tile + gridDim.x);
        }
        for (int r = 0; r < width; r++) {
            u32 res[E * N];
            point(res, r, tile);
            u64* p = out + (size_t)r * ostride + tile * MPYC_TILE_LIMBS + o;
            stg_v4(p, res);
            stg_v4(p + TileItem<L>::H, res + 4);
        }
        if (more) {
#pragma unroll
            for (int i = 0; i < KR; i++)
#pragma unroll
                for (int q = 0; q < E * N; q++) cur[i][q] = nxt[i][q];
        }
    }
    // partial last tile: one element per thread, stored directly
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = ntiles * TE + (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth)
        recombine_element<L, KIND, SMALL>(f, rows, k, width, stab, out, ostride, h * (size_t)L);
}

// ---------------------------------------------------------------------------------------
// PRF chunk -> field element (thresha.py:257-261: int.from_bytes(chunk, 'little') % bound), shared by the K4 kernels.
//   bound = 2^b (bound_bits > 0): mask, no reduction.
//   bound = p, pseudo-Mersenne with a limb-aligned power 2^(64L) = cp (mod p), cp = c << (64L - k) < 2^59:
//       the chunk is cut into L-limb pieces X_q and X = sum_q X_q cp^q is gathered in ONE (L+1)-limb accumulator
//       with 64-bit-constant multiplications, then reduced once  (PrssFold::ok; e.g. 2^256-189: X0 + 189 X1)
//   otherwise: Horner over 64-bit limbs from the top, one reduce_small per limb.
// ---------------------------------------------------------------------------------------

struct PrssFold {
    u64 pw[5];    // cp^q
    bool ok;
};

template <int L, int KIND>
__device__ __forceinline__ PrssFold prss_fold_setup(const FieldParams& f, int nl) {
    PrssFold s;
    s.ok = false;
#pragma unroll
    for (int q = 0; q < 5; q++) s.pw[q] = 0;
    if constexpr (KIND != KIND_GENERIC) {
        const u32 sh = 64u * L - f.k;                       // 0 for the aligned kind
        const int pieces = (nl + L - 1) / L;
        if (f.c < (1ull << 16) && sh <= 43 && pieces <= 5) {   // cp < 2^59
            const u64 cp = f.c << sh;
            s.pw[0] = 1;
            s.ok = true;
#pragma unroll
            for (int q = 1; q < 5; q++) {
                if (q < pieces) {
                    if (__umul64hi(s.pw[q - 1], cp) != 0) s.ok = false;
                    s.pw[q] = s.pw[q - 1] * cp;
                }
            }
        }
    }
    return s;
}

// limb w of the chunk at src (little-endian; chunk_bytes need not be a multiple of 8)
__device__ __forceinline__ u64 prss_chunk_limb(const unsigned char* src, int w, int chunk_bytes, bool aligned8) {
    const int lo = w * 8;
    if (lo >= chunk_bytes) return 0;
    if (aligned8) return *reinterpret_cast<const u64*>(src + lo);
    const int hi = min(lo + 8, chunk_bytes);
    u64 limb = 0;
    for (int bb = hi - 1; bb >= lo; bb--) limb = (limb << 8) | src[bb];
    return limb;
}

// A8: chunk_bytes % 8 == 0 and src 8-byte aligned (shared-memory tiles): limbs are read as whole words
template <int L, int KIND, bool A8>
__device__ __forceinline__ void prss_value(u32* v, const unsigned char* src, int chunk_bytes, int nl, int bound_bits,
                                           const PrssFold& fold, const FieldParams& f) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    auto limb_at = [&](int w) -> u64 {
        if constexpr (A8) return w < nl ? reinterpret_cast<const u64*>(src)[w] : 0ull;
        else return prss_chunk_limb(src, w, chunk_bytes, false);
    };
    if (bound_bits > 0) {          // bound 2^b <= p: mask, no reduction (nl <= L)
        zero_n<N>(v);
#pragma unroll
        for (int l = 0; l < L; l++) {
            if (l < nl) {
                u64 limb = limb_at(l);
                const int top = bound_bits - 64 * l;
                if (top < 64) limb &= top > 0 ? ((1ull << top) - 1) : 0ull;
                set64(v, l, limb);
            }
        }
        return;
    }
    u32 x[N + 2];                  // (L+1)-limb value < 2^(k+64) whose residue is the result
    constexpr int MAXP = (L + 4 + L - 1) / L;   // pieces of a chunk of at most L+4 limbs
    // aligned pseudo-Mersenne fields always fold (cp = c < 2^16): the Horner form is not even compiled for them
    if (KIND == KIND_PM_ALIGNED || fold.ok) {
#pragma unroll
        for (int l = 0; l < L; l++) set64(x, l, limb_at(l));
        x[N] = x[N + 1] = 0;
#pragma unroll
        for (int q = 1; q < MAXP; q++) {
            if (q * L < nl) {       // warp-uniform
                u32 piece[N];
#pragma unroll
                for (int l = 0; l < L; l++) set64(piece, l, limb_at(q * L + l));
                F::mac_const(x, piece, fold.pw[q]);
            }
        }
    } else if constexpr (KIND != KIND_PM_ALIGNED) {
        zero_n<N>(v);
        for (int w = nl - 1; w >= 1; w--) {   // v <- (v * 2^64 + limb) mod p, limb by limb from the top
            set64(x, 0, limb_at(w));
#pragma unroll
            for (int l = 0; l < N; l++) x[l + 2] = v[l];
            F::reduce_small(v, x, f);
        }
        set64(x, 0, limb_at(0));
#pragma unroll
        for (int l = 0; l < N; l++) x[l + 2] = v[l];
    }
    F::reduce_small(v, x, f);
}

// table entry == table form of 1 ?  (then multiplying by it and dividing R' back out is the identity)
template <int L, int KIND>
__device__ __forceinline__ bool prss_is_one(const u64* w, const FieldParams& f) {
    bool one = true;
#pragma unroll
    for (int l = 0; l < L; l++) one = one && (w[l] == (KIND == KIND_GENERIC ? f.r1[l] : (l == 0 ? 1ull : 0ull)));
    return one;
}

// One key subset's contribution for one element (d chunks at `base`, chunk_bytes apart).
//   SMALL = false: acc (WACC limbs) += f_S(i) * y   with y = sum_j v_j w_j mod p, full products against table-form constants
//   SMALL = true : acc (WSM limbs)  += |num_S| * (+-y), y = sum_j v_j w_j mod p with plain-integer weights; the caller
//                  reduces once and multiplies by D^-1 (api.cu: prss_small_table)
//   SIMPLE (with SMALL): d == 1 and weight 1 known at compile time -- the plain pseudorandom share of thresha.py:163-173
template <int L, int KIND, bool SMALL, bool A8, bool SIMPLE = false>
__device__ __forceinline__ void prss_subset(u32* acc, const unsigned char* base, int d, int chunk_bytes, int nl, int bound_bits,
                                            bool unit_w, const PrssFold& fold, const u64* coef_S, const u64* wts,
                                            const FieldParams& f) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    u32 y[N];
    if constexpr (SMALL && SIMPLE) {
        prss_value<L, KIND, A8>(y, base, chunk_bytes, nl, bound_bits, fold, f);
        if (coef_S[1] != 0) {                 // negative coefficient: -|c| y = |c| (p - y)   (warp-uniform)
            u32 t[N];
            sub_n<N>(t, as32(f.p), y);
            copy_n<N>(y, t);
        }
        F::mac_const(acc, y, coef_S[0]);
    } else if constexpr (SMALL) {
        u32 inner[F::WSM];
        zero_n<F::WSM>(inner);
        for (int j = 0; j < d; j++) {
            u32 v[N];
            prss_value<L, KIND, A8>(v, base + (size_t)j * chunk_bytes, chunk_bytes, nl, bound_bits, fold, f);
            if (unit_w) copy_n<N>(y, v);
            else F::mac_const(inner, v, wts[j]);
        }
        if (!unit_w) F::reduce_small(y, inner, f);
        if (coef_S[1] != 0) {                 // negative coefficient: -|c| y = |c| (p - y)   (warp-uniform)
            u32 t[N];
            sub_n<N>(t, as32(f.p), y);
            copy_n<N>(y, t);
        }
        F::mac_const(acc, y, coef_S[0]);
    } else {
        u32 inner[F::WACC];
        zero_n<F::WACC>(inner);
        for (int j = 0; j < d; j++) {
            u32 v[N];
            prss_value<L, KIND, A8>(v, base + (size_t)j * chunk_bytes, chunk_bytes, nl, bound_bits, fold, f);
            if (unit_w) copy_n<N>(y, v);
            else F::mac(inner, v, as32(wts + (size_t)j * L));
        }
        if (!unit_w) F::finish(y, inner, f);
        F::mac(acc, y, as32(coef_S));
    }
}

// final value of an element from its accumulator
template <int L, int KIND, bool SMALL>
__device__ __forceinline__ void prss_finish(u32* r, const u32* acc, const u64* dinv, const FieldParams& f) {
    typedef Fp<L, KIND> F;
    if constexpr (SMALL) {
        u32 t[2 * L];
        F::reduce_small(t, acc, f);
        F::mul(r, t, as32(dinv), f);
    } else {
        F::finish(r, acc, f);
    }
}

// ---------------------------------------------------------------------------------------
// K4: PRSS linear step.  For element h and subset S the PRF output is d chunks of chunk_bytes
// little-endian bytes at bytes + S*subset_stride + (h*d + j)*chunk_bytes.
// tab = [coef_S (nsub entries) | weight_j (d entries)], table form.
// ---------------------------------------------------------------------------------------

template <int L, int KIND, bool SMALL>
__global__ void __launch_bounds__(MPYC_THREADS, 2)
k_prss_combine(FieldParams f, const unsigned char* __restrict__ bytes, size_t subset_stride, int nsub, int d,
               int chunk_bytes, int bound_bits, const u64* __restrict__ gtab, u32 tab_bytes, u64* __restrict__ out,
               size_t n) {
    extern __shared__ __align__(16) u64 stab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(stab, gtab, tab_bytes, &mbar);
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int CS = SMALL ? 2 : L;                      // table words per subset coefficient
    constexpr int WA = SMALL ? F::WSM : F::WACC;
    const u64* coef = stab;
    const u64* wts = stab + (size_t)nsub * CS;
    const u64* dinv = wts + d;                             // SMALL only
    const int nl = (chunk_bytes + 7) >> 3;   // limbs per chunk
    const PrssFold fold = prss_fold_setup<L, KIND>(f, nl);
    const bool unit_w = d == 1 && (SMALL ? wts[0] == 1 : prss_is_one<L, KIND>(wts, f));
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        u32 acc[WA];
        zero_n<WA>(acc);
        for (int S = 0; S < nsub; S++)
            prss_subset<L, KIND, SMALL, false>(acc, bytes + (size_t)S * subset_stride + h * (size_t)d * chunk_bytes, d, chunk_bytes,
                                               nl, bound_bits, unit_w, fold, coef + (size_t)S * CS, wts, f);
        u32 r[N];
        prss_finish<L, KIND, SMALL>(r, acc, dinv, f);
        store_limbs<L, false>(out + h * L, r);
    }
}

// K4 (tiled form): one CTA owns a tile of MPYC_THREADS consecutive elements and walks the key subsets; the
// tile's PRF bytes of subset S+1 (MPYC_THREADS*d*chunk_bytes contiguous bytes) are fetched global -> shared
// memory by ONE TMA bulk copy while the threads convert and accumulate subset S from the other buffer
// (double buffering, one mbarrier per buffer).  HBM is read in full coalesced lines instead of one byte per
// thread at a stride of chunk_bytes.  Requires bytes and subset_stride 16-byte aligned.  A8: chunk_bytes % 8 == 0
// (the tile base is 16-byte aligned, so every chunk is read as whole 64-bit words from shared memory).
// smem layout: [table tab_bytes (rounded to 128)] [buffer 0: tile_bytes] [buffer 1: tile_bytes]
template <int L, int KIND, bool SMALL, bool A8, bool SIMPLE>
__global__ void __launch_bounds__(MPYC_THREADS, 2)
k_prss_tiles(FieldParams f, const unsigned char* __restrict__ bytes, size_t subset_stride, int nsub, int d, int chunk_bytes,
             int bound_bits, const u64* __restrict__ gtab, u32 tab_bytes, u64* __restrict__ out, size_t n, u32 tile_bytes) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) u64 mbar_tab;
    __shared__ __align__(8) u64 mbar_buf[2];
    u64* stab = reinterpret_cast<u64*>(smem_raw);
    const u32 tab_room = (tab_bytes + 127u) & ~127u;
    unsigned char* const buf0 = smem_raw + tab_room;   // buffer b at buf0 + b * tile_bytes
    tma_stage_table(stab, gtab, tab_bytes, &mbar_tab);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar_buf[0])));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar_buf[1])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int CS = SMALL ? 2 : L;                      // table words per subset coefficient
    constexpr int WA = SMALL ? F::WSM : F::WACC;
    const u64* coef = stab;
    const u64* wts = stab + (size_t)nsub * CS;
    const u64* dinv = wts + d;                             // SMALL only
    const int nl = (chunk_bytes + 7) >> 3;
    const size_t per_elem = (size_t)d * chunk_bytes;
    const size_t ntiles = (n + MPYC_THREADS - 1) / MPYC_THREADS;
    u32 phases = 0;                                      // bit b: parity the next wait on buffer b expects
    const PrssFold fold = prss_fold_setup<L, KIND>(f, nl);
    const bool unit_w = d == 1 && (SMALL ? wts[0] == 1 : prss_is_one<L, KIND>(wts, f));
    for (size_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const size_t h0 = tile * MPYC_THREADS;
        const size_t cnt = min((size_t)MPYC_THREADS, n - h0);
        const u32 nbytes = (u32)((cnt * per_elem + 15) & ~(size_t)15);   // the caller pads every subset to 16 bytes
        const unsigned char* src0 = bytes + h0 * per_elem;
        auto issue = [&](int S) {   // thread 0: bulk copy of subset S's bytes for this tile into buffer S & 1
            const u32 bar = smem_u32(&mbar_buf[S & 1]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(nbytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             smem_u32(buf0 + (size_t)(S & 1) * tile_bytes)),
                         "l"(src0 + (size_t)S * subset_stride), "r"(nbytes), "r"(bar)
                         : "memory");
        };
        if (threadIdx.x == 0) issue(0);
        const size_t h = h0 + threadIdx.x;
        u32 outer[WA];
        zero_n<WA>(outer);
        for (int S = 0; S < nsub; S++) {
            const int b = S & 1;
            if (threadIdx.x == 0 && S + 1 < nsub) issue(S + 1);   // buffer (S+1)&1 was released by the barrier below
            u32 done = 0;
            while (!done) {
                asm volatile(
                    "{\n\t.reg .pred p;\n\t"
                    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                    "selp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done)
                    : "r"(smem_u32(&mbar_buf[b])), "r"((phases >> b) & 1u)
                    : "memory");
            }
            phases ^= 1u << b;
            if (h < n)
                prss_subset<L, KIND, SMALL, A8, SIMPLE>(outer, buf0 + (size_t)b * tile_bytes + (size_t)threadIdx.x * d * chunk_bytes, d,
                                                        chunk_bytes, nl, bound_bits, unit_w, fold, coef + (size_t)S * CS, wts, f);
            __syncthreads();   // every thread is done with buffer b: it may be refilled (by issue(S+2) next trip)
        }
        if (h < n) {
            u32 r[N];
            prss_finish<L, KIND, SMALL>(r, outer, dinv, f);
            store_limbs<L, false>(out + h * L, r);
        }
    }
}

// ---------------------------------------------------------------------------------------
// K1c: modular matrix product C[r x c] = A[r x k] @ B[k x c] mod p (finfields.py:1126-1146; the
// np_matmul inner step, runtime.py:2531).  Integer work on the IMAD pipe -- no tensor cores for
// >= 64-bit moduli.  One thread owns one output column for TM consecutive rows: B[l][j] is read
// coalesced once per row tile, the A tile is staged in shared memory and broadcast; the k products
// of a dot product are accumulated lazily and reduced once (every 2^20 terms for huge k).
// GENERIC fields: A is converted to table form while it is staged, so REDC divides R' back out.
// ---------------------------------------------------------------------------------------

#define MPYC_MM_KT 64   // k-chunk of the A tile held in shared memory

// Split-k form (ksplit > 1; few output rows, long dot products -- e.g. np_cnnmnist's 1 x 3136 @ 3136 x 1024 layer, which
// has only 4 column tiles): work item w = (slice s, tile) computes the partial products over k-slice s and writes them,
// reduced, to C + s*r*c; the sum over the slices is K7's (Launch::matmul).  ksplit == 1 writes the result itself.
template <int L, int KIND, int TM>
__global__ void MPYC_LB
k_matmul(FieldParams f, const u64* __restrict__ A, const u64* __restrict__ B, u64* __restrict__ C, size_t r, size_t k,
         size_t c, size_t kslice, size_t ksplit) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    __shared__ u32 sA[TM][MPYC_MM_KT][N];
    const size_t col_tiles = (c + MPYC_THREADS - 1) / MPYC_THREADS;
    const size_t row_tiles = (r + TM - 1) / TM;
    const size_t tiles = col_tiles * row_tiles;
    for (size_t w = blockIdx.x; w < tiles * ksplit; w += gridDim.x) {
        const size_t tile = w % tiles, slice = w / tiles;
        const size_t k_lo = slice * kslice, k_hi = min(k, k_lo + kslice);
        u64* Cs = C + slice * r * c * L;
        const size_t i0 = (tile / col_tiles) * TM;
        const size_t j = (tile % col_tiles) * MPYC_THREADS + threadIdx.x;
        u32 acc[TM][F::WACC];
        u32 partial[TM][N];
#pragma unroll
        for (int a = 0; a < TM; a++) {
            zero_n<F::WACC>(acc[a]);
            zero_n<N>(partial[a]);
        }
        u32 lazy = 0;
        for (size_t l0 = k_lo; l0 < k_hi; l0 += MPYC_MM_KT) {
            const int kt = (int)min((size_t)MPYC_MM_KT, k_hi - l0);
            __syncthreads();
            for (int idx = threadIdx.x; idx < TM * kt; idx += MPYC_THREADS) {
                const int a = idx / kt, l = idx % kt;
                u32 x[N];
                if (i0 + a < r) load_limbs<L, false>(x, A + ((i0 + a) * k + l0 + l) * L);
                else zero_n<N>(x);
                F::to_dom(x, x, f);
#pragma unroll
                for (int w = 0; w < N; w++) sA[a][l][w] = x[w];
            }
            __syncthreads();
            if (j < c) {
                for (int l = 0; l < kt; l++) {
                    u32 b[N];
                    load_limbs<L, false>(b, B + ((l0 + l) * c + j) * L);
#pragma unroll
                    for (int a = 0; a < TM; a++) {
                        u32 av[N];
#pragma unroll
                        for (int w = 0; w < N; w++) av[w] = sA[a][l][w];
                        F::mac(acc[a], b, av);
                    }
                }
            }
            lazy += kt;
            if (lazy + MPYC_MM_KT > FF_MAX_LAZY_TERMS) {   // fold the lazy sums before they can overflow
#pragma unroll
                for (int a = 0; a < TM; a++) {
                    u32 t[N];
                    F::finish(t, acc[a], f);
                    F::add(partial[a], partial[a], t, f);
                    zero_n<F::WACC>(acc[a]);
                }
                lazy = 0;
            }
        }
        if (j < c) {
#pragma unroll
            for (int a = 0; a < TM; a++) {
                if (i0 + a < r) {
                    u32 t[N];
                    F::finish(t, acc[a], f);
                    F::add(t, t, partial[a], f);
                    store_limbs<L, false>(Cs + ((i0 + a) * c + j) * L, t);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// utilities
// ---------------------------------------------------------------------------------------

__device__ __forceinline__ u64 splitmix64_dev(u64 x) {
    u64 z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

template <int L, int KIND>
__global__ void MPYC_LB
k_fill_random(FieldParams f, u64* __restrict__ out, size_t n, u64 base) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        u64 x[L + 1];
        u32 r[2 * L];
#pragma unroll
        for (int w = 0; w <= L; w++) x[w] = splitmix64_dev(base + h * (L + 1) + w);
        // keep bits(p)+64 bits so that the value is < 2^64 p (precondition of reduce_small)
        const u32 keep = f.k + 64;   // <= 64 (L+1)
        if (keep < 64u * (L + 1)) {
            const u32 top = keep >> 6, sh = keep & 63;
#pragma unroll
            for (int w = 0; w <= L; w++) {
                if ((u32)w > top) x[w] = 0;
                else if ((u32)w == top) x[w] = sh ? (x[w] & ((1ull << sh) - 1)) : 0;
            }
        }
        u32 x32[2 * L + 2];
#pragma unroll
        for (int w = 0; w <= L; w++) set64(x32, w, x[w]);
        Fp<L, KIND>::reduce_small(r, x32, f);
        store_limbs<L, false>(out + h * L, r);
    }
}

static __global__ void MPYC_LB
k_count_mismatch(const u64* __restrict__ a, const u64* __restrict__ b, size_t n_elems, int L, unsigned long long* count) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    unsigned long long local = 0;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n_elems; h += nth) {
        u64 d = 0;
        for (int l = 0; l < L; l++) d |= a[h * L + l] ^ b[h * L + l];
        local += d != 0;
    }
    for (int off = 16; off > 0; off >>= 1) local += __shfl_down_sync(0xffffffffu, local, off);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

#include "local.cuh"
#include "reduce.cuh"
#include "layout.cuh"
