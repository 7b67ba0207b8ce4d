// K7: sums and running sums of a field array along one axis.  Any C-ordered array is viewed as (O, R, I): R is the length
// of the axis, O the product of the axes before it, I the product of the axes after it.
//
//   k_sum_cols, k_sum_rows     out[o, i] = init + sum_{r < R} in[o, r, i]       np.sum / ndarray.sum (finfields.py:1332-1337)
//   k_scan_cols, k_scan_rows   out[o, inc + r, i] = sum_{r' <= r} in[o, r', i]  np.cumsum / np.cumulative_sum
//
// Two forms, chosen by the launcher from the shape:
//   * columns (I >= 32): a thread owns a column (o, i) and walks R; consecutive threads hold consecutive i, so every
//     warp access is one contiguous segment.  UNROLL rows are requested before the first addition.
//   * rows (I < 32): a warp reads P = floor(32 / I) whole rows per step as one contiguous segment of P*I elements.
//     Lane l owns row stripe l / I and column l % I; after the walk the lanes of one column are combined with
//     shuffles (sum: a tree over the stripes; scan: a Hillis-Steele scan at distances I*2^j per step).
// Either form can take one slice of R per work item (split R, launch_impl.cuh): a sum then writes its slice's reduced
// partial to part[s][o][i], a scan starts its slice from a carry-in (the inclusive scan of those partials at s-1).
//
// Sums accumulate lazily in (L+1)-limb words (Fp::WSM) and reduce once per output: a slice of at most 2^31 rows keeps
// every sum below 2^(k+31), where the launcher sets q32 (Fp::reduce_small_q32).  Scans keep a canonical running sum.
// Loads and stores are 16-byte vectors for even L on 16-byte aligned arrays (VEC), else one 8-byte access per limb.
#pragma once

#define MPYC_RED_UNROLL 8

template <int L, bool VEC>
__device__ __forceinline__ void red_load(u32* v, const u64* p) {
    if constexpr (VEC) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) ldg_v4(v + 4 * q, p + 2 * q);
    } else {
#pragma unroll
        for (int q = 0; q < L; q++) ldg_v2(v + 2 * q, p + q);
    }
}

template <int L, bool VEC>
__device__ __forceinline__ void red_store(u64* p, const u32* v) {
    if constexpr (VEC) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) stg_v4(p + 2 * q, v + 4 * q);
    } else {
#pragma unroll
        for (int q = 0; q < L; q++) stg_v2(p + q, v + 2 * q);
    }
}

// reduce a lazy sum, add init (add_init != 0), store one element
template <int L, int KIND, bool VEC>
__device__ __forceinline__ void sum_finish(const FieldParams& f, const u32* acc, const ScalarParam& init, int add_init, u64* dst) {
    typedef Fp<L, KIND> F;
    u32 r[F::N];
    F::reduce_small_q32(r, acc, f);
    if (add_init) F::add(r, r, as32(init.v), f);
    red_store<L, VEC>(dst, r);
}

// work item w = (slice s, column c = o*I + i) of S*O*I; rows [s*rs, min(R, (s+1)*rs)); result to out[w]
template <int L, int KIND, bool VEC>
__global__ void MPYC_LB
k_sum_cols(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
           ScalarParam init, int add_init) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int U = MPYC_RED_UNROLL;
    const size_t cols = O * I, items = S * cols;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < items; w += nth) {
        const size_t s = w / cols, c = w % cols, o = c / I, i = c % I;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        const u64* p = in + ((o * R + r_lo) * I + i) * L;
        const size_t step = I * L;
        u32 acc[F::WSM];
        zero_n<F::WSM>(acc);
        size_t r = r_lo;
        for (; r + U <= r_hi; r += U, p += U * step) {
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) red_load<L, VEC>(x[u], p + u * step);
#pragma unroll
            for (int u = 0; u < U; u++) acc_add<N, F::WSM>(acc, x[u]);
        }
        for (; r < r_hi; r++, p += step) {
            u32 x[N];
            red_load<L, VEC>(x, p);
            acc_add<N, F::WSM>(acc, x);
        }
        sum_finish<L, KIND, VEC>(f, acc, init, add_init, out + w * L);
    }
}

// warp item w = (slice s, o) of S*O; I < 32.  Result for column i to out[(s*O + o)*I + i]
template <int L, int KIND, bool VEC>
__global__ void MPYC_LB
k_sum_rows(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
           ScalarParam init, int add_init) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int U = MPYC_RED_UNROLL;
    const int lane = threadIdx.x & 31;
    const int Ii = (int)I, P = 32 / Ii;
    const int stripe = lane / Ii, col = lane % Ii;
    const bool active = stripe < P;
    const size_t items = S * O;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
        const size_t s = w / O, o = w % O;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        const u64* base = in + (o * R * I + col) * L;
        u32 acc[F::WSM];
        zero_n<F::WSM>(acc);
        for (size_t r0 = r_lo; r0 < r_hi; r0 += (size_t)P * U) {     // warp-uniform trip count
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_load<L, VEC>(x[u], base + r * I * L);
                else zero_n<N>(x[u]);
            }
#pragma unroll
            for (int u = 0; u < U; u++) acc_add<N, F::WSM>(acc, x[u]);
        }
        // tree over the stripes of each column: stripe 0 ends with the column's total (< 2^(k+31) like every partial)
        for (int d = 1; d < P; d <<= 1) {
            u32 t[F::WSM];
#pragma unroll
            for (int j = 0; j < F::WSM; j++) t[j] = __shfl_down_sync(0xffffffffu, acc[j], d * Ii);
            if (stripe % (2 * d) == 0 && stripe + d < P) acc_add<F::WSM, F::WSM>(acc, t);
        }
        if (lane < Ii) sum_finish<L, KIND, VEC>(f, acc, init, add_init, out + (w * I + col) * L);
    }
}

// work item w = (slice s, column c); the running sum starts from carry[(s-1)*O*I + c] (s > 0, carry != nullptr).
// The output has R + inc rows per o; inc == 1 puts a zero in row 0.
template <int L, int KIND, bool VEC>
__global__ void MPYC_LB
k_scan_cols(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
            const u64* __restrict__ carry, int inc) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int U = 4;
    const size_t cols = O * I, items = S * cols, Rout = R + inc;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < items; w += nth) {
        const size_t s = w / cols, c = w % cols, o = c / I, i = c % I;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        u32 acc[N];
        zero_n<N>(acc);
        if (s > 0 && carry) red_load<L, VEC>(acc, carry + ((s - 1) * cols + c) * L);
        u64* q = out + ((o * Rout + r_lo + inc) * I + i) * L;
        if (inc && s == 0) red_store<L, VEC>(q - I * L, acc);
        const u64* p = in + ((o * R + r_lo) * I + i) * L;
        const size_t step = I * L;
        size_t r = r_lo;
        for (; r + U <= r_hi; r += U, p += U * step, q += U * step) {
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) red_load<L, VEC>(x[u], p + u * step);
#pragma unroll
            for (int u = 0; u < U; u++) {
                F::add(acc, acc, x[u], f);
                red_store<L, VEC>(q + u * step, acc);
            }
        }
        for (; r < r_hi; r++, p += step, q += step) {
            u32 x[N];
            red_load<L, VEC>(x, p);
            F::add(acc, acc, x, f);
            red_store<L, VEC>(q, acc);
        }
    }
}

// warp item w = (slice s, o); I < 32.  Per step: P rows in, an inclusive scan over the stripes of each column, plus the
// column's carry; the last stripe's result is the next step's carry.
template <int L, int KIND, bool VEC>
__global__ void MPYC_LB
k_scan_rows(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
            const u64* __restrict__ carry, int inc) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int U = 4;
    const int lane = threadIdx.x & 31;
    const int Ii = (int)I, P = 32 / Ii;
    const int stripe = lane / Ii, col = lane % Ii;
    const bool active = stripe < P;
    const int last = (P - 1) * Ii + col;                  // lane of this column's last stripe
    const size_t items = S * O, Rout = R + inc;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
        const size_t s = w / O, o = w % O;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        const u64* src = in + (o * R * I + col) * L;
        u64* dst = out + ((o * Rout + inc) * I + col) * L;
        u32 cy[N];
        zero_n<N>(cy);
        if (s > 0 && carry && active) red_load<L, VEC>(cy, carry + (((s - 1) * O + o) * I + col) * L);   // every stripe
        if (inc && s == 0 && lane < Ii) red_store<L, VEC>(dst - I * L, cy);
        for (size_t r0 = r_lo; r0 < r_hi; r0 += (size_t)P * U) {
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_load<L, VEC>(x[u], src + r * I * L);
                else zero_n<N>(x[u]);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                for (int d = 1; d < P; d <<= 1) {
                    u32 t[N];
#pragma unroll
                    for (int j = 0; j < N; j++) t[j] = __shfl_up_sync(0xffffffffu, x[u][j], d * Ii);
                    if (stripe >= d) F::add(x[u], x[u], t, f);
                }
                F::add(x[u], x[u], cy, f);
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_store<L, VEC>(dst + r * I * L, x[u]);
#pragma unroll
                for (int j = 0; j < N; j++) cy[j] = __shfl_sync(0xffffffffu, x[u][j], last);
            }
        }
    }
}
