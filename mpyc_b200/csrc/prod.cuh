// K13: products, running products and all / any of a field array along one axis.  The array is viewed as (O, R, I) as
// K7 views it (reduce.cuh): R is the length of the axis, O the product of the axes before it, I of those after it.
//
//   k_prod_cols, k_prod_rows        out[o, i] = init * prod_{r < R} in[o, r, i]        np.prod / ndarray.prod (finfields.py:1339-1349)
//   k_cumprod_cols, k_cumprod_rows  out[o, inc + r, i] = prod_{r' <= r} in[o, r', i]   np.cumprod / np.cumulative_prod
//   k_allany_cols, k_allany_rows    out[o, i] = (#{r : in[o, r, i] != 0} == R) or (.. != 0) as 0 / 1   np.all / np.any
//
// The same two forms as K7, chosen by the launcher from the shape (inst_prod.cu):
//   * columns (I >= 32, or R * I < 32): a thread owns a column (o, i) and walks R; for I >= 32 a warp access is one
//     contiguous segment.
//   * rows (I < 32): a warp reads P = floor(32 / I) whole rows per step; lane l owns row stripe l / I and column l % I,
//     and the stripes of a column are combined with shuffles at the end (a tree for prod and all / any, a Hillis-Steele
//     scan at distances I*2^j for the running product).
// Products cannot be accumulated lazily as sums are, and each F::mul depends on the one before it, so a product thread
// keeps A independent partial products (PrdCfg) that it multiplies together once at the end; a running product has no
// such freedom and walks its column in order.  Either form can take one slice of R per work item (split R, like K7):
// a product or all / any then writes its slice's partial to part[s][o][i], a running product starts from a carry-in.
// Values stay canonical throughout (F::mul of canonical operands).  Loads and stores are K7's (red_load / red_store):
// 16-byte vectors for even L on 16-byte aligned arrays, else 8-byte accesses, so operands need 8-byte alignment only.
#pragma once

// two CTAs of MPYC_THREADS per SM (the occupancy the launcher's split decision plans for): at most 128 registers
#define MPYC_PRD_LB __launch_bounds__(MPYC_THREADS, 2)

template <int L>
struct PrdCfg {
    static constexpr int A = L <= 2 ? 4 : 2;    // independent partial products per thread
};

template <int N>
__device__ __forceinline__ void prd_one(u32* v) {
    zero_n<N>(v);
    v[0] = 1;
}

// multiply the partials together, then by init (mul_init != 0), store one element
template <int L, int KIND, bool VEC, int A>
__device__ __forceinline__ void prod_finish(const FieldParams& f, u32 (*acc)[2 * L], const ScalarParam& init, int mul_init, u64* dst) {
    typedef Fp<L, KIND> F;
#pragma unroll
    for (int a = 1; a < A; a++) F::mul(acc[0], acc[0], acc[a], f);
    if (mul_init) F::mul(acc[0], acc[0], as32(init.v), f);
    red_store<L, VEC>(dst, acc[0]);
}

// work item w = (slice s, column c = o*I + i) of S*O*I; rows [s*rs, min(R, (s+1)*rs)); result to out[w]
template <int L, int KIND, bool VEC>
__global__ void MPYC_PRD_LB
k_prod_cols(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
            ScalarParam init, int mul_init) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int A = PrdCfg<L>::A;
    const size_t cols = O * I, items = S * cols;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < items; w += nth) {
        const size_t s = w / cols, c = w % cols, o = c / I, i = c % I;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        const u64* p = in + ((o * R + r_lo) * I + i) * L;
        const size_t step = I * L;
        u32 acc[A][N];
#pragma unroll
        for (int a = 0; a < A; a++) prd_one<N>(acc[a]);
        size_t r = r_lo;
        for (; r + A <= r_hi; r += A, p += A * step) {
            u32 x[A][N];
#pragma unroll
            for (int a = 0; a < A; a++) red_load<L, VEC>(x[a], p + a * step);
#pragma unroll
            for (int a = 0; a < A; a++) F::mul(acc[a], acc[a], x[a], f);
        }
        for (; r < r_hi; r++, p += step) {
            u32 x[N];
            red_load<L, VEC>(x, p);
            F::mul(acc[0], acc[0], x, f);
        }
        prod_finish<L, KIND, VEC, A>(f, acc, init, mul_init, out + w * L);
    }
}

// warp item w = (slice s, o) of S*O; I < 32.  Result for column i to out[(s*O + o)*I + i]
template <int L, int KIND, bool VEC>
__global__ void MPYC_PRD_LB
k_prod_rows(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
            ScalarParam init, int mul_init) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int A = PrdCfg<L>::A;
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
        u32 acc[A][N];
#pragma unroll
        for (int a = 0; a < A; a++) prd_one<N>(acc[a]);
        for (size_t r0 = r_lo; r0 < r_hi; r0 += (size_t)P * A) {     // warp-uniform trip count
            u32 x[A][N];
#pragma unroll
            for (int a = 0; a < A; a++) {
                const size_t r = r0 + (size_t)a * P + stripe;
                if (active && r < r_hi) red_load<L, VEC>(x[a], base + r * I * L);
                else prd_one<N>(x[a]);
            }
#pragma unroll
            for (int a = 0; a < A; a++) F::mul(acc[a], acc[a], x[a], f);
        }
#pragma unroll
        for (int a = 1; a < A; a++) F::mul(acc[0], acc[0], acc[a], f);
        // tree over the stripes of each column: stripe 0 ends with the column's product
        for (int d = 1; d < P; d <<= 1) {
            u32 t[N];
#pragma unroll
            for (int j = 0; j < N; j++) t[j] = __shfl_down_sync(0xffffffffu, acc[0][j], d * Ii);
            if (stripe % (2 * d) == 0 && stripe + d < P) F::mul(acc[0], acc[0], t, f);
        }
        if (lane < Ii) prod_finish<L, KIND, VEC, 1>(f, acc, init, mul_init, out + (w * I + col) * L);
    }
}

// work item w = (slice s, column c); the running product starts from carry[(s-1)*O*I + c] (s > 0, carry != nullptr).
// The output has R + inc rows per o; inc == 1 puts a one in row 0.
template <int L, int KIND, bool VEC>
__global__ void MPYC_PRD_LB
k_cumprod_cols(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
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
        prd_one<N>(acc);
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
                F::mul(acc, acc, x[u], f);
                red_store<L, VEC>(q + u * step, acc);
            }
        }
        for (; r < r_hi; r++, p += step, q += step) {
            u32 x[N];
            red_load<L, VEC>(x, p);
            F::mul(acc, acc, x, f);
            red_store<L, VEC>(q, acc);
        }
    }
}

// warp item w = (slice s, o); I < 32.  Per step: P rows in, an inclusive product scan over the stripes of each column
// (Hillis-Steele), times the column's carry; the last stripe's result is the next step's carry.
template <int L, int KIND, bool VEC>
__global__ void MPYC_PRD_LB
k_cumprod_rows(FieldParams f, const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S,
               const u64* __restrict__ carry, int inc) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    constexpr int U = 2;
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
        prd_one<N>(cy);
        if (s > 0 && carry && active) red_load<L, VEC>(cy, carry + (((s - 1) * O + o) * I + col) * L);   // every stripe
        if (inc && s == 0 && lane < Ii) red_store<L, VEC>(dst - I * L, cy);
        for (size_t r0 = r_lo; r0 < r_hi; r0 += (size_t)P * U) {
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_load<L, VEC>(x[u], src + r * I * L);
                else prd_one<N>(x[u]);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                for (int d = 1; d < P; d <<= 1) {
                    u32 t[N];
#pragma unroll
                    for (int j = 0; j < N; j++) t[j] = __shfl_up_sync(0xffffffffu, x[u][j], d * Ii);
                    if (stripe >= d) F::mul(x[u], x[u], t, f);
                }
                F::mul(x[u], x[u], cy, f);
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_store<L, VEC>(dst + r * I * L, x[u]);
#pragma unroll
                for (int j = 0; j < N; j++) cy[j] = __shfl_sync(0xffffffffu, x[u][j], last);
            }
        }
    }
}

template <int L>
__device__ __forceinline__ bool prd_nonzero(const u32* x) {
    u32 v = 0;
#pragma unroll
    for (int j = 0; j < 2 * L; j++) v |= x[j];
    return v != 0;
}

// 1 if the slice's count of nonzero elements is its length (all) or positive (any), else 0, as L canonical limbs
template <int L, bool VEC, bool ANY>
__device__ __forceinline__ void allany_finish(unsigned long long cnt, size_t len, u64* dst) {
    u32 v[2 * L];
    zero_n<2 * L>(v);
    v[0] = ANY ? (cnt != 0) : (cnt == len);
    red_store<L, VEC>(dst, v);
}

// work item w = (slice s, column c) of S*O*I, as k_prod_cols
template <int L, bool VEC, bool ANY>
__global__ void MPYC_LB
k_allany_cols(const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S) {
    constexpr int N = 2 * L;
    constexpr int U = MPYC_RED_UNROLL;
    const size_t cols = O * I, items = S * cols;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < items; w += nth) {
        const size_t s = w / cols, c = w % cols, o = c / I, i = c % I;
        const size_t r_lo = s * rs, r_hi = min(R, r_lo + rs);
        const u64* p = in + ((o * R + r_lo) * I + i) * L;
        const size_t step = I * L;
        unsigned long long cnt = 0;
        size_t r = r_lo;
        for (; r + U <= r_hi; r += U, p += U * step) {
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) red_load<L, VEC>(x[u], p + u * step);
#pragma unroll
            for (int u = 0; u < U; u++) cnt += prd_nonzero<L>(x[u]);
        }
        for (; r < r_hi; r++, p += step) {
            u32 x[N];
            red_load<L, VEC>(x, p);
            cnt += prd_nonzero<L>(x);
        }
        allany_finish<L, VEC, ANY>(cnt, r_hi - r_lo, out + w * L);
    }
}

// warp item w = (slice s, o) of S*O; I < 32, as k_prod_rows
template <int L, bool VEC, bool ANY>
__global__ void MPYC_LB
k_allany_rows(const u64* __restrict__ in, u64* __restrict__ out, size_t O, size_t R, size_t I, size_t rs, size_t S) {
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
        unsigned long long cnt = 0;
        for (size_t r0 = r_lo; r0 < r_hi; r0 += (size_t)P * U) {     // warp-uniform trip count
            u32 x[U][N];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t r = r0 + (size_t)u * P + stripe;
                if (active && r < r_hi) red_load<L, VEC>(x[u], base + r * I * L);
                else zero_n<N>(x[u]);
            }
#pragma unroll
            for (int u = 0; u < U; u++) cnt += prd_nonzero<L>(x[u]);
        }
        for (int d = 1; d < P; d <<= 1) {
            const unsigned long long t = __shfl_down_sync(0xffffffffu, cnt, d * Ii);
            if (stripe % (2 * d) == 0 && stripe + d < P) cnt += t;
        }
        if (lane < Ii) allany_finish<L, VEC, ANY>(cnt, r_hi - r_lo, out + (w * I + col) * L);
    }
}
