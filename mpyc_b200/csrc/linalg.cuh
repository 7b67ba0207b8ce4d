// K9: determinants, linear solves and inverses of prime-field matrices (FiniteFieldArray.gauss_det / gauss_solve /
// gauss_inv, mpyc/finfields.py:872-955), without a modular inversion per pivot.
//
// Division-free elimination: at step k the pivot row x (the first row >= k with a nonzero entry in column k, taken only
// when a[k][k] == 0 -- the reference's rule) is swapped with row k, and every other row i is replaced by
//   R_i <- p_k R_i - a_ik R_k          (p_k = a[k][k] after the swap)
// on the columns j > k (column k becomes 0 and is never read again).  Row i is then the reference's row times a
// nonzero factor, so every "is it zero" decision, and so every swap, is the reference's.  With P_k = p_0 ... p_k:
//   det:   only rows i > k are updated.  Row k has been scaled by P_{k-1}, so the reference's pivot is p_k / P_{k-1} and
//          its determinant (which ignores the sign of the swaps) is P_{n-1} / (P_0 P_1 ... P_{n-2}): one inversion per
//          matrix, gathered over a whole stack into one Montgomery-trick batch (k_inv_batch).
//   solve: Gauss-Jordan, rows i != k are updated.  The diagonal of row i ends as p_i p_{i+1} ... p_{n-1} =
//          P_{n-1} / P_{i-1}, so X_i = Y_i P_{i-1} P_{n-1}^-1: one Fermat inversion per system.
// A column without a pivot means a singular matrix: det 0, or the singular flag for solve.
//
//   k_lin_tile        the whole elimination in shared memory; a group of G threads (a warp for n <= 32, several
//                     matrices per CTA, else the whole CTA) owns one matrix.  Pivot search is a group-wide atomicMin.
//   k_lin_load        step form: the augmented matrix (A | B) or (A | I) into a global workspace
//   k_lin_pivot       step form, one CTA per pivot: find and swap the pivot row, record p_k, its row and the flag
//   k_lin_update      step form: the division-free update of the active block
//   k_lin_det_finish  step form: P_{n-1} / (P_0 ... P_{n-2}) (one thread)
//   k_lin_row_scales  step form: P_{i-1} P_{n-1}^-1 for every row (one thread)
//   k_lin_scale_rows  step form: X_i = Y_i * scale_i
// Offsets into global memory are 64-bit.
#pragma once

template <int L>
__device__ __forceinline__ void store_plain(u64* p, const u32* v) {
#pragma unroll
    for (int q = 0; q < L; q++) p[q] = (u64)v[2 * q] | ((u64)v[2 * q + 1] << 32);
}

template <int L>
__device__ __forceinline__ void set_one(u32* v) {
    zero_n<2 * L>(v);
    v[0] = 1;
}

template <int G>
__device__ __forceinline__ void group_sync() {
    if constexpr (G == 32) __syncwarp();
    else __syncthreads();
}

// element (i, j) of the augmented n x (n + nrhs) matrix (A | B), or (A | I) when B is null
template <int L>
__device__ __forceinline__ void lin_source(u32* v, const u64* A, const u64* B, size_t n, size_t nrhs, size_t i, size_t j) {
    if (j < n) {
        load_plain<L>(v, A + (i * n + j) * L);
    } else if (B) {
        load_plain<L>(v, B + (i * nrhs + (j - n)) * L);
    } else {
        zero_n<2 * L>(v);
        v[0] = i == j - n;
    }
}

// a_ij <- piv a_ij - a_ik a_kj
template <int L, int KIND>
__device__ __forceinline__ void lin_eliminate(u64* aij, const u32* piv, const u32* aik, const u64* akj, const FieldParams& f) {
    typedef Fp<L, KIND> F;
    u32 x[2 * L], y[2 * L];
    load_plain<L>(x, aij);
    load_plain<L>(y, akj);
    F::mul(x, x, piv, f);
    F::mul(y, aik, y, f);
    F::sub(x, x, y, f);
    store_plain<L>(aij, x);
}

template <int L, int KIND>
__device__ __forceinline__ void lin_invert(u32* r, const u32* a, const ExpParams& ex, const FieldParams& f) {
    typedef Fp<L, KIND> F;
    F::to_dom(r, a, f);
    F::dpow_uniform(r, r, ex.e, ex.ebits, f);
    F::from_dom(r, r, f);
}

// Tile form.  det (SOLVE false): matrix b of A (batch x n x n) -> out[b] = P_{n-1}, den[b] = P_0 ... P_{n-2} (0 and 1 when
// singular).  solve: A (n x n), B (n x nrhs, null: identity) -> out = X (n x nrhs); *flag = 1 when singular.
// Shared memory per group: the n x W matrix, then (solve) the n + 1 values P_{i-1} and P_{n-1}^-1.
template <int L, int KIND, int G, bool SOLVE>
__global__ void MPYC_LB
k_lin_tile(FieldParams f, ExpParams ex, const u64* __restrict__ A, const u64* __restrict__ B, u64* __restrict__ out,
           u64* __restrict__ den, int* flag, size_t batch, int n, int nrhs) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    extern __shared__ u64 lin_smem[];
    __shared__ int slot[MPYC_THREADS / 32];
    const int g = threadIdx.x / G, lane = threadIdx.x % G;
    const size_t b = (size_t)blockIdx.x * (blockDim.x / G) + g;
    if (b >= batch) return;                         // only warp groups can be spare: they sync by themselves
    const int W = SOLVE ? n + nrhs : n;
    u64* M = lin_smem + (size_t)g * ((size_t)n * W + (SOLVE ? n + 1 : 0)) * L;
    u64* sc = M + (size_t)n * W * L;
    const u64* Ab = A + b * (size_t)n * n * L;
    for (int e = lane; e < n * W; e += G) {
        u32 v[N];
        lin_source<L>(v, Ab, B, n, nrhs, e / W, e % W);
        store_plain<L>(M + (size_t)e * L, v);
    }
    u32 P[N], Q[N];
    set_one<L>(P);
    set_one<L>(Q);
    bool singular = false;
    group_sync<G>();
    for (int k = 0; k < n; k++) {
        if (lane == 0) slot[g] = n;
        group_sync<G>();
        for (int i = k + lane; i < n; i += G) {
            u32 v[N];
            load_plain<L>(v, M + ((size_t)i * W + k) * L);
            if (!is_zero_n<N>(v)) {
                atomicMin(&slot[g], i);
                break;
            }
        }
        group_sync<G>();
        const int x = slot[g];
        if (x == n) {
            singular = true;
            break;
        }
        if (x != k) {
            for (int j = k + lane; j < W; j += G)
#pragma unroll
                for (int q = 0; q < L; q++) {
                    u64* u = M + ((size_t)k * W + j) * L + q;
                    u64* w = M + ((size_t)x * W + j) * L + q;
                    const u64 t = *u;
                    *u = *w;
                    *w = t;
                }
        }
        group_sync<G>();
        u32 piv[N];
        load_plain<L>(piv, M + ((size_t)k * W + k) * L);
        const int nr = SOLVE ? n - 1 : n - 1 - k, nc = W - 1 - k;
        for (int e = lane; e < nr * nc; e += G) {
            const int r = e / nc, j = k + 1 + e % nc;
            const int i = SOLVE ? (r < k ? r : r + 1) : k + 1 + r;
            u32 aik[N];
            load_plain<L>(aik, M + ((size_t)i * W + k) * L);
            lin_eliminate<L, KIND>(M + ((size_t)i * W + j) * L, piv, aik, M + ((size_t)k * W + j) * L, f);
        }
        if (lane == 0) {
            if constexpr (SOLVE) store_plain<L>(sc + (size_t)k * L, P);
            F::mul(P, P, piv, f);
            if (!SOLVE && k < n - 1) F::mul(Q, Q, P, f);
        }
        group_sync<G>();
    }
    if constexpr (!SOLVE) {
        if (lane == 0) {
            if (singular) {
                zero_n<N>(P);
                set_one<L>(Q);
            }
            store_plain<L>(out + b * L, P);
            store_plain<L>(den + b * L, Q);
        }
    } else {
        if (singular) {
            if (lane == 0) *flag = 1;
            return;
        }
        if (lane == 0) {
            u32 iv[N];
            lin_invert<L, KIND>(iv, P, ex, f);
            store_plain<L>(sc + (size_t)n * L, iv);
        }
        group_sync<G>();
        u32 iv[N];
        load_plain<L>(iv, sc + (size_t)n * L);
        for (int e = lane; e < n * nrhs; e += G) {
            const int i = e / nrhs, j = e % nrhs;
            u32 y[N], s[N];
            load_plain<L>(y, M + ((size_t)i * W + n + j) * L);
            load_plain<L>(s, sc + (size_t)i * L);
            F::mul(s, s, iv, f);
            F::mul(y, y, s, f);
            store_plain<L>(out + (size_t)e * L, y);
        }
    }
}

// ---- step form: one matrix in a global n x W workspace M -------------------------------------------------------------

template <int L>
__global__ void MPYC_LB
k_lin_load(const u64* __restrict__ A, const u64* __restrict__ B, u64* __restrict__ M, size_t n, size_t nrhs, size_t W) {
    const size_t items = n * W, nth = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < items; e += nth) {
        u32 v[2 * L];
        lin_source<L>(v, A, B, n, nrhs, e / W, e % W);
        store_plain<L>(M + e * L, v);
    }
}

// one CTA: pivot row of column k, swapped into row k; piv[k] = p_k, row[k] = its original row; *flag = 1 when there is
// none.  Nothing happens once the flag is set.
template <int L>
__global__ void MPYC_LB
k_lin_pivot(u64* M, size_t n, size_t W, size_t k, u64* piv, long long* row, int* flag) {
    __shared__ unsigned long long slot;
    if (*flag) return;
    if (threadIdx.x == 0) slot = n;
    __syncthreads();
    for (size_t i = k + threadIdx.x; i < n; i += blockDim.x) {
        u32 v[2 * L];
        load_plain<L>(v, M + (i * W + k) * L);
        if (!is_zero_n<2 * L>(v)) {
            atomicMin(&slot, (unsigned long long)i);
            break;
        }
    }
    __syncthreads();
    const size_t x = slot;
    if (x == n) {
        if (threadIdx.x == 0) *flag = 1;
        return;
    }
    if (x != k) {
        for (size_t j = k + threadIdx.x; j < W; j += blockDim.x)
#pragma unroll
            for (int q = 0; q < L; q++) {
                const u64 t = M[(k * W + j) * L + q];
                M[(k * W + j) * L + q] = M[(x * W + j) * L + q];
                M[(x * W + j) * L + q] = t;
            }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < L; q++) piv[k * L + q] = M[(k * W + k) * L + q];
        row[k] = (long long)x;
    }
}

// rows i > k (det) or i != k (solve), columns k < j < W: a_ij <- p_k a_ij - a_ik a_kj.  Consecutive threads take
// consecutive columns of a row.
template <int L, int KIND, bool SOLVE>
__global__ void MPYC_LB
k_lin_update(FieldParams f, u64* M, size_t n, size_t W, size_t k, const int* flag) {
    if (*flag) return;
    const size_t nr = SOLVE ? n - 1 : n - 1 - k, nc = W - 1 - k, items = nr * nc;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    u32 piv[2 * L];
    load_plain<L>(piv, M + (k * W + k) * L);
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < items; e += nth) {
        const size_t r = e / nc, j = k + 1 + e % nc;
        const size_t i = SOLVE ? (r < k ? r : r + 1) : k + 1 + r;
        u32 aik[2 * L];
        load_plain<L>(aik, M + (i * W + k) * L);
        lin_eliminate<L, KIND>(M + (i * W + j) * L, piv, aik, M + (k * W + j) * L, f);
    }
}

template <int L, int KIND>
__global__ void k_lin_det_finish(FieldParams f, ExpParams ex, const u64* __restrict__ piv, size_t n, const int* flag,
                                 u64* __restrict__ out) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    u32 P[N], Q[N], v[N];
    set_one<L>(P);
    set_one<L>(Q);
    if (*flag) {
        zero_n<N>(P);
        store_plain<L>(out, P);
        return;
    }
    for (size_t k = 0; k < n; k++) {
        load_plain<L>(v, piv + k * L);
        F::mul(P, P, v, f);
        if (k + 1 < n) F::mul(Q, Q, P, f);
    }
    lin_invert<L, KIND>(v, Q, ex, f);
    F::mul(P, P, v, f);
    store_plain<L>(out, P);
}

// scale[i] = P_{i-1} P_{n-1}^-1
template <int L, int KIND>
__global__ void k_lin_row_scales(FieldParams f, ExpParams ex, const u64* __restrict__ piv, size_t n, const int* flag,
                                 u64* __restrict__ scale) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    if (blockIdx.x != 0 || threadIdx.x != 0 || *flag) return;
    u32 P[N], v[N];
    set_one<L>(P);
    for (size_t k = 0; k < n; k++) {
        store_plain<L>(scale + k * L, P);
        load_plain<L>(v, piv + k * L);
        F::mul(P, P, v, f);
    }
    lin_invert<L, KIND>(P, P, ex, f);
    for (size_t k = 0; k < n; k++) {
        load_plain<L>(v, scale + k * L);
        F::mul(v, v, P, f);
        store_plain<L>(scale + k * L, v);
    }
}

// X (n x nrhs) = the right-hand columns of M, row i times scale[i]
template <int L, int KIND>
__global__ void MPYC_LB
k_lin_scale_rows(FieldParams f, const u64* __restrict__ M, size_t n, size_t W, size_t nrhs, const u64* __restrict__ scale,
                 const int* flag, u64* __restrict__ X) {
    typedef Fp<L, KIND> F;
    if (*flag) return;
    const size_t items = n * nrhs, nth = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < items; e += nth) {
        const size_t i = e / nrhs, j = e % nrhs;
        u32 y[2 * L], s[2 * L];
        load_plain<L>(y, M + (i * W + (W - nrhs) + j) * L);
        load_plain<L>(s, scale + i * L);
        F::mul(y, y, s, f);
        store_plain<L>(X + e * L, y);
    }
}
