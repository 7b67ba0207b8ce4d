// K14: C = X @ W or C = W @ X mod p, X a canonical prime-field matrix, W a public matrix of 64-bit integers (int64, or
// uint64 when `wuns`), all row-major and contiguous (FiniteFieldArray.__matmul__ / __rmatmul__ with an integer ndarray,
// finfields.py:1126-1146; Runtime.np_argmax / np_argmin's `u @ np.arange(n)`, runtime.py:3750-3757, and np_matmul with a
// public operand, runtime.py:2482-2541).
//
// A term is x * w with w a plain 64-bit constant: two IMAD.WIDE rows of N = 2L 32-bit limbs (MulInt::mac), against the N^2
// of a full product in K1c -- W never exists as field limbs, and is read as 8 bytes per entry instead of 8L.
//
// Signs: -|w| x = |w| (p - x), so one accumulator serves both signs and there is one reduction per output.  The columns
// form with X on the left stages both x and p - x of its tile in shared memory and each thread picks the copy its entry's
// sign asks for (the two addresses lie in different banks); with W on the left the sign is warp-uniform and the thread
// negates its own x once per term.  p - 0 = p represents 0.
//
// Bound: y <= p and |w| <= 2^64 - 1 give terms < p 2^64, so T terms sum to < T p 2^64.  The reduction (Fp::finish on the
// zero-extended sum) needs < 2^(2k + 20) for pseudo-Mersenne fields (k >= 56) and < p R' for generic ones.  The lazy sums
// fold into a canonical partial every T <= 2^12 terms (FOLD), well before K1c's 2^20: T p 2^64 < 2^(k + 76) <= 2^(2k + 20)
// for every k >= 56, and the sum fits N + 3 words.  2^20 would do for k >= 64 only, and a fold costs one reduction per
// 4096 terms, under 1 % of the 2N IMADs each term takes.
// Generic fields: finish is a REDC and divides by R'; X stays canonical, and the reduced result is multiplied back by R'
// once per output (Fp::to_dom) instead of converting every x to table form, which would cost a full product per term.
//
// Two forms, chosen by the launcher from the shape (inst_matmul_int.cu):
//   * columns (c >= 32): K1c's tiling.  A thread owns one output column for TM rows; the left operand's k-chunk is staged
//     in shared memory -- field limbs (x and p - x) when X is on the left, int64 when W is.
//   * rows (c < 32): a warp owns one output row i.  As in K7's rows form, lane l owns stripe l / c and column l % c, P =
//     floor(32 / c) stripes walk k in steps of P, each step reading P consecutive entries of the left row and P whole rows
//     of the right operand (P * c contiguous elements); a shuffle tree over the stripes combines the lazy sums (their
//     total term count obeys the fold bound).  c = 1 -- matrix-vector products and argmax's `u @ arange(n)` -- keeps all
//     32 lanes busy, where K1c's c = 1 would run one thread per CTA.
// Both forms take one slice of k per work item when the outputs cannot fill two CTAs per SM: slice s writes its reduced
// partial to C + s r c, and K7's sum adds the slices up (as split-k K1c does).
#pragma once

#define MPYC_MI_KT 64   // k-chunk of the left tile held in shared memory (columns form)
#define MPYC_MI_U 4     // entries per lane loaded before their multiplies (rows form)

template <int L, int KIND>
struct MulInt {
    typedef Fp<L, KIND> F;
    static constexpr int N = 2 * L;
    static constexpr int W = N + 3;                                         // accumulator words (see the bound above)
    static constexpr u32 FOLD = 1u << 12;                                   // terms per lazy sum

    // |w| and its sign
    static __device__ __forceinline__ u64 magnitude(u64 w, int wuns, bool& minus) {
        minus = !wuns && (long long)w < 0;
        return minus ? 0ull - w : w;
    }

    // acc += y * v
    static __device__ __forceinline__ void mac(u32* acc, const u32* y, u64 v) {
        mac_small<N, W>(acc, y, (u32)v);
        mac_small<N, W - 1>(acc + 1, y, (u32)(v >> 32));
    }

    // r = acc mod p, divided by R' for generic fields (finish's REDC)
    static __device__ __forceinline__ void reduce(u32* r, const u32* acc, const FieldParams& f) {
        u32 t[F::WACC];
#pragma unroll
        for (int i = 0; i < F::WACC; i++) t[i] = i < W ? acc[i] : 0u;
        F::finish(r, t, f);
    }

    // out = reduce(acc) + partial, back in canonical form
    static __device__ __forceinline__ void store(u64* out, const u32* acc, const u32* partial, const FieldParams& f) {
        u32 t[N];
        reduce(t, acc, f);
        F::add(t, t, partial, f);
        F::to_dom(t, t, f);
        store_limbs<L, false>(out, t);
    }
};

// work item w = (slice s, tile) of ksplit * tiles; a tile is TM rows x MPYC_THREADS columns of C.  X (r x k) @ W (k x c), or
// with WLEFT W (r x k) @ X (k x c).
template <int L, int KIND, int TM, bool WLEFT>
__global__ void MPYC_LB
k_matmul_int_cols(FieldParams f, const u64* __restrict__ X, const u64* __restrict__ Wm, int wuns, u64* __restrict__ C,
                  size_t r, size_t k, size_t c, size_t kslice, size_t ksplit) {
    typedef MulInt<L, KIND> M;
    constexpr int N = 2 * L;
    __shared__ u32 sX[WLEFT ? 1 : TM][MPYC_MI_KT][2][N];    // x and p - x
    __shared__ u64 sW[WLEFT ? TM : 1][MPYC_MI_KT];
    const size_t col_tiles = (c + MPYC_THREADS - 1) / MPYC_THREADS;
    const size_t tiles = col_tiles * ((r + TM - 1) / TM);
    for (size_t w = blockIdx.x; w < tiles * ksplit; w += gridDim.x) {
        const size_t tile = w % tiles, slice = w / tiles;
        const size_t k_lo = slice * kslice, k_hi = min(k, k_lo + kslice);
        const size_t i0 = (tile / col_tiles) * TM;
        const size_t j = (tile % col_tiles) * MPYC_THREADS + threadIdx.x;
        u32 acc[TM][M::W];
        u32 partial[TM][N];
#pragma unroll
        for (int a = 0; a < TM; a++) {
            zero_n<M::W>(acc[a]);
            zero_n<N>(partial[a]);
        }
        u32 lazy = 0;
        for (size_t l0 = k_lo; l0 < k_hi; l0 += MPYC_MI_KT) {
            const int kt = (int)min((size_t)MPYC_MI_KT, k_hi - l0);
            __syncthreads();
            for (int idx = threadIdx.x; idx < TM * kt; idx += MPYC_THREADS) {
                const int a = idx / kt, l = idx % kt;
                const bool in = i0 + a < r;
                if constexpr (WLEFT) {
                    sW[a][l] = in ? Wm[(i0 + a) * k + l0 + l] : 0ull;
                } else {
                    u32 x[N], nx[N];
                    if (in) load_limbs<L, false>(x, X + ((i0 + a) * k + l0 + l) * L);
                    else zero_n<N>(x);
                    sub_n<N>(nx, as32(f.p), x);
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        sX[a][l][0][q] = x[q];
                        sX[a][l][1][q] = nx[q];
                    }
                }
            }
            __syncthreads();
            if (j < c) {
                for (int l = 0; l < kt; l++) {
                    if constexpr (WLEFT) {
                        u32 x[N], nx[N];
                        load_limbs<L, false>(x, X + ((l0 + l) * c + j) * L);
                        sub_n<N>(nx, as32(f.p), x);
#pragma unroll
                        for (int a = 0; a < TM; a++) {
                            bool minus;
                            const u64 mag = M::magnitude(sW[a][l], wuns, minus);
                            u32 y[N];
#pragma unroll
                            for (int q = 0; q < N; q++) y[q] = minus ? nx[q] : x[q];
                            M::mac(acc[a], y, mag);
                        }
                    } else {
                        bool minus;
                        const u64 mag = M::magnitude(Wm[(l0 + l) * c + j], wuns, minus);
                        const int sgn = minus ? 1 : 0;
#pragma unroll
                        for (int a = 0; a < TM; a++) {
                            u32 y[N];
#pragma unroll
                            for (int q = 0; q < N; q++) y[q] = sX[a][l][sgn][q];
                            M::mac(acc[a], y, mag);
                        }
                    }
                }
            }
            lazy += kt;
            if (lazy + MPYC_MI_KT > M::FOLD) {   // fold the lazy sums before they pass the bound
#pragma unroll
                for (int a = 0; a < TM; a++) {
                    u32 t[N];
                    M::reduce(t, acc[a], f);
                    Fp<L, KIND>::add(partial[a], partial[a], t, f);
                    zero_n<M::W>(acc[a]);
                }
                lazy = 0;
            }
        }
        if (j < c) {
            u64* Cs = C + slice * r * c * L;
#pragma unroll
            for (int a = 0; a < TM; a++)
                if (i0 + a < r) M::store(Cs + ((i0 + a) * c + j) * L, acc[a], partial[a], f);
        }
    }
}

// lanes of one column combine their lazy sums: stripe 0 ends with the column's total
template <int L, int KIND>
__device__ __forceinline__ void mul_int_tree(u32* acc, int stripe, int P, int Ci) {
    constexpr int W = MulInt<L, KIND>::W;
    for (int d = 1; d < P; d <<= 1) {
        u32 t[W];
#pragma unroll
        for (int q = 0; q < W; q++) t[q] = __shfl_down_sync(0xffffffffu, acc[q], d * Ci);
        if (stripe % (2 * d) == 0 && stripe + d < P) acc_add<W, W>(acc, t);
    }
}

// warp item w = (slice s, row i) of ksplit * r; c < 32.  Result for column col to C[(s r + i) c + col]
template <int L, int KIND, bool WLEFT>
__global__ void MPYC_LB
k_matmul_int_rows(FieldParams f, const u64* __restrict__ X, const u64* __restrict__ Wm, int wuns, u64* __restrict__ C,
                  size_t r, size_t k, size_t c, size_t kslice, size_t ksplit) {
    typedef MulInt<L, KIND> M;
    constexpr int N = 2 * L;
    constexpr int U = MPYC_MI_U;
    const int lane = threadIdx.x & 31;
    const int Ci = (int)c, P = 32 / Ci;
    const int stripe = lane / Ci, col = lane % Ci;
    const bool active = stripe < P;
    const u32 step = (u32)(P * U);
    const size_t items = ksplit * r;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
        const size_t s = w / r, i = w % r;
        const size_t k_lo = s * kslice, k_hi = min(k, k_lo + kslice);
        u32 acc[M::W];
        u32 partial[N];
        zero_n<M::W>(acc);
        zero_n<N>(partial);
        u32 lazy = 0;
        for (size_t l0 = k_lo; l0 < k_hi; l0 += step) {     // warp-uniform trip count
            u32 x[U][N];
            u64 wv[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t l = l0 + (size_t)u * P + stripe;
                if (active && l < k_hi) {
                    if constexpr (WLEFT) {
                        wv[u] = Wm[i * k + l];
                        load_limbs<L, false>(x[u], X + (l * c + col) * L);
                    } else {
                        wv[u] = Wm[l * c + col];
                        load_limbs<L, false>(x[u], X + (i * k + l) * L);
                    }
                } else {
                    wv[u] = 0;
                    zero_n<N>(x[u]);
                }
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                bool minus;
                const u64 mag = M::magnitude(wv[u], wuns, minus);
                u32 nx[N];
                sub_n<N>(nx, as32(f.p), x[u]);
                select_n<N>(x[u], nx, minus);
                M::mac(acc, x[u], mag);
            }
            lazy += step;
            if (lazy + step > M::FOLD) {                        // the stripes' terms together stay within the bound
                mul_int_tree<L, KIND>(acc, stripe, P, Ci);
                if (lane < Ci) {
                    u32 t[N];
                    M::reduce(t, acc, f);
                    Fp<L, KIND>::add(partial, partial, t, f);
                }
                zero_n<M::W>(acc);
                lazy = 0;
            }
        }
        mul_int_tree<L, KIND>(acc, stripe, P, Ci);
        if (lane < Ci) M::store(C + ((s * r + i) * c + col) * L, acc, partial, f);
    }
}
