// K10: 1-D convolution of prime-field vectors (np.convolve of FiniteFieldArrays, mpyc/finfields.py:766-819; the local
// step of Runtime.np_convolve, runtime.py:2580-2634, and of the secret-shift branch of Runtime.np_roll,
// runtime.py:3300-3314).  With the shorter operand H (s taps) and the longer X (g elements):
//   full[k] = sum_t H[t] X[k - t]     (0 <= t < s, 0 <= k - t < g)
// and the kernel computes full[lo .. lo + count) only.
//
// A CTA owns a run of T = MPYC_THREADS * TM consecutive outputs, a thread TM consecutive ones.  The CTA walks the taps
// that meet its run in chunks of at most MPYC_CV_KT: each chunk stages the taps (table form for GENERIC fields, as K1c
// stages A) and the window of X they reach in shared memory.  A thread keeps TM elements of X in registers as a ring:
// going from tap t to t + 1 every output of the thread moves one element down X, so each tap costs one broadcast load
// of H[t], one new element of X and TM lazy products (F::mac).  The ring slot of an element is its index mod TM, so the
// tap loop is unrolled by TM and the rotation costs no moves.  Out-of-range taps and elements read as zero.
//
// The window is stored as N planes of 32-bit words with one padding word per 32 (x -> x + x / 32): the TM-strided
// loads of a warp's threads then fall in distinct banks.
//
// Split form (slice < s): work item (slice q, tile) takes only the taps in [q * slice, (q + 1) * slice) and writes its
// reduced partial sums to C + q * count; the launcher sums the slices with K7 (as split-k K1c does).
#pragma once

#define MPYC_CV_KT 128   // taps staged per chunk

// two CTAs per SM: at most 128 registers, which TM = 2 meets without spills for every L
template <int L, int KIND, int TM>
__global__ void __launch_bounds__(MPYC_THREADS, 2)
k_conv(FieldParams f, const u64* __restrict__ X, size_t g, const u64* __restrict__ H, size_t s, u64* __restrict__ C,
       size_t lo, size_t count, size_t slice, size_t nslices) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L, T = MPYC_THREADS * TM, WIN = T + MPYC_CV_KT, WP = WIN + WIN / 32;
    static_assert((32 % TM) == 0 && MPYC_CV_KT % TM == 0, "TM must divide the bank count and the chunk");
    __shared__ u32 sH[MPYC_CV_KT][N];
    __shared__ u32 sX[N][WP];
    const size_t tiles = (count + T - 1) / T;
    for (size_t w = blockIdx.x; w < tiles * nslices; w += gridDim.x) {
        const size_t tile = w % tiles, q = w / tiles;
        const size_t k0 = lo + tile * T;                  // the tile's first output
        const size_t kt0 = k0 + (size_t)threadIdx.x * TM;  // this thread's first output
        // the taps of this slice that meet outputs [k0, k0 + T): 0 <= k - t < g
        const size_t t_lo = max(k0 + 1 > g ? k0 + 1 - g : (size_t)0, q * slice);
        const size_t t_hi = min(min(s, k0 + T), q * slice + slice);
        u32 acc[TM][F::WACC];
#pragma unroll
        for (int j = 0; j < TM; j++) zero_n<F::WACC>(acc[j]);
        u32 lazy = 0;
        for (size_t t0 = t_lo; t0 < t_hi; t0 += MPYC_CV_KT) {
            const int kt = (int)min((size_t)MPYC_CV_KT, t_hi - t0);
            const int ktr = (kt + TM - 1) / TM * TM;      // whole turns of the ring; the taps past kt are zero
            __syncthreads();
            for (int u = threadIdx.x; u < ktr; u += MPYC_THREADS) {
                u32 h[N];
                if (u < kt) {
                    load_limbs<L, false>(h, H + (t0 + u) * L);
                    F::to_dom(h, h, f);
                } else {
                    zero_n<N>(h);
                }
#pragma unroll
                for (int x = 0; x < N; x++) sH[u][x] = h[x];
            }
            // element e of the window is X[xb + e]
            const long long xb = (long long)k0 - (long long)t0 - ktr;
            for (int e = threadIdx.x; e < T + ktr; e += MPYC_THREADS) {
                const long long i = xb + e;
                u32 v[N];
                if (i >= 0 && i < (long long)g) load_limbs<L, false>(v, X + (size_t)i * L);
                else zero_n<N>(v);
                const int p = e + (e >> 5);
#pragma unroll
                for (int x = 0; x < N; x++) sX[x][p] = v[x];
            }
            __syncthreads();
            // at chunk tap tt, output j of the thread needs X[kt0 + j - t0 - tt] = window element
            // threadIdx.x * TM + ktr + j - tt, kept in ring slot (j - tt) mod TM
            const int eb = threadIdx.x * TM + ktr;
            u32 ring[TM][N];
#pragma unroll
            for (int j = 0; j < TM; j++) {
                const int p = eb + j + ((eb + j) >> 5);
#pragma unroll
                for (int x = 0; x < N; x++) ring[j][x] = sX[x][p];
            }
            for (int tb = 0; tb < ktr; tb += TM) {
#pragma unroll
                for (int u = 0; u < TM; u++) {
                    u32 h[N];
#pragma unroll
                    for (int x = 0; x < N; x++) h[x] = sH[tb + u][x];
#pragma unroll
                    for (int j = 0; j < TM; j++) F::mac(acc[j], ring[(j - u + TM) % TM], h);
                    // the next tap needs X[kt0 - t0 - tt - 1] (element eb - tt - 1) in place of X[kt0 + TM - 1 - t0 - tt]
                    const int e = eb - (tb + u) - 1;
                    const int p = e + (e >> 5);
#pragma unroll
                    for (int x = 0; x < N; x++) ring[TM - 1 - u][x] = sX[x][p];
                }
            }
            lazy += ktr;
            if (lazy + MPYC_CV_KT > FF_MAX_LAZY_TERMS) {   // fold the lazy sums before they can overflow: the reduced
                u32 one[N];                                // sum goes back as one product, sum * 1 (table form of 1)
                F::dom_one(one, f);
#pragma unroll
                for (int j = 0; j < TM; j++) {
                    u32 r[N];
                    F::finish(r, acc[j], f);
                    zero_n<F::WACC>(acc[j]);
                    F::mac(acc[j], r, one);
                }
                lazy = 1;
            }
        }
        u64* Cq = C + q * count * L;
#pragma unroll
        for (int j = 0; j < TM; j++) {
            if (kt0 + j < lo + count) {
                u32 r[N];
                F::finish(r, acc[j], f);
                store_limbs<L, false>(Cq + (kt0 + j - lo) * L, r);
            }
        }
    }
}
