// K14's launcher (matmul_int.cuh): the columns form for c >= 32, the rows form below; k is split into slices when the
// outputs' work items cannot fill two CTAs per SM (matmul_int_plan).  The slice partials (S, r, c) live in scratch from the
// library's pool and K7 sums them along S.
#include "launch_impl.cuh"
#include "matmul_int.cuh"

namespace {

struct KSplit {
    size_t S, kslice;
};

// Slices keep >= 64 terms (a shared-memory chunk, columns) / >= 1024 terms (rows form), as K13's prod_plan.
KSplit matmul_int_plan(bool cols, size_t items, size_t k) {
    const size_t want = (size_t)mpyc_sm_count() * 2 * MPYC_THREADS;      // threads
    const size_t most = cols ? k / MPYC_MI_KT : k / 1024;
    size_t S = items < want ? std::min((want + items - 1) / items, most) : 1;
    if (S < 2) return KSplit{1, std::max<size_t>(k, 1)};
    size_t ks = (k + S - 1) / S;
    if (cols) ks = (ks + MPYC_MI_KT - 1) / MPYC_MI_KT * MPYC_MI_KT;       // whole chunks
    return KSplit{(k + ks - 1) / ks, ks};
}

template <int L, int KIND, bool WLEFT>
cudaError_t matmul_int_k(const FieldParams& fp, const u64* X, const u64* W, int wuns, u64* C, size_t r, size_t k, size_t c,
                         cudaStream_t st) {
    const bool cols = c >= 32;
    const int tm = r >= 4 ? 4 : 1;        // rows per thread in the columns form, as K1c
    const size_t tiles = (c + MPYC_THREADS - 1) / MPYC_THREADS * ((r + tm - 1) / tm);
    const KSplit pl = matmul_int_plan(cols, cols ? tiles * MPYC_THREADS : r * 32, k);
    u64* dst = C;
    u64* part = nullptr;                  // (S, r, c) slice sums
    if (pl.S > 1) {
        cudaError_t e = mpyc_scratch_alloc(&part, pl.S * r * c * L * sizeof(u64), st);
        if (e != cudaSuccess) return e;
        dst = part;
    }
    cudaError_t e;
    if (!cols)
        e = launch_kernel(k_matmul_int_rows<L, KIND, WLEFT>, pl.S * r * 32, 0, st, fp, X, W, wuns, dst, r, k, c, pl.kslice, pl.S);
    else if (tm == 4)
        e = launch_kernel(k_matmul_int_cols<L, KIND, 4, WLEFT>, pl.S * tiles * MPYC_THREADS, 0, st, fp, X, W, wuns, dst, r, k, c,
                          pl.kslice, pl.S);
    else
        e = launch_kernel(k_matmul_int_cols<L, KIND, 1, WLEFT>, pl.S * tiles * MPYC_THREADS, 0, st, fp, X, W, wuns, dst, r, k, c,
                          pl.kslice, pl.S);
    if (e == cudaSuccess && pl.S > 1) e = Launch<L>::sum_axis(fp, part, C, 1, pl.S, r * c, nullptr, st);
    if (part) cudaFreeAsync(part, st);
    return e;
}

template <int L>
cudaError_t matmul_int_l(const FieldParams& fp, const u64* X, const u64* W, bool wuns, bool w_left, u64* C, size_t r, size_t k,
                         size_t c, cudaStream_t st) {
    if (r == 0 || c == 0) return cudaSuccess;
    const int u = wuns ? 1 : 0;
#define M(K)                                                                                   \
    return w_left ? matmul_int_k<L, K, true>(fp, X, W, u, C, r, k, c, st)                      \
                  : matmul_int_k<L, K, false>(fp, X, W, u, C, r, k, c, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_matmul_int(const FieldParams& fp, const u64* X, const u64* W, bool w_unsigned, bool w_left, u64* C, size_t r,
                              size_t k, size_t c, cudaStream_t st) {
    switch (fp.L) {
        case 1: return matmul_int_l<1>(fp, X, W, w_unsigned, w_left, C, r, k, c, st);
        case 2: return matmul_int_l<2>(fp, X, W, w_unsigned, w_left, C, r, k, c, st);
        case 3: return matmul_int_l<3>(fp, X, W, w_unsigned, w_left, C, r, k, c, st);
        case 4: return matmul_int_l<4>(fp, X, W, w_unsigned, w_left, C, r, k, c, st);
    }
    return cudaErrorInvalidValue;
}
