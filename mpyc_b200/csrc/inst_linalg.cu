// K9's launchers (linalg.cuh): the form is chosen from n, the right-hand side, L and the device's shared-memory limit.
//   tile: the matrix with its right-hand side (and, for solve, n + 1 row scales) fits one CTA's shared memory.  Matrices
//         of n <= 32 get one warp each, up to 8 to a CTA; larger ones the whole CTA.
//   step: two launches per pivot on a global workspace (k_lin_pivot, k_lin_update); the host does not synchronise inside
//         the loop, the singular flag is read once at the end (solve).  A stack of matrices too large for a tile runs
//         the step form one matrix after the other.
#include "launch_impl.cuh"
#include "linalg.cuh"

namespace {

// e = p - 2 (Fermat inverses)
ExpParams fermat_exponent(const FieldParams& fp) {
    ExpParams ex;
    memset(&ex, 0, sizeof ex);
    u64 borrow = 2;
    for (int i = 0; i < 4; i++) {
        const u64 before = fp.p[i];
        ex.e[i] = before - borrow;
        borrow = before < borrow ? 1 : 0;
    }
    ex.ebits = 0;
    for (int i = 7; i >= 0 && !ex.ebits; i--)
        if (ex.e[i]) ex.ebits = 64 * i + 64 - __builtin_clzll(ex.e[i]);
    return ex;
}

// dynamic shared memory a CTA of `kernel` may use: the device's opt-in limit per block less the kernel's static shared
// memory (the two together must not exceed the limit)
template <class... KArgs>
size_t smem_limit(void (*kernel)(KArgs...)) {
    int dev = 0, v = 0;
    cudaFuncAttributes fa;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(kernel)) != cudaSuccess)
        return 0;
    return (size_t)v > fa.sharedSizeBytes ? (size_t)v - fa.sharedSizeBytes : 0;
}

// dynamic shared memory of one tile-form group: n x W elements plus, for solve, n + 1 row scales; 0 when it does not fit
// within limit (smem_limit of the tile kernel), which sends the call to the step form
size_t tile_bytes(size_t n, size_t W, bool solve, int L, size_t limit) {
    if (n > 1024 || W > 2048) return 0;
    const size_t b = (n * W + (solve ? n + 1 : 0)) * 8 * (size_t)L;
    return b <= limit ? b : 0;
}

template <class... KArgs, class... Args>
cudaError_t launch_tile(void (*kernel)(KArgs...), size_t batch, int G, size_t per_group, size_t limit, cudaStream_t st,
                        Args... args) {
    int groups = 1;
    if (G == 32) {
        groups = (int)std::min<size_t>(MPYC_THREADS / 32, limit / per_group);
        groups = (int)std::min<size_t>((size_t)groups, batch);
    }
    const size_t smem = per_group * groups;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    const size_t grid = (batch + groups - 1) / groups;
    kernel<<<(unsigned)grid, G * groups, smem, st>>>(args...);
    g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <int L, int KIND>
cudaError_t step_eliminate(const FieldParams& fp, bool solve, u64* M, size_t n, size_t W, u64* piv, long long* row, int* flag,
                           cudaStream_t st) {
    for (size_t k = 0; k < n; k++) {
        k_lin_pivot<L><<<1, MPYC_THREADS, 0, st>>>(M, n, W, k, piv, row, flag);
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        const size_t items = (solve ? n - 1 : n - 1 - k) * (W - 1 - k);
        e = solve ? launch_kernel(k_lin_update<L, KIND, true>, items, 0, st, fp, M, n, W, k, (const int*)flag)
                  : launch_kernel(k_lin_update<L, KIND, false>, items, 0, st, fp, M, n, W, k, (const int*)flag);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// a stream-ordered workspace, freed on the same stream when it goes out of scope
struct Scratch {
    void* p = nullptr;
    cudaStream_t st;
    explicit Scratch(cudaStream_t s) : st(s) {}
    cudaError_t get(size_t bytes) { return cudaMallocAsync(&p, bytes, st); }
    ~Scratch() {
        if (p) cudaFreeAsync(p, st);
    }
};

size_t round256(size_t b) { return (b + 255) / 256 * 256; }

template <int L, int KIND>
cudaError_t det_k(const FieldParams& fp, const u64* a, size_t batch, size_t n, u64* out, cudaStream_t st) {
    const ExpParams ex = fermat_exponent(fp);
    const int G = n <= 32 ? 32 : MPYC_THREADS;
    const auto tile = n <= 32 ? k_lin_tile<L, KIND, 32, false> : k_lin_tile<L, KIND, MPYC_THREADS, false>;
    const size_t E = 8 * L, limit = smem_limit(tile);
    const size_t per = tile_bytes(n, n, false, L, limit);
    Scratch w(st);
    if (per) {
        // numerators, denominators, their inverses, k_inv_batch's zero flag
        const size_t vb = round256(batch * E);
        cudaError_t e = w.get(3 * vb + 256);
        if (e != cudaSuccess) return e;
        u64* num = (u64*)w.p;
        u64* den = (u64*)((char*)w.p + vb);
        u64* inv = (u64*)((char*)w.p + 2 * vb);
        int* zf = (int*)((char*)w.p + 3 * vb);
        if ((e = cudaMemsetAsync(zf, 0, sizeof(int), st)) != cudaSuccess) return e;
        e = launch_tile(tile, batch, G, per, limit, st, fp, ex, a, (const u64*)nullptr, num, den, zf, batch, (int)n, 0);
        if (e != cudaSuccess) return e;
        if ((e = Launch<L>::inv_batch(fp, ex, den, inv, zf, batch, st)) != cudaSuccess) return e;
        return Launch<L>::binop(fp, OP_MUL, num, inv, nullptr, out, batch, st);
    }
    const size_t mb = round256(n * n * E), pb = round256(n * E), rb = round256(n * sizeof(long long));
    cudaError_t e = w.get(mb + pb + rb + 256);
    if (e != cudaSuccess) return e;
    u64* M = (u64*)w.p;
    u64* piv = (u64*)((char*)w.p + mb);
    long long* row = (long long*)((char*)w.p + mb + pb);
    int* flag = (int*)((char*)w.p + mb + pb + rb);
    for (size_t b = 0; b < batch; b++) {
        if ((e = cudaMemsetAsync(flag, 0, sizeof(int), st)) != cudaSuccess) return e;
        e = launch_kernel(k_lin_load<L>, n * n, 0, st, a + b * n * n * L, (const u64*)nullptr, M, n, (size_t)0, n);
        if (e != cudaSuccess) return e;
        if ((e = step_eliminate<L, KIND>(fp, false, M, n, n, piv, row, flag, st)) != cudaSuccess) return e;
        k_lin_det_finish<L, KIND><<<1, 32, 0, st>>>(fp, ex, piv, n, flag, out + b * L);
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <int L, int KIND>
cudaError_t solve_k(const FieldParams& fp, const u64* a, size_t n, const u64* b, size_t nrhs, u64* x, int* singular,
                    cudaStream_t st) {
    const ExpParams ex = fermat_exponent(fp);
    const int G = n <= 32 ? 32 : MPYC_THREADS;
    const auto tile = n <= 32 ? k_lin_tile<L, KIND, 32, true> : k_lin_tile<L, KIND, MPYC_THREADS, true>;
    const size_t E = 8 * L, W = n + nrhs, limit = smem_limit(tile);
    const size_t per = tile_bytes(n, W, true, L, limit);
    Scratch w(st);
    int* flag = nullptr;
    cudaError_t e;
    if (per) {
        if ((e = w.get(256)) != cudaSuccess) return e;
        flag = (int*)w.p;
        if ((e = cudaMemsetAsync(flag, 0, sizeof(int), st)) != cudaSuccess) return e;
        e = launch_tile(tile, 1, G, per, limit, st, fp, ex, a, b, x, (u64*)nullptr, flag, (size_t)1, (int)n, (int)nrhs);
        if (e != cudaSuccess) return e;
    } else {
        const size_t mb = round256(n * W * E), pb = round256(n * E), rb = round256(n * sizeof(long long));
        if ((e = w.get(mb + 2 * pb + rb + 256)) != cudaSuccess) return e;
        u64* M = (u64*)w.p;
        u64* piv = (u64*)((char*)w.p + mb);
        u64* scale = (u64*)((char*)w.p + mb + pb);
        long long* row = (long long*)((char*)w.p + mb + 2 * pb);
        flag = (int*)((char*)w.p + mb + 2 * pb + rb);
        if ((e = cudaMemsetAsync(flag, 0, sizeof(int), st)) != cudaSuccess) return e;
        if ((e = launch_kernel(k_lin_load<L>, n * W, 0, st, a, b, M, n, nrhs, W)) != cudaSuccess) return e;
        if ((e = step_eliminate<L, KIND>(fp, true, M, n, W, piv, row, flag, st)) != cudaSuccess) return e;
        k_lin_row_scales<L, KIND><<<1, 32, 0, st>>>(fp, ex, piv, n, flag, scale);
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        e = launch_kernel(k_lin_scale_rows<L, KIND>, n * nrhs, 0, st, fp, (const u64*)M, n, W, nrhs, (const u64*)scale,
                          (const int*)flag, x);
        if (e != cudaSuccess) return e;
    }
    int h = 0;
    if ((e = cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    *singular = h;
    return cudaSuccess;
}

template <class Fn>
cudaError_t with_cell(const FieldParams& fp, Fn&& fn) {
#define LIN_CELL(LL)                                                                                       \
    case LL:                                                                                               \
        switch (fp.kind) {                                                                                 \
            case KIND_GENERIC: return fn(std::integral_constant<int, LL>(), std::integral_constant<int, KIND_GENERIC>());       \
            case KIND_PM_ALIGNED: return fn(std::integral_constant<int, LL>(), std::integral_constant<int, KIND_PM_ALIGNED>()); \
            case KIND_PM_SHIFT: return fn(std::integral_constant<int, LL>(), std::integral_constant<int, KIND_PM_SHIFT>());     \
        }                                                                                                  \
        return cudaErrorInvalidValue;
    switch (fp.L) {
        LIN_CELL(1)
        LIN_CELL(2)
        LIN_CELL(3)
        LIN_CELL(4)
    }
#undef LIN_CELL
    return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_det(const FieldParams& fp, const u64* a, size_t batch, size_t n, u64* out, cudaStream_t st) {
    return with_cell(fp, [&](auto Lc, auto Kc) { return det_k<decltype(Lc)::value, decltype(Kc)::value>(fp, a, batch, n, out, st); });
}

cudaError_t launch_solve(const FieldParams& fp, const u64* a, size_t n, const u64* b, size_t nrhs, u64* x, int* singular,
                         cudaStream_t st) {
    return with_cell(fp, [&](auto Lc, auto Kc) {
        return solve_k<decltype(Lc)::value, decltype(Kc)::value>(fp, a, n, b, nrhs, x, singular, st);
    });
}
