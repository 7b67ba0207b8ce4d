// K8's copy launcher (layout.cuh): one translation unit for every element size, since layout does not depend on the field.
#include "launch_impl.cuh"

namespace {

bool divides(size_t u, long long x) { return (x % (long long)u) == 0; }

// the widest unit U in {16, 8, 1} bytes that divides both base addresses, every offset and outer stride in bytes and the
// row length: the runs form then moves U-byte words
size_t run_unit(const CopyPlan& p, size_t E, const void* src, const void* dst) {
    for (size_t u : {(size_t)16, (size_t)8}) {
        bool ok = divides(u, (long long)reinterpret_cast<uintptr_t>(src)) && divides(u, (long long)reinterpret_cast<uintptr_t>(dst)) &&
                  divides(u, p.soff * (long long)E) && divides(u, p.doff * (long long)E) && divides(u, p.ext[p.rank - 1] * (long long)E);
        for (int k = 0; ok && k < p.rank - 1; k++) ok = divides(u, p.sstr[k] * (long long)E) && divides(u, p.dstr[k] * (long long)E);
        if (ok) return u;
    }
    return 1;
}

// the plan in units of u bytes (innermost stride 1 on both sides, no index table on it)
CopyPlan in_units(const CopyPlan& p, size_t E, size_t u) {
    CopyPlan q = p;
    const long long s = (long long)E, d = (long long)u;
    q.soff = p.soff * s / d;
    q.doff = p.doff * s / d;
    for (int k = 0; k < p.rank - 1; k++) {
        q.sstr[k] = p.sstr[k] * s / d;
        q.dstr[k] = p.dstr[k] * s / d;
    }
    q.ext[p.rank - 1] = p.ext[p.rank - 1] * s / d;
    return q;
}

template <class T>
cudaError_t gather(const CopyPlan& p, const void* src, void* dst, cudaStream_t st) {
    size_t n = 1;
    for (int k = 0; k < p.rank; k++) n *= (size_t)p.ext[k];
    if (n <= 0x7fffffffu)
        return launch_kernel(k_copy_gather<T, u32>, n, 0, st, p, (const T*)src, (T*)dst, (u32)n);
    return launch_kernel(k_copy_gather<T, u64>, n, 0, st, p, (const T*)src, (T*)dst, (u64)n);
}

template <class T>
cudaError_t permute(const CopyPlan& p, int ax, const void* src, void* dst, cudaStream_t st) {
    size_t tiles = (size_t)((p.ext[ax] + 31) / 32) * (size_t)((p.ext[p.rank - 1] + 31) / 32);
    for (int k = 0; k < p.rank - 1; k++)
        if (k != ax) tiles *= (size_t)p.ext[k];
    // 64-bit tile numbers: their arithmetic is once per 32 x 32 tile
    return launch_kernel(k_copy_permute<T, u64>, tiles * MPYC_THREADS, 0, st, p, ax, (const T*)src, (T*)dst, (u64)tiles);
}

// calls fn(T) with the element type that moves E bytes: 16-byte words when both sides allow them
template <class Fn>
cudaError_t with_elem(size_t E, bool wide, Fn&& fn) {
    switch (E) {
        case 1: return fn(ViewElem<unsigned char, 1>());
        case 8: return fn(ViewElem<u64, 1>());
        case 16: return wide ? fn(ViewElem<uint4, 1>()) : fn(ViewElem<u64, 2>());
        case 24: return fn(ViewElem<u64, 3>());
        case 32: return wide ? fn(ViewElem<uint4, 2>()) : fn(ViewElem<u64, 4>());
    }
    return cudaErrorInvalidValue;
}

// 16-byte element accesses: both bases and every element offset a multiple of 16 bytes
bool elems_aligned16(const CopyPlan& p, size_t E, const void* src, const void* dst) {
    if (E % 16) return false;
    return divides(16, (long long)reinterpret_cast<uintptr_t>(src)) && divides(16, (long long)reinterpret_cast<uintptr_t>(dst));
}

}  // namespace

cudaError_t launch_copy_view(const CopyPlan& p, size_t E, const void* src, void* dst, cudaStream_t st) {
    for (int k = 0; k < p.rank; k++)
        if (p.ext[k] == 0) return cudaSuccess;
    if (p.rank == 0) {
        CopyPlan q = p;                                  // one element: a rank-1 view of extent 1
        q.rank = 1, q.ext[0] = 1, q.sstr[0] = q.dstr[0] = 1, q.six = q.dix = -1;
        return launch_copy_view(q, E, src, dst, st);
    }
    const int in = p.rank - 1;
    const bool runs = p.sstr[in] == 1 && p.dstr[in] == 1 && p.six != in && p.dix != in;
    if (runs) {
        const size_t u = run_unit(p, E, src, dst);
        const CopyPlan q = in_units(p, E, u);
        if (u == 16) return gather<ViewElem<uint4, 1>>(q, src, dst, st);
        if (u == 8) return gather<ViewElem<u64, 1>>(q, src, dst, st);
        return gather<ViewElem<unsigned char, 1>>(q, src, dst, st);
    }
    const bool wide = elems_aligned16(p, E, src, dst);
    int ax = -1;
    if (p.dstr[in] == 1 && p.dix != in && p.six != in && p.ext[in] > 1)
        for (int k = in - 1; k >= 0 && ax < 0; k--)
            if ((p.sstr[k] == 1 || p.sstr[k] == -1) && p.six != k && p.dix != k && p.ext[k] > 1) ax = k;
    if (ax >= 0) return with_elem(E, wide, [&](auto t) { return permute<decltype(t)>(p, ax, src, dst, st); });
    return with_elem(E, wide, [&](auto t) { return gather<decltype(t)>(p, src, dst, st); });
}
