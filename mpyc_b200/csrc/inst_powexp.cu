// K12's launcher (powexp.cuh).  The fixed-base form takes its comb tables as dynamic shared memory; the caller keeps
// them within MPYC_PE_SMEM_MAX, so that two CTAs fit an SM next to the default carve-out.
#include "launch_impl.cuh"
#include "powexp.cuh"

namespace {

template <int L>
cudaError_t powexp_l(const FieldParams& fp, const u64* a, const u64* tab, u32 tab_bytes, int w, int nwin, const u64* e,
                     int el, int ebits, const unsigned char* sgn, u64* out, size_t n, cudaStream_t st) {
    if (tab) {
        // the opt-in limit is set for the largest tables: the kernel's static shared memory (its mbarrier) counts against
        // the default 48 KB too, so a 48 KB table (64-bit exponents at L = 3) already needs it
#define M(K)                                                                                                             \
    {                                                                                                                    \
        auto kernel = k_powexp_fixed<L, K>;                                                                              \
        const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MPYC_PE_SMEM_MAX); \
        if (err != cudaSuccess) return err;                                                                              \
        return launch_kernel(kernel, n, tab_bytes, st, fp, tab, tab_bytes, w, nwin, e, el, sgn, out, n);                 \
    }
        KIND_SWITCH(fp.kind, M)
#undef M
    } else {
        const int npairs = (ebits + 1) / 2;
#define M(K) return launch_kernel(k_powexp_elem<L, K>, n, 0, st, fp, a, e, el, npairs, out, n)
        KIND_SWITCH(fp.kind, M)
#undef M
    }
    return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_powexp(const FieldParams& fp, const u64* a, const u64* tab, u32 tab_bytes, int w, int nwin, const u64* e,
                          int el, int ebits, const unsigned char* sgn, u64* out, size_t n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    switch (fp.L) {
        case 1: return powexp_l<1>(fp, a, tab, tab_bytes, w, nwin, e, el, ebits, sgn, out, n, st);
        case 2: return powexp_l<2>(fp, a, tab, tab_bytes, w, nwin, e, el, ebits, sgn, out, n, st);
        case 3: return powexp_l<3>(fp, a, tab, tab_bytes, w, nwin, e, el, ebits, sgn, out, n, st);
        case 4: return powexp_l<4>(fp, a, tab, tab_bytes, w, nwin, e, el, ebits, sgn, out, n, st);
    }
    return cudaErrorInvalidValue;
}
