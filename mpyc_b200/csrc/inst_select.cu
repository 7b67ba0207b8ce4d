// K11's select launcher (select.cuh): 16-byte element accesses for even L when out and every store side are 16-byte
// aligned, 8-byte accesses otherwise (views that start mid-buffer).
#include "launch_impl.cuh"
#include "select.cuh"

namespace {

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <int L>
cudaError_t select_l(const FieldParams& fp, const unsigned char* mask, bool invert, const SelectSide& xs, const SelectSide& ys,
                     u64* out, size_t n, cudaStream_t st) {
    const bool w16 = L % 2 == 0 && aligned16(out) && (!xs.x || aligned16(xs.x)) && (!ys.x || aligned16(ys.x));
    const int inv = invert ? 1 : 0;
    if constexpr (L % 2 == 0) {
        if (w16) {
#define M(K) return launch_kernel(k_select<L, K, true>, n, 0, st, fp, mask, inv, xs, ys, out, n)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return launch_kernel(k_select<L, K, false>, n, 0, st, fp, mask, inv, xs, ys, out, n)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

SelectSide side(const u64* x, const u64* s, const u64* t, int L) {
    SelectSide sd = {};
    sd.x = x;
    bool unit = true;
    for (int i = 0; i < L; i++) {
        sd.s[i] = s[i];
        sd.t[i] = t[i];
        unit = unit && s[i] == (i == 0 ? 1u : 0u) && t[i] == 0;
    }
    sd.unit = unit ? 1 : 0;
    return sd;
}

}  // namespace

cudaError_t launch_select(const FieldParams& fp, const unsigned char* mask, bool invert, const u64* x, const u64* xs,
                          const u64* xt, const u64* y, const u64* ys, const u64* yt, u64* out, size_t n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const SelectSide a = side(x, xs, xt, (int)fp.L), b = side(y, ys, yt, (int)fp.L);
    switch (fp.L) {
        case 1: return select_l<1>(fp, mask, invert, a, b, out, n, st);
        case 2: return select_l<2>(fp, mask, invert, a, b, out, n, st);
        case 3: return select_l<3>(fp, mask, invert, a, b, out, n, st);
        case 4: return select_l<4>(fp, mask, invert, a, b, out, n, st);
    }
    return cudaErrorInvalidValue;
}
