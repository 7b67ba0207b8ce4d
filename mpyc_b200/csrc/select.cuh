// K11: k_select -- out[h] = (mask[h] != 0) != invert ? X(h) : Y(h), the np.where of field arrays and raw share values
// (finfields.py:766-819 via np.where; Runtime._np_is_zero, runtime.py:3614-3615; Runtime.np_lsb, runtime.py:1819).
// Each side is a store read through a public affine map, x[h] * s + t (s == 1, t == 0 skips the arithmetic), or the
// public constant t when its store is null -- so a raw value with a pending `1 - z` is selected without a flush launch
// first.  Only the chosen side is read and computed.  An HBM streamer like the K6 kernels: one element per thread and
// trip, 16-byte accesses for even L when every element buffer is 16-byte aligned (W16), 8-byte accesses otherwise, so
// operands need only 8-byte alignment.  Offsets are 64-bit.
#pragma once

struct SelectSide {
    u64 s[4];
    u64 t[4];
    const u64* x;      // null: the constant t
    int unit;          // s == 1 and t == 0: the store as it is
};

template <int L, bool W16>
__device__ __forceinline__ void sel_load(u32* v, const u64* p) {
    if constexpr (W16) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) ldg_v4(v + 4 * q, p + 2 * q);
    } else {
        load_limbs<L, false>(v, p);
    }
}
template <int L, bool W16>
__device__ __forceinline__ void sel_store(u64* p, const u32* v) {
    if constexpr (W16) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) stg_v4(p + 2 * q, v + 4 * q);
    } else {
        store_limbs<L, false>(p, v);
    }
}

template <int L, int KIND, bool W16>
__device__ __forceinline__ void sel_side(u32* r, const SelectSide& sd, size_t h, const FieldParams& f) {
    constexpr int N = 2 * L;
    if (sd.x == nullptr) {
#pragma unroll
        for (int i = 0; i < N; i++) r[i] = as32(sd.t)[i];
        return;
    }
    sel_load<L, W16>(r, sd.x + h * L);
    if (sd.unit) return;
    u32 s[N], t[N], pr[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        s[i] = as32(sd.s)[i];
        t[i] = as32(sd.t)[i];
    }
    Fp<L, KIND>::mul(pr, r, s, f);
    Fp<L, KIND>::add(r, pr, t, f);
}

template <int L, int KIND, bool W16>
__global__ void MPYC_LB
k_select(FieldParams f, const unsigned char* __restrict__ mask, int invert, SelectSide xs, SelectSide ys, u64* __restrict__ out,
         size_t n) {
    static_assert(!W16 || L % 2 == 0, "16-byte accesses need an even limb count");
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        const bool pick_x = (mask[h] != 0) != (invert != 0);
        u32 r[N];
        if (pick_x) sel_side<L, KIND, W16>(r, xs, h, f);
        else sel_side<L, KIND, W16>(r, ys, h, f);
        sel_store<L, W16>(out + h * L, r);
    }
}
