// K12: out[h] = base(h)^e[h] mod p with one exponent per element (PrimeFieldArray._pow with an exponent array,
// finfields.py:1409-1414; gmpy.powmod_exp_list, gmpy.py:288-290, in Runtime._np_pow_public_int_base_secret_integral_exponent,
// runtime.py:1389-1425).  Exponents are EL = ceil(B / 64) <= 4 little-endian 64-bit limbs per element, B the call's
// largest bit length; they are not reduced.  Two forms, both with a loop bound that is the same for every thread:
//   k_powexp_fixed  one public base: a fixed-base comb.  The host builds g(j, d) = base^(d 2^(w j)) for j < ceil(B / w),
//                   d < 2^w (and the same for base^-1 when a sign byte is given); each CTA stages the tables into shared
//                   memory with one TMA bulk copy.  An element costs ceil(B / w) - 1 table products and no squarings.
//   k_powexp_elem   per-element bases: left-to-right square-and-multiply over 2-bit digits with x, x^2, x^3 kept in
//                   registers -- two squarings and one product per digit (1.5 products per bit), branch-free.
// Products are the domain products of ff_arith.cuh (plain for pseudo-Mersenne fields, Montgomery for generic ones: the
// tables are staged in that form).  Offsets are 64-bit; element and exponent buffers need 8-byte alignment only.
#pragma once

// at most 128 registers: two CTAs of MPYC_THREADS per SM
#define MPYC_PE_LB __launch_bounds__(MPYC_THREADS, 2)

template <int L>
__device__ __forceinline__ void pe_load_smem(u32* v, const u64* p) {
#pragma unroll
    for (int q = 0; q < L; q++) {
        const u64 x = p[q];
        v[2 * q] = (u32)x;
        v[2 * q + 1] = (u32)(x >> 32);
    }
}

// tab: (1 or 2 tables) x nwin x 2^w entries of L limbs, tab_bytes in all; sgn (may be null): nonzero selects the second
// table (base^-1) for that element
template <int L, int KIND>
__global__ void MPYC_PE_LB
k_powexp_fixed(FieldParams f, const u64* __restrict__ tab, u32 tab_bytes, int w, int nwin, const u64* __restrict__ e, int el,
               const unsigned char* __restrict__ sgn, u64* __restrict__ out, size_t n) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    extern __shared__ __align__(16) u64 pe_tab[];
    __shared__ __align__(8) u64 mbar;
    tma_stage_table(pe_tab, tab, tab_bytes, &mbar);
    const u64 mask = (1ull << w) - 1;
    const size_t side = ((size_t)nwin << w) * L;   // limbs per table
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        const u64* eh = e + h * el;
        const u64* t = pe_tab + ((sgn != nullptr && sgn[h]) ? side : 0);
        // a 128-bit window (lo, hi) slides over the exponent limbs, so a digit may straddle two of them
        u64 lo = eh[0], hi = el > 1 ? eh[1] : 0;
        int q = 1, off = 0;
        u32 acc[N], x[N];
        for (int j = 0; j < nwin; j++) {
            const u64 d = (off ? (lo >> off) | (hi << (64 - off)) : lo) & mask;
            pe_load_smem<L>(x, t + (((size_t)j << w) + d) * L);
            if (j == 0) copy_n<N>(acc, x);
            else F::dmul(acc, acc, x, f);
            off += w;
            if (off >= 64) {
                off -= 64;
                lo = hi;
                q++;
                hi = q < el ? eh[q] : 0;
            }
        }
        F::from_dom(acc, acc, f);
        store_limbs<L, false>(out + h * L, acc);
    }
}

// npairs = ceil(B / 2) 2-bit digits, the same for every element (leading zero digits square 1)
template <int L, int KIND>
__global__ void MPYC_PE_LB
k_powexp_elem(FieldParams f, const u64* __restrict__ a, const u64* __restrict__ e, int el, int npairs, u64* __restrict__ out,
              size_t n) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        u32 x1[N], x2[N], x3[N], acc[N];
        load_limbs<L, false>(x1, a + h * L);
        F::to_dom(x1, x1, f);
        F::dmul(x2, x1, x1, f);
        F::dmul(x3, x2, x1, f);
        F::dom_one(acc, f);
        const u64* eh = e + h * el;
        int q = -1;
        u64 ew = 0;
        for (int t = npairs - 1; t >= 0; t--) {
            const int qt = (2 * t) >> 6;
            if (qt != q) {
                q = qt;
                ew = eh[q];
            }
            const u32 d = (u32)(ew >> ((2 * t) & 63)) & 3u;
            F::dmul(acc, acc, acc, f);
            F::dmul(acc, acc, acc, f);
            u32 m[N];
            F::dom_one(m, f);
            select_n<N>(m, x1, d == 1);
            select_n<N>(m, x2, d == 2);
            select_n<N>(m, x3, d == 3);
            F::dmul(acc, acc, m, f);
        }
        F::from_dom(acc, acc, f);
        store_limbs<L, false>(out + h * L, acc);
    }
}
