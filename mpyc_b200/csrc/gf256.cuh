// GF(2^8) = GF(2)[X]/(poly) kernels: one byte per element (the AES field of demos/np_aes.py when
// poly = 283).  Replaces BinaryFieldArray over gfpx.BinaryPolynomial objects
// (reference mpyc/finfields.py:1542-1563, mpyc/gfpx.py:983-1045,1085-1096) and the GF(2^8)
// instances of thresha.np_random_split / np_recombine (points are the field elements whose
// integer encoding is the party index, thresha.py:54,61).
//
// Bulk kernels work on 8 packed bytes per 64-bit word (SWAR shift-and-add multiplication);
// constant multipliers (Vandermonde / Lagrange entries) only XOR the needed x^b multiples.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "gf_ops.h"

extern std::atomic<unsigned long long> g_mpyc_launches;
int mpyc_grid_size(const void* kernel, size_t items, size_t dyn_smem);

#define GF_THREADS 256
#define GF_MAX_TAB 2048
#define GF_LADDER_T 4     // degrees up to this keep the x^b multiples of the coefficient words in registers

struct GfTab {
    unsigned char v[GF_MAX_TAB];
};
struct GfRows {
    const unsigned char* p[64];
};

// 8 bytes at a time: multiply every byte of a by x
__device__ __forceinline__ unsigned long long gf_xtime8(unsigned long long a, unsigned long long red) {
    unsigned long long hi = (a >> 7) & 0x0101010101010101ull;
    return ((a & 0x7F7F7F7F7F7F7F7Full) << 1) ^ (hi * red);
}
// bytewise product of two packed words
__device__ __forceinline__ unsigned long long gf_mul8(unsigned long long a, unsigned long long b, unsigned long long red) {
    unsigned long long acc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        unsigned long long m = ((b >> i) & 0x0101010101010101ull) * 0xFFull;
        acc ^= a & m;
        a = gf_xtime8(a, red);
    }
    return acc;
}
// packed word times one constant byte c (warp-uniform)
__device__ __forceinline__ unsigned long long gf_mulc8(unsigned long long a, unsigned c, unsigned long long red) {
    unsigned long long acc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if ((c >> i) & 1u) acc ^= a;
        if ((c >> (i + 1)) == 0) break;   // c is warp-uniform: no xtime beyond its top bit
        a = gf_xtime8(a, red);
    }
    return acc;
}

// ---- elementwise: op 0/1 xor, 2 mul, 3 neg(copy); scalar >= 0 broadcasts b -----------------------
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_binop(unsigned poly, int op, const unsigned char* __restrict__ a, const unsigned char* __restrict__ b, int scalar,
           unsigned char* __restrict__ out, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long red = poly & 0xFFu;
    const bool al = (((uintptr_t)a | (uintptr_t)out | (scalar >= 0 || op == 3 ? 0 : (uintptr_t)b)) & 7u) == 0;
    const size_t nw = al ? n / 8 : 0;
    for (size_t w = tid; w < nw; w += nth) {
        unsigned long long x = ((const unsigned long long*)a)[w];
        unsigned long long y = (scalar >= 0) ? (unsigned long long)scalar * 0x0101010101010101ull
                                             : (op == 3 ? 0ull : ((const unsigned long long*)b)[w]);
        unsigned long long r = op == 2 ? gf_mul8(x, y, red) : (op == 3 ? x : x ^ y);
        ((unsigned long long*)out)[w] = r;
    }
    for (size_t h = nw * 8 + tid; h < n; h += nth) {
        unsigned x = a[h], y = scalar >= 0 ? (unsigned)scalar : (op == 3 ? 0u : b[h]);
        out[h] = (unsigned char)(op == 2 ? gf_mul1(x, y, poly) : (op == 3 ? x : x ^ y));
    }
}

static __global__ void __launch_bounds__(GF_THREADS)
k_gf_pow(unsigned poly, const unsigned char* __restrict__ a, unsigned long long e, unsigned char* __restrict__ out,
         int* zero_flag, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        unsigned x = a[h];
        if (zero_flag && x == 0) *zero_flag = 1;
        out[h] = (unsigned char)gf_pow1(x, e, poly);
    }
}

// ---- split: shares[i][h] = sum_j (i+1)^j M[j][h]; tab[i*(t+1)+j] = (i+1)^j ------------------------
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_split(unsigned poly, GfTab tab, const unsigned char* __restrict__ secrets, const unsigned char* __restrict__ coeffs,
           size_t cstride, unsigned char* __restrict__ shares, size_t sstride, size_t n, int t, int m) {
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long red = poly & 0xFFu;
    const bool al = ((((uintptr_t)secrets | (uintptr_t)shares | (t ? (uintptr_t)coeffs : 0)) & 7u) == 0) &&
                    (cstride % 8 == 0 || t <= 1) && (sstride % 8 == 0 || m <= 1);
    const size_t nw = al ? n / 8 : 0;
    if (t <= GF_LADDER_T) {
        // x^b multiples of every coefficient word once (only up to the top bit any share needs for that
        // column), then each share only XORs the multiples selected by the bits of its (warp-uniform)
        // Vandermonde entries
        int depth[GF_LADDER_T];
#pragma unroll
        for (int j = 0; j < GF_LADDER_T; j++) {
            unsigned any = 0;
            if (j < t)
                for (int i = 0; i < m; i++) any |= tab.v[i * (t + 1) + j + 1];
            depth[j] = 32 - __clz(any | 1u);
        }
        for (size_t w = tid; w < nw; w += nth) {
            unsigned long long lad[GF_LADDER_T][8];
            const unsigned long long s0 = ((const unsigned long long*)secrets)[w];
#pragma unroll
            for (int j = 0; j < GF_LADDER_T; j++) {
                if (j < t) {
                    unsigned long long x = ((const unsigned long long*)(coeffs + (size_t)j * cstride))[w];
#pragma unroll
                    for (int b = 0; b < 8; b++) {
                        lad[j][b] = x;
                        if (b + 1 < depth[j]) x = gf_xtime8(x, red);
                    }
                }
            }
            for (int i = 0; i < m; i++) {
                unsigned long long acc = s0;
#pragma unroll
                for (int j = 0; j < GF_LADDER_T; j++) {
                    if (j < t) {
                        const unsigned c = tab.v[i * (t + 1) + j + 1];
#pragma unroll
                        for (int b = 0; b < 8; b++)
                            if ((c >> b) & 1u) acc ^= lad[j][b];
                    }
                }
                ((unsigned long long*)(shares + (size_t)i * sstride))[w] = acc;
            }
        }
    } else {
        for (size_t w = tid; w < nw; w += nth) {
            for (int i = 0; i < m; i++) {
                unsigned long long acc = ((const unsigned long long*)secrets)[w];
                for (int j = 1; j <= t; j++) {
                    unsigned long long x = ((const unsigned long long*)(coeffs + (size_t)(j - 1) * cstride))[w];
                    acc ^= gf_mulc8(x, tab.v[i * (t + 1) + j], red);
                }
                ((unsigned long long*)(shares + (size_t)i * sstride))[w] = acc;
            }
        }
    }
    for (size_t h = nw * 8 + tid; h < n; h += nth) {
        for (int i = 0; i < m; i++) {
            unsigned acc = secrets[h];
            for (int j = 1; j <= t; j++) acc ^= gf_mul1(coeffs[(size_t)(j - 1) * cstride + h], tab.v[i * (t + 1) + j], poly);
            shares[(size_t)i * sstride + h] = (unsigned char)acc;
        }
    }
}

// ---- split, vector form: 16 bytes (two packed words) per thread and access, t <= GF_HORNER_T -------------
// Horner in the point: share_i = s + x_i (c_1 + x_i (c_2 + ... x_i c_t)), x_i = i+1.  Multiplying by the
// warp-uniform constant x_i needs only bitlen(x_i)-1 xtime steps (none for party 1, one for parties 2 and 3),
// so the demo shape m=3, t=1 costs 2 xtime steps per 16 elements' worth of words and the kernel streams.
#define GF_HORNER_T 4

struct __align__(16) GfW2 {
    unsigned long long a, b;
};
__device__ __forceinline__ GfW2 gf_ld16(const unsigned char* p) {
    GfW2 v;
    asm("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.a), "=l"(v.b) : "l"(p));
    return v;
}
__device__ __forceinline__ void gf_st16(unsigned char* p, GfW2 v) {
    asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(v.a), "l"(v.b) : "memory");
}
// v * x for a warp-uniform constant x of nb significant bits (1 <= nb <= 8)
__device__ __forceinline__ GfW2 gf_mulc16(GfW2 v, unsigned x, int nb, unsigned long long red) {
    GfW2 acc = {0ull, 0ull};
    for (int b = 0; b < nb; b++) {
        if ((x >> b) & 1u) {
            acc.a ^= v.a;
            acc.b ^= v.b;
        }
        if (b + 1 < nb) {
            v.a = gf_xtime8(v.a, red);
            v.b = gf_xtime8(v.b, red);
        }
    }
    return acc;
}

// shares of one 16-byte group from its registers
template <int T>
__device__ __forceinline__ void gf_split_group(const GfW2& s0, const GfW2* c, unsigned char* __restrict__ shares, size_t sstride,
                                               size_t g, int m, unsigned long long red) {
    for (int i = 0; i < m; i++) {
        const unsigned x = (unsigned)(i + 1);
        const int nb = 32 - __clz(x);
        GfW2 acc = s0;
        if constexpr (T > 0) {
            acc = c[T - 1];
#pragma unroll
            for (int j = T - 1; j >= 0; j--) {
                acc = gf_mulc16(acc, x, nb, red);
                const GfW2 nxt = j > 0 ? c[j - 1] : s0;
                acc.a ^= nxt.a;
                acc.b ^= nxt.b;
            }
        }
        gf_st16(shares + (size_t)i * sstride + 16 * g, acc);
    }
}

#ifndef GF_SPLIT_PREFETCH
#define GF_SPLIT_PREFETCH 1   // software-pipelined main loop (0: GF_SPLIT_U groups per trip, all loads first)
#endif
#ifndef GF_SPLIT_U
#define GF_SPLIT_U 2   // 16-byte groups in flight per thread (ncu round 1: long-scoreboard bound at one group, 0.84-0.86 of peak)
#endif

template <int T>
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_split_vec(unsigned poly, const unsigned char* __restrict__ secrets, const unsigned char* __restrict__ coeffs,
               size_t cstride, unsigned char* __restrict__ shares, size_t sstride, size_t ngroups, int m) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const unsigned long long red = poly & 0xFFu;
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
#if GF_SPLIT_PREFETCH
    // software pipeline (as k_split for 1-limb prime fields): the T+1 input vectors of group g+nth are requested before
    // the shares of group g are computed and stored
    GfW2 s0 = {0ull, 0ull}, c[T > 0 ? T : 1];
    auto fetch = [&](GfW2& s, GfW2* cc, size_t grp) {
        s = gf_ld16(secrets + 16 * grp);
#pragma unroll
        for (int j = 0; j < T; j++) cc[j] = gf_ld16(coeffs + (size_t)j * cstride + 16 * grp);
    };
    if (g < ngroups) fetch(s0, c, g);
    for (; g < ngroups; g += nth) {
        const bool more = g + nth < ngroups;
        GfW2 s1 = {0ull, 0ull}, c1[T > 0 ? T : 1];
        if (more) fetch(s1, c1, g + nth);
        gf_split_group<T>(s0, c, shares, sstride, g, m, red);
        s0 = s1;
#pragma unroll
        for (int j = 0; j < T; j++) c[j] = c1[j];
    }
#else
    constexpr int U = GF_SPLIT_U;
    for (; g + (U - 1) * nth < ngroups; g += U * nth) {      // all loads of the U groups are issued before the first xtime
        GfW2 s0[U];
        GfW2 c[U][T > 0 ? T : 1];
#pragma unroll
        for (int u = 0; u < U; u++) {
            s0[u] = gf_ld16(secrets + 16 * (g + u * nth));
#pragma unroll
            for (int j = 0; j < T; j++) c[u][j] = gf_ld16(coeffs + (size_t)j * cstride + 16 * (g + u * nth));
        }
#pragma unroll
        for (int u = 0; u < U; u++) gf_split_group<T>(s0[u], c[u], shares, sstride, g + u * nth, m, red);
    }
    for (; g < ngroups; g += nth) {
        const GfW2 s0 = gf_ld16(secrets + 16 * g);
        GfW2 c[T > 0 ? T : 1];
#pragma unroll
        for (int j = 0; j < T; j++) c[j] = gf_ld16(coeffs + (size_t)j * cstride + 16 * g);
        gf_split_group<T>(s0, c, shares, sstride, g, m, red);
    }
#endif
}

// ---- recombine, vector form (width 1): 16 bytes per thread and access ----------------------------------
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_recombine_vec(unsigned poly, GfTab lam, GfRows rows, int k, unsigned char* __restrict__ out, size_t ngroups) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const unsigned long long red = poly & 0xFFu;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += nth) {
        GfW2 acc = {0ull, 0ull};
        for (int i0 = 0; i0 < k; i0 += 4) {
            GfW2 v[4];
#pragma unroll
            for (int b = 0; b < 4; b++)
                if (i0 + b < k) v[b] = gf_ld16(rows.p[i0 + b] + 16 * g);
#pragma unroll
            for (int b = 0; b < 4; b++)
                if (i0 + b < k) {
                    const unsigned l = lam.v[i0 + b];
                    const GfW2 t = gf_mulc16(v[b], l, 32 - __clz(l | 1u), red);
                    acc.a ^= t.a;
                    acc.b ^= t.b;
                }
        }
        gf_st16(out + 16 * g, acc);
    }
}

// ---- recombine: out[r][h] = sum_i lam[r*k+i] * rows[i][h] --------------------------------------------
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_recombine(unsigned poly, GfTab lam, GfRows rows, int k, int width, unsigned char* __restrict__ out, size_t ostride,
               size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long red = poly & 0xFFu;
    uintptr_t bits = (uintptr_t)out;
    for (int i = 0; i < k; i++) bits |= (uintptr_t)rows.p[i];
    const bool al = ((bits & 7u) == 0) && (ostride % 8 == 0 || width <= 1);
    const size_t nw = al ? n / 8 : 0;
    if (width == 1) {
        for (size_t w = tid; w < nw; w += nth) {
            unsigned long long acc = 0;
            for (int i = 0; i < k; i++) acc ^= gf_mulc8(((const unsigned long long*)rows.p[i])[w], lam.v[i], red);
            ((unsigned long long*)out)[w] = acc;
        }
    } else {
        for (size_t w = tid; w < nw; w += nth) {
            for (int r = 0; r < width; r++) {
                unsigned long long acc = 0;
                for (int i = 0; i < k; i++) acc ^= gf_mulc8(((const unsigned long long*)rows.p[i])[w], lam.v[r * k + i], red);
                ((unsigned long long*)(out + (size_t)r * ostride))[w] = acc;
            }
        }
    }
    for (size_t h = nw * 8 + tid; h < n; h += nth) {
        for (int r = 0; r < width; r++) {
            unsigned acc = 0;
            for (int i = 0; i < k; i++) acc ^= gf_mul1(rows.p[i][h], lam.v[r * k + i], poly);
            out[(size_t)r * ostride + h] = (unsigned char)acc;
        }
    }
}

// ---- PRSS: out[h] = sum_S coef[S] * sum_j (bytes[S][h*d+j] & mask) * w[j]; tab = coef | w --------------
// mask = 2^b - 1 for a PRF bound 2^b <= 256 (thresha.py:261: chunk % bound; b = 1 for runtime.random_bits on
// characteristic-2 fields, runtime.py:4138,4218), 0xFF for the full byte.
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_prss(unsigned poly, GfTab tab, const unsigned char* __restrict__ bytes, size_t subset_stride, int nsub, int d,
          unsigned mask, unsigned char* __restrict__ out, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        unsigned acc = 0;
        for (int S = 0; S < nsub; S++) {
            unsigned y = 0;
            for (int j = 0; j < d; j++) y ^= gf_mul1(bytes[(size_t)S * subset_stride + h * d + j] & mask, tab.v[nsub + j], poly);
            acc ^= gf_mul1(y, tab.v[S], poly);
        }
        out[h] = (unsigned char)acc;
    }
}

static __global__ void __launch_bounds__(GF_THREADS)
k_gf_fill(unsigned long long base, unsigned char* __restrict__ out, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) {
        unsigned long long z = base + h + 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        out[h] = (unsigned char)((z ^ (z >> 31)) & 0xFF);
    }
}

static __global__ void __launch_bounds__(GF_THREADS)
k_gf_mismatch(const unsigned char* __restrict__ a, const unsigned char* __restrict__ b, size_t n, unsigned long long* count) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    unsigned long long local = 0;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += nth) local += a[h] != b[h];
    for (int off = 16; off > 0; off >>= 1) local += __shfl_down_sync(0xffffffffu, local, off);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

// ---- matmul: C[r x c] = A[r x k] @ B[k x c] over GF(2^8), one thread per output element -----------------
static __global__ void __launch_bounds__(GF_THREADS)
k_gf_matmul(unsigned poly, const unsigned char* __restrict__ A, const unsigned char* __restrict__ B,
            unsigned char* __restrict__ C, size_t r, size_t k, size_t c) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < r * c; o += nth) {
        const size_t i = o / c, j = o % c;
        unsigned acc = 0;
        for (size_t l = 0; l < k; l++) acc ^= gf_mul1(A[i * k + l], B[l * c + j], poly);
        C[o] = (unsigned char)acc;
    }
}

// ---- host wrappers ---------------------------------------------------------------------------------

#define GF_LAUNCH(kernel, items, st, ...)                                                   \
    do {                                                                                    \
        if ((items) == 0) return cudaSuccess;                                               \
        int grid__ = mpyc_grid_size((const void*)kernel, (items), 0);                       \
        if (grid__ <= 0) return cudaErrorLaunchFailure;                                     \
        kernel<<<grid__, GF_THREADS, 0, st>>>(__VA_ARGS__);                                 \
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);                            \
        return cudaGetLastError();                                                          \
    } while (0)

static inline cudaError_t gf256_binop(unsigned poly, int op, const unsigned char* a, const unsigned char* b, int scalar,
                                      unsigned char* out, size_t n, cudaStream_t st) {
    GF_LAUNCH(k_gf_binop, (n + 7) / 8, st, poly, op, a, b, scalar, out, n);
}
static inline cudaError_t gf256_pow(unsigned poly, const unsigned char* a, unsigned long long e, unsigned char* out,
                                    int* zero_flag, size_t n, cudaStream_t st) {
    GF_LAUNCH(k_gf_pow, n, st, poly, a, e, out, zero_flag, n);
}
static inline cudaError_t gf256_split(unsigned poly, const unsigned char* secrets, const unsigned char* coeffs,
                                      size_t cstride, unsigned char* shares, size_t sstride, size_t n, int t, int m,
                                      cudaStream_t st) {
    if ((size_t)m * (t + 1) > GF_MAX_TAB) return cudaErrorNotSupported;
    GfTab tab;
    for (int i = 0; i < m; i++) {
        unsigned x = 1;
        for (int j = 0; j <= t; j++) {
            tab.v[i * (t + 1) + j] = (unsigned char)x;
            x = gf_mul1(x, (unsigned)(i + 1), poly);
        }
    }
    // vector form for the bulk when every row is 16-byte aligned; the scalar kernel finishes the tail
    const bool al16 = ((((uintptr_t)secrets | (uintptr_t)shares | (t ? (uintptr_t)coeffs : 0)) & 15u) == 0) &&
                      (cstride % 16 == 0 || t <= 1) && (sstride % 16 == 0 || m <= 1);
    if (al16 && t <= GF_HORNER_T && m <= 255 && n >= 16 && (n % 16 == 0 || n >= 4096)) {   // small ragged calls: one launch
        const size_t groups = n / 16, done = groups * 16;
        int grid = 0;
        cudaError_t e = cudaSuccess;
#define GF_SPLIT_VEC(T)                                                                                           \
    case T:                                                                                                       \
        grid = mpyc_grid_size((const void*)k_gf_split_vec<T>, groups, 0);                                         \
        if (grid <= 0) return cudaErrorLaunchFailure;                                                             \
        k_gf_split_vec<T><<<grid, GF_THREADS, 0, st>>>(poly, secrets, coeffs, cstride, shares, sstride, groups, m); \
        break
        switch (t) {
            GF_SPLIT_VEC(0);
            GF_SPLIT_VEC(1);
            GF_SPLIT_VEC(2);
            GF_SPLIT_VEC(3);
            GF_SPLIT_VEC(4);
        }
#undef GF_SPLIT_VEC
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
        if (e != cudaSuccess || done == n) return e;
        // tail (< 16 elements): byte path of the scalar kernel on the remaining columns
        GF_LAUNCH(k_gf_split, 1, st, poly, tab, secrets + done, coeffs ? coeffs + done : coeffs, cstride, shares + done,
                  sstride, n - done, t, m);
    }
    GF_LAUNCH(k_gf_split, (n + 7) / 8, st, poly, tab, secrets, coeffs, cstride, shares, sstride, n, t, m);
}
// Lagrange coefficients over GF(2^8); returns 0 or MPYC_B200_EZERODIV (-3)
static inline int gf256_lambda(unsigned poly, const int64_t* xs, int k, const int64_t* x_rs, int width, unsigned char* lam) {
    for (int r = 0; r < width; r++)
        for (int i = 0; i < k; i++) {
            unsigned num = 1, den = 1;
            for (int j = 0; j < k; j++) {
                if (j == i) continue;
                num = gf_mul1(num, (unsigned)((x_rs[r] ^ xs[j]) & 0xFF), poly);
                den = gf_mul1(den, (unsigned)((xs[i] ^ xs[j]) & 0xFF), poly);
            }
            if (den == 0) return -3;
            lam[r * k + i] = (unsigned char)gf_mul1(num, gf_pow1(den, 254, poly), poly);
        }
    return 0;
}
static inline cudaError_t gf256_recombine(unsigned poly, const unsigned char* const* rows, int k, int width,
                                          const unsigned char* lam, unsigned char* out, size_t ostride, size_t n,
                                          cudaStream_t st) {
    if ((size_t)k * width > GF_MAX_TAB || k > 64) return cudaErrorNotSupported;
    GfTab tab;
    for (int i = 0; i < k * width; i++) tab.v[i] = lam[i];
    GfRows r;
    for (int i = 0; i < 64; i++) r.p[i] = i < k ? rows[i] : nullptr;
    uintptr_t bits = (uintptr_t)out;
    for (int i = 0; i < k; i++) bits |= (uintptr_t)rows[i];
    if (width == 1 && (bits & 15u) == 0 && n >= 16 && (n % 16 == 0 || n >= 4096)) {
        const size_t groups = n / 16, done = groups * 16;
        int grid = mpyc_grid_size((const void*)k_gf_recombine_vec, groups, 0);
        if (grid <= 0) return cudaErrorLaunchFailure;
        k_gf_recombine_vec<<<grid, GF_THREADS, 0, st>>>(poly, tab, r, k, out, groups);
        g_mpyc_launches.fetch_add(1, std::memory_order_relaxed);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess || done == n) return e;
        for (int i = 0; i < k; i++) r.p[i] += done;
        GF_LAUNCH(k_gf_recombine, 1, st, poly, tab, r, k, width, out + done, ostride, n - done);
    }
    GF_LAUNCH(k_gf_recombine, (n + 7) / 8, st, poly, tab, r, k, width, out, ostride, n);
}
static inline cudaError_t gf256_prss(unsigned poly, const unsigned char* bytes, size_t subset_stride, int nsub, int d,
                                     const unsigned char* coef_w, unsigned mask, unsigned char* out, size_t n, cudaStream_t st) {
    if ((size_t)nsub + d > GF_MAX_TAB) return cudaErrorNotSupported;
    GfTab tab;
    for (int i = 0; i < nsub + d; i++) tab.v[i] = coef_w[i];
    GF_LAUNCH(k_gf_prss, n, st, poly, tab, bytes, subset_stride, nsub, d, mask, out, n);
}
static inline cudaError_t gf256_fill(unsigned long long base, unsigned char* out, size_t n, cudaStream_t st) {
    GF_LAUNCH(k_gf_fill, n, st, base, out, n);
}
static inline cudaError_t gf256_mismatch(const unsigned char* a, const unsigned char* b, size_t n, unsigned long long* count,
                                         cudaStream_t st) {
    GF_LAUNCH(k_gf_mismatch, n, st, a, b, n, count);
}
static inline cudaError_t gf256_matmul(unsigned poly, const unsigned char* A, const unsigned char* B, unsigned char* C,
                                       size_t r, size_t k, size_t c, cudaStream_t st) {
    GF_LAUNCH(k_gf_matmul, r * c, st, poly, A, B, C, r, k, c);
}
