// K15: GF(2^8) algebra on byte elements for the S-box steps of demos/np_aes.py (launcher inst_gf.cu).
//
//   k_gf_bits_compose      out[i] = sum_j x[i*l + j] X^j mod poly: np.sum(v << arange(l), axis=-1) of BinaryPolynomial
//                          values, reduced as the field array that receives it reduces (runtime.py:4415, 4483).  Reduction
//                          mod poly is a ring homomorphism from GF(2)[X], so summing the reduced terms is exact.
//   k_gf_binop_view        out = a_view (+ or *) b_view under any NumPy broadcast: K8's k_binop_view for one-byte elements
//   k_gf_matmul_batched    C[b] = A[b] @ B[b], a side of batch stride 0 broadcast (NumPy's matmul of stacks); a broadcast A
//                          of at most GF_MM_SMEM entries sits in shared memory, so (8, 8) @ (n, 8, 1) is one launch
//
// Products in the batched matmul go through log / exp tables of a generator g of GF(2^8)* built per call on the host
// (t.exp holds g^0 .. g^509, so log a + log b needs no reduction mod 255); bits_compose and binop_view use gf_mul1.
// Item numbers and offsets are 64-bit throughout.
#pragma once
#include "gf_ops.h"

#define GF_MM_SMEM 4096   // entries of a broadcast A kept in shared memory
#define GF_LOG0 0xFFFFu   // log entry of 0

struct GfLogExp {
    unsigned short log[256];
    unsigned char exp[512];
};

// a polynomial of degree < 32 reduced mod poly (degree 8)
__device__ __forceinline__ unsigned gf_reduce32(unsigned v, unsigned poly) {
#pragma unroll
    for (int b = 31; b >= 8; b--)
        if ((v >> b) & 1u) v ^= poly << (b - 8);
    return v;
}

// Terms are collected unreduced in chunks of 24 (x_j X^(j - j0) has degree < 31), each chunk is reduced once and scaled by
// X^j0 mod poly (x24 = X^24 mod poly advances the scale).  l == 8 on 8-byte aligned rows: one 64-bit load per row.
static __global__ void MPYC_LB k_gf_bits_compose(unsigned poly, unsigned x24, const unsigned char* __restrict__ x, size_t n,
                                                size_t l, unsigned char* __restrict__ out) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const bool word = l == 8 && (reinterpret_cast<uintptr_t>(x) & 7u) == 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += nth) {
        const unsigned char* row = x + i * l;
        unsigned acc = 0;
        if (word) {
            const unsigned long long v = *reinterpret_cast<const unsigned long long*>(row);
#pragma unroll
            for (int j = 0; j < 8; j++) acc ^= (unsigned)((v >> (8 * j)) & 0xFFu) << j;
            acc = gf_reduce32(acc, poly);
        } else {
            unsigned scale = 1;
            for (size_t j0 = 0; j0 < l; j0 += 24) {
                const size_t m = l - j0 < 24 ? l - j0 : 24;
                unsigned part = 0;
                for (size_t j = 0; j < m; j++) part ^= (unsigned)row[j0 + j] << j;
                part = gf_reduce32(part, poly);
                acc ^= j0 ? gf_mul1(part, scale, poly) : part;
                scale = gf_mul1(scale, x24, poly);
            }
        }
        out[i] = (unsigned char)acc;
    }
}

// out[w] = a[view a of w] (op) b[view b of w], op 0: + (XOR), 2: *; out contiguous in C order over p.ext
template <int OP>
static __global__ void MPYC_LB k_gf_binop_view(unsigned poly, BinopPlan p, const unsigned char* __restrict__ a,
                                              const unsigned char* __restrict__ b, unsigned char* __restrict__ out, size_t n) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n; w += nth) {
        long long ao = p.aoff, bo = p.boff;
        size_t r = w;
        for (int k = p.rank - 1; k >= 0; k--) {
            const size_t e = (size_t)p.ext[k];
            const long long c = (long long)(r % e);
            r /= e;
            ao += c * p.astr[k];
            bo += c * p.bstr[k];
        }
        const unsigned x = a[ao], y = b[bo];
        out[w] = (unsigned char)(OP == 2 ? gf_mul1(x, y, poly) : x ^ y);
    }
}

// one thread per output element (b, i, j) of the (batch, r, c) result, consecutive threads on consecutive outputs
template <bool SMEM_A>
static __global__ void MPYC_LB k_gf_matmul_batched(GfLogExp t, const unsigned char* __restrict__ A, size_t as,
                                                  const unsigned char* __restrict__ B, size_t bs, unsigned char* __restrict__ C,
                                                  size_t batch, size_t r, size_t k, size_t c) {
    __shared__ unsigned short lg[256];
    __shared__ unsigned char ex[512];
    __shared__ unsigned short la[SMEM_A ? GF_MM_SMEM : 1];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lg[i] = t.log[i];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) ex[i] = t.exp[i];
    __syncthreads();
    if (SMEM_A) {
        for (size_t i = threadIdx.x; i < r * k; i += blockDim.x) la[i] = lg[A[i]];
        __syncthreads();
    }
    const size_t nth = (size_t)gridDim.x * blockDim.x, rc = r * c, total = batch * rc;
    for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += nth) {
        const size_t bi = o / rc, rem = o - bi * rc, i = rem / c, j = rem - i * c;
        const unsigned char* a = A + bi * as + i * k;
        const unsigned char* bcol = B + bi * bs + j;
        unsigned acc = 0;
        for (size_t l = 0; l < k; l++) {
            const unsigned x = SMEM_A ? la[i * k + l] : lg[a[l]], y = lg[bcol[l * c]];
            if (x != GF_LOG0 && y != GF_LOG0) acc ^= ex[x + y];
        }
        C[o] = (unsigned char)acc;
    }
}
