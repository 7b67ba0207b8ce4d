// GF(2^8) = GF(2)[X]/(poly) arithmetic on one element, for device code and host tables (gf256.cuh: K5, gf_local.cuh: K15)
#pragma once
#include <cuda_runtime.h>

__host__ __device__ __forceinline__ unsigned gf_mul1(unsigned a, unsigned b, unsigned poly) {
    unsigned acc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        acc ^= (b & 1u) ? a : 0u;
        b >>= 1;
        a <<= 1;
        if (a & 0x100u) a ^= poly;
    }
    return acc & 0xFFu;
}

__host__ __device__ __forceinline__ unsigned gf_pow1(unsigned a, unsigned long long e, unsigned poly) {
    unsigned r = 1;
    for (int i = 63; i >= 0; i--) {
        r = gf_mul1(r, r, poly);
        if ((e >> i) & 1ull) r = gf_mul1(r, a, poly);
    }
    return r;
}
