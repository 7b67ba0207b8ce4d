// K15's launcher (gf_local.cuh): GF(2^8) bit composition, broadcast arithmetic and stacked matrix products.
#include "launch_impl.cuh"
#include "gf_local.cuh"

namespace {

// log / exp tables of the smallest generator of GF(2^8)* (an irreducible poly of degree 8 has one: the group is cyclic)
bool log_exp_tables(unsigned poly, GfLogExp& t) {
    for (unsigned g = 2; g < 256; g++) {
        if (gf_pow1(g, 85, poly) == 1 || gf_pow1(g, 51, poly) == 1 || gf_pow1(g, 15, poly) == 1) continue;   // 255 = 3 * 5 * 17
        unsigned x = 1;
        for (int i = 0; i < 512; i++) {
            t.exp[i] = (unsigned char)x;
            x = gf_mul1(x, g, poly);
        }
        t.log[0] = GF_LOG0;
        for (int i = 0; i < 255; i++) t.log[t.exp[i]] = (unsigned short)i;
        return true;
    }
    return false;
}

}  // namespace

cudaError_t launch_gf_bits_compose(unsigned poly, const unsigned char* x, size_t n, size_t l, unsigned char* out, cudaStream_t st) {
    const unsigned x24 = gf_pow1(2, 24, poly);
    return launch_kernel(k_gf_bits_compose, n, 0, st, poly, x24, x, n, l, out);
}

cudaError_t launch_gf_binop_view(unsigned poly, int op, const BinopPlan& p, const unsigned char* a, const unsigned char* b,
                                 unsigned char* out, cudaStream_t st) {
    size_t n = 1;
    for (int k = 0; k < p.rank; k++) n *= (size_t)p.ext[k];
    if (op == OP_MUL) return launch_kernel(k_gf_binop_view<2>, n, 0, st, poly, p, a, b, out, n);
    return launch_kernel(k_gf_binop_view<0>, n, 0, st, poly, p, a, b, out, n);
}

cudaError_t launch_gf_matmul_batched(unsigned poly, const unsigned char* A, size_t as, const unsigned char* B, size_t bs,
                                     unsigned char* C, size_t batch, size_t r, size_t k, size_t c, cudaStream_t st) {
    GfLogExp t;
    if (!log_exp_tables(poly, t)) return cudaErrorInvalidValue;
    const size_t n = batch * r * c;
    if (as == 0 && r * k <= GF_MM_SMEM)
        return launch_kernel(k_gf_matmul_batched<true>, n, 0, st, t, A, as, B, bs, C, batch, r, k, c);
    return launch_kernel(k_gf_matmul_batched<false>, n, 0, st, t, A, as, B, bs, C, batch, r, k, c);
}
