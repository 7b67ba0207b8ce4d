// K10's launcher (conv.cuh).  The shorter operand supplies the taps.  Every L runs TM = 2 outputs per thread: k_conv
// then needs 128 registers or fewer (2 CTAs per SM) and no spills for L = 1..4, and on an H100 it was faster than TM = 4
// at L = 1 and 2 (at TM = 4 L = 2 takes 138-216 registers, one CTA per SM; DESIGN.md section 5).  TM = 8 spills.  The
// form is chosen from the shapes, L and the SM count:
//   tiles: one work item per run of T = MPYC_THREADS * TM outputs, over all the taps that meet it;
//   split: when the window has too few runs to fill the machine (two length-4096 operands give 8191 outputs, a few
//          runs), the taps are cut into slices of whole chunks, each (slice, run) writes its partial sums to
//          stream-ordered scratch and K7 adds the slices up, as split-k K1c does (Launch::matmul).
#include "launch_impl.cuh"
#include "conv.cuh"

namespace {

template <int L>
cudaError_t conv_l(const FieldParams& fp, const u64* a, size_t m, const u64* b, size_t n, size_t lo, size_t count, u64* c,
                   cudaStream_t st) {
    constexpr int TM = 2;
    constexpr size_t T = (size_t)MPYC_THREADS * TM;
    const bool a_taps = m <= n;
    const u64* H = a_taps ? a : b;
    const u64* X = a_taps ? b : a;
    const size_t s = a_taps ? m : n, g = a_taps ? n : m;
    const size_t tiles = (count + T - 1) / T;
    // split when the runs alone cannot fill the machine: aim at ~2 CTAs per SM, slices of whole chunks
    size_t nslices = 1;
    const size_t want = (size_t)mpyc_sm_count() * 2;
    const size_t chunks = (s + MPYC_CV_KT - 1) / MPYC_CV_KT;
    if (tiles < want && chunks >= 2) nslices = std::min((want + tiles - 1) / tiles, chunks);
    const size_t slice = (chunks + nslices - 1) / nslices * MPYC_CV_KT;
    nslices = (s + slice - 1) / slice;
    u64* dst = c;
    u64* part = nullptr;
    if (nslices > 1) {
        cudaError_t e = cudaMallocAsync(&part, nslices * count * L * sizeof(u64), st);
        if (e != cudaSuccess) return e;
        dst = part;
    }
    cudaError_t e = cudaErrorInvalidValue;
#define M(K) e = launch_kernel(k_conv<L, K, TM>, tiles * nslices * MPYC_THREADS, 0, st, fp, X, g, H, s, dst, lo, count, slice, nslices)
    switch (fp.kind) {
        case KIND_GENERIC: M(KIND_GENERIC); break;
        case KIND_PM_ALIGNED: M(KIND_PM_ALIGNED); break;
        case KIND_PM_SHIFT: M(KIND_PM_SHIFT); break;
        default: break;
    }
#undef M
    if (e == cudaSuccess && nslices > 1) e = Launch<L>::sum_axis(fp, part, c, 1, nslices, count, nullptr, st);   // the slices' sum
    if (part) cudaFreeAsync(part, st);
    return e;
}

}  // namespace

cudaError_t launch_convolve(const FieldParams& fp, const u64* a, size_t m, const u64* b, size_t n, size_t lo, size_t count,
                            u64* c, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    switch (fp.L) {
        case 1: return conv_l<1>(fp, a, m, b, n, lo, count, c, st);
        case 2: return conv_l<2>(fp, a, m, b, n, lo, count, c, st);
        case 3: return conv_l<3>(fp, a, m, b, n, lo, count, c, st);
        case 4: return conv_l<4>(fp, a, m, b, n, lo, count, c, st);
    }
    return cudaErrorInvalidValue;
}
