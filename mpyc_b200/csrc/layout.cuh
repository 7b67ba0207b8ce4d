// K8: copies between strided views of element arrays, and prime-field arithmetic on broadcast views.  Layout does not
// depend on the field: an element is E raw bytes (E = 1 for GF(2^8), 8L for L-limb prime fields).
//
//   k_copy_gather    dst_view <- src_view, one item per thread: the `runs` and `gather` forms
//   k_copy_permute   dst_view <- src_view through 32 x 32 element tiles in shared memory: the `permute` form
//   k_binop_view     out = a_view (op) b_view, out contiguous in C order; broadcast axes have stride 0
//
// A view is an element offset plus extents and signed element strides over axes ordered outer .. inner (rank <= 6,
// adjacent axes already collapsed by the host); one axis of a copy view may take its offsets from a device int64 index
// table (offset = index[c] * stride).  The launcher (inst_layout.cu) picks the form from the collapsed plan:
//   * runs: the innermost axis has stride 1 on both sides.  The plan is rescaled to units of U = 16, 8 or 1 bytes (the
//     widest that divides every offset, stride and row length in bytes, and both base addresses), so a warp moves
//     consecutive U-byte words of each run: k_copy_gather on U-byte items.
//   * permute: the destination's innermost axis has stride 1 but the source's does not, and another axis has source
//     stride +-1.  A tile is read along that axis and written along the innermost one, both coalesced (.T, swapaxes,
//     transpose(axes)).
//   * gather: everything else (steps other than +-1 or an index table on the innermost axis, flips): one element per item,
//     consecutive threads on consecutive innermost coordinates.
// Item numbers and the coordinate arithmetic of k_copy_gather are 32-bit when the item count fits (IDX = u32), else
// 64-bit; k_copy_permute numbers its tiles in 64 bits; offsets are always 64-bit.
#pragma once

#define MPYC_VIEW_RANK 6

// a copy between two views of equal extents
struct CopyPlan {
    int rank;
    int six, dix;                                  // axis whose src / dst offsets come from sidx / didx, or -1
    long long ext[MPYC_VIEW_RANK];
    long long sstr[MPYC_VIEW_RANK], dstr[MPYC_VIEW_RANK];
    long long soff, doff;
    const long long* sidx;
    const long long* didx;
};

// out (contiguous, extents ext) = a (op) b
struct BinopPlan {
    int rank;
    long long ext[MPYC_VIEW_RANK];
    long long astr[MPYC_VIEW_RANK], bstr[MPYC_VIEW_RANK];
    long long aoff, boff;
};

// one element of W words of type U
template <class U, int W>
struct ViewElem {
    U w[W];
};

// element offsets of item w (C order over ext) in both views, skipping the axes in `skip` (a bit mask)
template <class IDX>
__device__ __forceinline__ IDX view_offsets(const CopyPlan& p, IDX w, int last, int skip, long long& so, long long& dof) {
    for (int k = last; k >= 0; k--) {
        if ((skip >> k) & 1) continue;
        const IDX e = (IDX)p.ext[k];
        const IDX c = w % e;
        w /= e;
        so += (k == p.six ? p.sidx[c] : (long long)c) * p.sstr[k];
        dof += (k == p.dix ? p.didx[c] : (long long)c) * p.dstr[k];
    }
    return w;
}

template <class T, class IDX>
__global__ void MPYC_LB
k_copy_gather(CopyPlan p, const T* __restrict__ src, T* __restrict__ dst, IDX n) {
    const IDX nth = (IDX)gridDim.x * blockDim.x;
    for (IDX w = (IDX)blockIdx.x * blockDim.x + threadIdx.x; w < n; w += nth) {
        long long so = p.soff, dof = p.doff;
        view_offsets<IDX>(p, w, p.rank - 1, 0, so, dof);
        dst[dof] = src[so];
    }
}

// Tiles of 32 coordinates along axis `ax` (source stride +-1) by 32 along the innermost axis (destination stride 1);
// `tiles` counts them over all other axes.  A 32 x 8 thread block reads rows of the tile along ax and writes its columns
// along the innermost axis.
template <class T, class IDX>
__global__ void MPYC_LB
k_copy_permute(CopyPlan p, int ax, const T* __restrict__ src, T* __restrict__ dst, IDX tiles) {
    __shared__ T tile[32][33];
    const int in = p.rank - 1;
    const long long ea = p.ext[ax], ej = p.ext[in];
    const IDX na = (IDX)((ea + 31) / 32), nj = (IDX)((ej + 31) / 32);
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (IDX t = blockIdx.x; t < tiles; t += gridDim.x) {
        const IDX tj = t % nj, ta = (t / nj) % na;
        long long so = p.soff, dof = p.doff;
        view_offsets<IDX>(p, t / nj / na, in - 1, 1 << ax, so, dof);
        const long long a0 = (long long)ta * 32, j0 = (long long)tj * 32;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const long long j = j0 + ty + 8 * k, a = a0 + tx;
            if (j < ej && a < ea) tile[ty + 8 * k][tx] = src[so + a * p.sstr[ax] + j * p.sstr[in]];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const long long a = a0 + ty + 8 * k, j = j0 + tx;
            if (a < ea && j < ej) dst[dof + a * p.dstr[ax] + j] = tile[tx][ty + 8 * k];
        }
    }
}

// out[w] = a[view a of w] (op) b[view b of w]: K1's arithmetic on operands read in place (a broadcast operand is never
// materialised); out is written in order, so the warp's stores are contiguous.
template <int L, int KIND, int OP>
__global__ void MPYC_LB
k_binop_view(FieldParams f, BinopPlan p, const u64* __restrict__ a, const u64* __restrict__ b, u64* __restrict__ out, size_t n) {
    constexpr int N = 2 * L;
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
        u32 x[N], y[N], z[N];
        load_limbs<L, false>(x, a + ao * L);
        load_limbs<L, false>(y, b + bo * L);
        apply_op<L, KIND, OP>(z, x, y, f);
        store_limbs<L, false>(out + w * L, z);
    }
}
