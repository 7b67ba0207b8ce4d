// K6: the local algebra of MPyC's protocols that the reference runs on RAW share values in NumPy object loops
// (SURVEY 8f N3 / N4) -- integer work between two openings that never touches the network:
//
//   k_fma            a*b + c, a*a + c          np_random_bits: `_r.value**2 + z.value`             runtime.py:4252
//   k_axpb           a*s + t (public s, t)     np_random_bits: `bits += 1; bits *= (p+1)>>1; bits <<= f`   :4267-4271
//                                              and every `x << f`, `x + (1 << l)`, `(z << 1) - 1` on raw values
//   k_low_bits       a & (2^b - 1)             np_trunc / np_sgn: `c.value & ((1<<f) - 1)`         :870, :3657
//   k_nonzero        a != 0 (bytes) + count    np_random_bits: `mask = _r2.value != 0`             :4254
//   k_bits_compose   sum_j bits[i, j] 2^e(j)   np_trunc / np_sgn / np_to_bits:
//                                              `np.sum(r_bits.reshape((n, f)) << shifts, axis=1)`  :860, :3651, :4415
//   k_bits_decompose (c[i] >> e(j)) & 1        np_sgn / np_to_bits: `np.right_shift.outer(c, shifts).T & 1`  :3660, :4423
//   k_conv2d         'same' 2-D correlation over input channels + bias, mod p
//                                              demos/np_cnnmnist.py:69-81 (convolvetensor's np.correlate loops)
//   k_transpose, k_binop_rows                  np_sgn's (l, n) bit-matrix algebra: `r_bits.T`, `s_sign - <matrix>` (row
//                                              broadcast); its `np.cumsum(.., axis=0)` is K7's scan  :3661-3672
//
// The reference computes these over the integers and reduces when the result enters a field array
// (`Zp.array(...)`, finfields.py:717-725); reduction is a ring homomorphism, so computing mod p throughout gives the
// same field array bit for bit.  The two operations that are NOT ring operations -- `&` and `>>` on an opened value
// -- are applied to canonical residues, exactly as the reference applies them to the canonical output of
// `self.output`.  All HBM-bound streamers except k_conv2d (integer issue).
#pragma once

struct AffineParams {
    u64 s[4];
    u64 t[4];
};

// one element (L limbs) with the widest access its size allows: 16 bytes for even L (base 16-byte aligned), else 8
template <int L>
__device__ __forceinline__ void ldg_elem(u32* v, const u64* p) {
    if constexpr (L % 2 == 0) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) ldg_v4(v + 4 * q, p + 2 * q);
    } else {
#pragma unroll
        for (int q = 0; q < L; q++) ldg_v2(v + 2 * q, p + q);
    }
}
template <int L>
__device__ __forceinline__ void stg_elem(u64* p, const u32* v) {
    if constexpr (L % 2 == 0) {
#pragma unroll
        for (int q = 0; q < L / 2; q++) stg_v4(p + 2 * q, v + 4 * q);
    } else {
#pragma unroll
        for (int q = 0; q < L; q++) stg_v2(p + q, v + 2 * q);
    }
}

// ---------------------------------------------------------------------------------------
// elementwise: fma / axpb / low_bits / nonzero
// ---------------------------------------------------------------------------------------

template <int L, int KIND, bool SQUARE, int E, bool VEC>
__device__ __forceinline__ void fma_item(const FieldParams& f, const u64* a, const u64* b, const u64* c, u64* out, size_t item) {
    constexpr int N = 2 * L;
    const size_t off = item * (size_t)(E * L);
    u32 x[E * N], y[E * N], z[E * N], r[E * N];
    load_limbs<E * L, VEC>(x, a + off);
    if constexpr (!SQUARE) load_limbs<E * L, VEC>(y, b + off);
    load_limbs<E * L, VEC>(z, c + off);
#pragma unroll
    for (int e = 0; e < E; e++) {
        u32 pr[N];
        Fp<L, KIND>::mul(pr, x + e * N, SQUARE ? x + e * N : y + e * N, f);
        Fp<L, KIND>::add(r + e * N, pr, z + e * N, f);
    }
    store_limbs<E * L, VEC>(out + off, r);
}

template <int L, int KIND, bool SQUARE, bool VEC>
__global__ void MPYC_LB
k_fma(FieldParams f, const u64* __restrict__ a, const u64* __restrict__ b, const u64* __restrict__ c, u64* __restrict__ out, size_t n) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    for (size_t it = tid; it < n_items; it += nth) fma_item<L, KIND, SQUARE, E, VEC>(f, a, b, c, out, it);
    if constexpr (E > 1)
        for (size_t h = n_items * E + tid; h < n; h += nth) fma_item<L, KIND, SQUARE, 1, false>(f, a, b, c, out, h);
}

template <int L, int KIND, int E, bool VEC>
__device__ __forceinline__ void axpb_item(const FieldParams& f, const u64* a, const u32* s, const u32* t, bool unit, u64* out, size_t item) {
    constexpr int N = 2 * L;
    const size_t off = item * (size_t)(E * L);
    u32 x[E * N], r[E * N];
    load_limbs<E * L, VEC>(x, a + off);
#pragma unroll
    for (int e = 0; e < E; e++) {
        u32 pr[N];
        if (unit) copy_n<N>(pr, x + e * N);             // s == 1: a shift of the affine map only (warp-uniform)
        else Fp<L, KIND>::mul(pr, x + e * N, s, f);
        Fp<L, KIND>::add(r + e * N, pr, t, f);
    }
    store_limbs<E * L, VEC>(out + off, r);
}

template <int L, int KIND, bool VEC>
__global__ void MPYC_LB
k_axpb(FieldParams f, AffineParams ap, int unit, const u64* __restrict__ a, u64* __restrict__ out, size_t n) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    u32 s[N], t[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        s[i] = as32(ap.s)[i];
        t[i] = as32(ap.t)[i];
    }
    for (size_t it = tid; it < n_items; it += nth) axpb_item<L, KIND, E, VEC>(f, a, s, t, unit != 0, out, it);
    if constexpr (E > 1)
        for (size_t h = n_items * E + tid; h < n; h += nth) axpb_item<L, KIND, 1, false>(f, a, s, t, unit != 0, out, h);
}

// out = a & mask (mask = 2^b - 1 as limbs); a canonical, so is the result
template <int L, bool VEC>
__global__ void MPYC_LB
k_low_bits(ScalarParam mask, const u64* __restrict__ a, u64* __restrict__ out, size_t n) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    for (size_t it = tid; it < n_items; it += nth) {
        u32 x[E * N];
        load_limbs<E * L, VEC>(x, a + it * (size_t)(E * L));
#pragma unroll
        for (int i = 0; i < E * N; i++) x[i] &= as32(mask.v)[i % N];
        store_limbs<E * L, VEC>(out + it * (size_t)(E * L), x);
    }
    if constexpr (E > 1)
        for (size_t h = n_items * E + tid; h < n; h += nth) {
            u32 x[N];
            load_limbs<L, false>(x, a + h * L);
#pragma unroll
            for (int i = 0; i < N; i++) x[i] &= as32(mask.v)[i];
            store_limbs<L, false>(out + h * L, x);
        }
}

// out8[h] = a[h] != 0 (may be null); *count += number of non-zero elements
template <int L, bool VEC>
__global__ void MPYC_LB
k_nonzero(const u64* __restrict__ a, unsigned char* __restrict__ out8, unsigned long long* count, size_t n) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_items = n / E;
    unsigned int mine = 0;
    for (size_t it = tid; it < n_items; it += nth) {
        u32 x[E * N];
        load_limbs<E * L, VEC>(x, a + it * (size_t)(E * L));
#pragma unroll
        for (int e = 0; e < E; e++) {
            const bool nz = !is_zero_n<N>(x + e * N);
            if (out8) out8[it * E + e] = nz;
            mine += nz;
        }
    }
    if constexpr (E > 1)
        for (size_t h = n_items * E + tid; h < n; h += nth) {
            u32 x[N];
            load_limbs<L, false>(x, a + h * L);
            const bool nz = !is_zero_n<N>(x);
            if (out8) out8[h] = nz;
            mine += nz;
        }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(count, (unsigned long long)mine);
}

// ---------------------------------------------------------------------------------------
// k_bits_decompose: out[j*ostride + i] = bit e(j) of c[i] as a field element, j < l;
// e(j) = j (ascending) or l-1-j (descending: np_sgn's shifts = arange(l-1, -1, -1)).  Reads E, writes l*E per element:
// a write stream, one coalesced row segment per (warp, j).
// ---------------------------------------------------------------------------------------

template <int L, bool VEC>
__global__ void MPYC_LB
k_bits_decompose(const u64* __restrict__ c, u64* __restrict__ out, size_t ostride, size_t n, int l, int descending) {
    constexpr int E = VEC ? VecItem<L>::E : 1;
    constexpr int N = 2 * L;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    const size_t n_items = (n + E - 1) / E;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += nth) {
        const size_t h0 = it * E;
        u32 x[E][N];
        if (VEC && h0 + E <= n) {
            u32 flat[E * N];
            load_limbs<E * L, VEC>(flat, c + h0 * L);
#pragma unroll
            for (int e = 0; e < E; e++) copy_n<N>(x[e], flat + e * N);
        } else {
#pragma unroll
            for (int e = 0; e < E; e++) {
                if (h0 + e < n) load_limbs<L, false>(x[e], c + (h0 + e) * L);
                else zero_n<N>(x[e]);
            }
        }
        for (int b = 0; b < l; b++) {                    // bit b of every element, then shift the elements down by one
            const size_t row = descending ? (size_t)(l - 1 - b) : (size_t)b;
            u32 o[E * N];
#pragma unroll
            for (int i = 0; i < E * N; i++) o[i] = 0;
#pragma unroll
            for (int e = 0; e < E; e++) {
                o[e * N] = x[e][0] & 1u;
#pragma unroll
                for (int i = 0; i < N - 1; i++) x[e][i] = __funnelshift_r(x[e][i], x[e][i + 1], 1);
                x[e][N - 1] >>= 1;
            }
            u64* dst = out + (row * ostride + h0) * L;
            if (VEC && h0 + E <= n) {
                store_limbs<E * L, VEC>(dst, o);
            } else {
#pragma unroll
                for (int e = 0; e < E; e++)
                    if (h0 + e < n) store_limbs<L, false>(dst + e * L, o + e * N);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// k_bits_compose: out[i] = sum_j bits[i*f + j] * 2^e(j) mod p;  e(j) = j or f-1-j.  `bits` are arbitrary residues
// (shares of bits).  Horner over groups of 32 bit positions from the top exponent; inside a group every 32-bit limb of an
// element is multiplied by its power of two and accumulated with one IMAD.WIDE (no carries), one reduction per group.
//
// Memory: row i of the (n, f) input is f*E contiguous bytes -- a thread walking its own row would touch one sector
// per warp lane and instruction.  So a CTA stages a tile of 256 rows x JB columns (~128 bytes of each row) in shared
// memory with 16-byte cp.async pieces issued in row-major piece order (8 consecutive threads fetch the 128 contiguous
// bytes of one row), three stages in flight across tile boundaries.  The row pitch in shared memory is sized from
// min(f, JB) at run time (narrow inputs such as np_trunc's f = 6 leave room for 4-5 CTAs per SM instead of 2) and is an
// odd number of 16-byte units so that the per-thread reads (thread = row) spread over the banks.  For odd L a row chunk
// may start on an odd 8-byte boundary: it gets an 8-byte head piece and is stored 8 bytes into its pitch, so that the
// rest still moves in aligned 16-byte pieces.
// ---------------------------------------------------------------------------------------

template <int L>
struct ComposeCfg {
    static constexpr int EB = 8 * L;                      // bytes per element
    static constexpr bool WIDE = (L % 2 == 0);            // even L: every element is 16-byte aligned
    static constexpr int JB = L == 1 ? 14 : (L == 2 ? 8 : 4);   // columns per stage (even): a row chunk is at most 8 copy slots
    static constexpr int G = 8;                           // copy slots per row (8 consecutive threads serve one row)
    static constexpr int STAGES = 3;
    // row pitch in shared memory for stages of at most `cols` columns: a multiple of 16 bytes with room for the row
    // chunk plus the 8-byte shift of rows that start on an odd 8-byte boundary (odd L), and an odd number of 16-byte
    // units so that the per-thread reads (thread = row) spread over the banks
    static __host__ __device__ int pitch(int cols) {
        const int units = (cols * EB + (WIDE ? 0 : 8) + 15) / 16;
        return ((units + 1) | 1) * 16;
    }
    // cp.async slots a full row chunk needs: 16-byte pieces, plus for odd L an 8-byte head (misaligned rows) and tail
    static_assert((WIDE ? JB * EB / 16 : (JB * EB + 8) / 16 + 1) <= G, "a row chunk must fit the copy slots of its 8 threads");
    static __host__ __device__ int smem(int fcols) { return STAGES * MPYC_THREADS * pitch(fcols < JB ? fcols : JB); }
};

template <int L>
__device__ __forceinline__ void lds_elem(u32* v, u32 saddr) {
    if constexpr (L % 2 == 0) {
#pragma unroll
        for (int q = 0; q < L / 2; q++)
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(v[4 * q]), "=r"(v[4 * q + 1]), "=r"(v[4 * q + 2]), "=r"(v[4 * q + 3]) : "r"(saddr + 16 * q));
    } else {
#pragma unroll
        for (int q = 0; q < L; q++)
            asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v[2 * q]), "=r"(v[2 * q + 1]) : "r"(saddr + 8 * q));
    }
}

__device__ __forceinline__ void cp_async16(u32 dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(u32 dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}

template <int L, int KIND>
__global__ void MPYC_LB
k_bits_compose(FieldParams f, const u64* __restrict__ bits, u64* __restrict__ out, size_t n, int fcols, int descending) {
    typedef Fp<L, KIND> F;
    typedef ComposeCfg<L> C;
    constexpr int N = 2 * L;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const u32 smem0 = smem_u32(smem_raw);
    const int t = threadIdx.x;
    const int nblk = (fcols + C::JB - 1) / C::JB;
    const int pitch = C::pitch(min(fcols, C::JB));
    const u32 stage_bytes = (u32)MPYC_THREADS * pitch;
    const size_t tiles = (n + MPYC_THREADS - 1) / MPYC_THREADS;
    const size_t my_tiles = tiles > blockIdx.x ? (tiles - blockIdx.x - 1) / gridDim.x + 1 : 0;
    const size_t units = my_tiles * (size_t)nblk;
    const unsigned char* gbase = reinterpret_cast<const unsigned char*>(bits);

    // column block b (in Horner order, top exponent first) of a row: first column and number of columns
    auto block_cols = [&](int b, int& col0, int& ncols) {
        if (descending) {                               // e(j) = f-1-j: columns 0, 1, ...
            col0 = b * C::JB;
            ncols = min(C::JB, fcols - col0);
        } else {                                        // e(j) = j: columns f-1, f-2, ...
            const int hi = fcols - b * C::JB;           // one past the top column of this block
            col0 = max(hi - C::JB, 0);
            ncols = hi - col0;
        }
    };
    // a row whose chunk starts on an odd 8-byte boundary is stored 8 bytes into its pitch, so that 16-byte aligned
    // global addresses land on 16-byte aligned shared addresses (odd L only)
    // odd L with an even number of columns on a 16-byte aligned base: every chunk starts and ends on a 16-byte boundary
    // (JB is even), so the plain 16-byte path applies (warp-uniform)
    const bool aligned = C::WIDE || ((fcols & 1) == 0 && (reinterpret_cast<uintptr_t>(gbase) & 15u) == 0);
    auto row_shift = [&](size_t row, int col0) -> u32 {
        if (aligned) return 0u;
        return (u32)((reinterpret_cast<uintptr_t>(gbase) + (row * (size_t)fcols + col0) * C::EB) & 8u);
    };
    // copy slot k of row (t >> 3) + 32 r: 8 consecutive threads fetch the contiguous chunk of one row, a warp 4 rows
    const int kslot = t & (C::G - 1), rsub = t >> 3;
    const size_t row_bytes = (size_t)fcols * C::EB;
    // (tile, column block) of the next unit to fetch and of the next unit to consume, advanced without divisions
    size_t itile = blockIdx.x, ctile = blockIdx.x;
    int ib = 0, cb = 0;
    u32 istage = 0, cstage = 0;                          // shared-memory stage of the next fetch / of the next consume
    auto issue = [&](size_t u) {
        if (u < units) {
            const size_t tile = itile;
            int col0, ncols;
            block_cols(ib, col0, ncols);
            if (++ib == nblk) {
                ib = 0;
                itile += gridDim.x;
            }
            const size_t row0 = tile * MPYC_THREADS;
            const int rows = (int)min((size_t)MPYC_THREADS, n - row0);
            const int rb = ncols * C::EB;               // bytes of one row chunk
            const unsigned char* tbase = gbase + (row0 * (size_t)fcols + col0) * C::EB;
            const u32 stage = smem0 + istage * stage_bytes;
#pragma unroll
            for (int r = 0; r < MPYC_THREADS / (MPYC_THREADS / C::G); r++) {
                const int row = rsub + (MPYC_THREADS / C::G) * r;
                if (row < rows) {
                    const unsigned char* src = tbase + row * row_bytes;
                    if (aligned) {
                        if (16 * kslot < rb) cp_async16(stage + row * pitch + 16 * kslot, src + 16 * kslot);
                    } else {
                        const u32 mis = (u32)(reinterpret_cast<uintptr_t>(src) & 8u);   // 0 or 8
                        const int off = mis ? (kslot == 0 ? 0 : 16 * kslot - 8) : 16 * kslot;
                        const int size = (mis && kslot == 0) ? 8 : min(16, rb - off);
                        const u32 dst = stage + row * pitch + mis + off;
                        if (size == 16) cp_async16(dst, src + off);
                        else if (size == 8) cp_async8(dst, src + off);
                    }
                }
            }
        }
        if (++istage == C::STAGES) istage = 0;
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

#pragma unroll
    for (int s = 0; s < C::STAGES - 1; s++) issue(s);
    // Horner over groups of up to 32 columns; inside a group column q (in Horner order) has the weight 2^(cnt-1-q), and
    // every 32-bit limb of the element is accumulated on its own: wacc[i] += x[i] * 2^(cnt-1-q) is ONE IMAD.WIDE.U32 and
    // cannot overflow 64 bits within 32 columns -- no carry chains in the inner loop.  A finished group G < 2^32 p is
    // folded as res = (res << cnt) + G mod p.
    u64 wacc[N];
    u32 res[N];
#pragma unroll
    for (int i = 0; i < N; i++) wacc[i] = 0;
    zero_n<N>(res);
    int idx = 0, cnt = 0;                                // column index within the row (Horner order), size of its group
    u32 w = 0;
    for (size_t u = 0; u < units; u++) {
        asm volatile("cp.async.wait_group %0;" ::"n"(C::STAGES - 2) : "memory");
        __syncthreads();                                 // stage u has landed for every thread; stage u-1 is free
        issue(u + C::STAGES - 1);
        const size_t tile = ctile;
        const int b = cb;
        if (++cb == nblk) {
            cb = 0;
            ctile += gridDim.x;
        }
        const size_t row = tile * MPYC_THREADS + t;
        int col0, ncols;
        block_cols(b, col0, ncols);
        if (b == 0) idx = 0;
        if (row < n) {
            const u32 base = smem0 + cstage * stage_bytes + t * pitch + row_shift(row, col0);
            for (int cidx = 0; cidx < ncols; cidx++, idx++) {
                const int lc = descending ? cidx : ncols - 1 - cidx;
                u32 x[N];
                lds_elem<L>(x, base + lc * C::EB);
                if ((idx & 31) == 0) {                   // a new group starts (warp-uniform)
                    cnt = min(32, fcols - idx);
                    w = 1u << (cnt - 1);
                }
#pragma unroll
                for (int i = 0; i < N; i++) wacc[i] += (u64)x[i] * w;
                w >>= 1;
                if (w == 0) {                            // group complete: fold it into the running result
                    u32 acc[N + 2];
                    u64 c = wacc[0];
                    acc[0] = (u32)c;
                    c >>= 32;
#pragma unroll
                    for (int i = 1; i < N; i++) {
                        c += wacc[i];                    // < 2^64: wacc[i] <= (2^32-1)^2, carry-in <= 2^32
                        acc[i] = (u32)c;
                        c >>= 32;
                    }
                    acc[N] = (u32)c;
                    acc[N + 1] = (u32)(c >> 32);
                    u32 sh[N + 1];                       // res << cnt, cnt in 1..32 (clamping funnel shift: 32 moves whole limbs)
                    sh[0] = __funnelshift_lc(0u, res[0], cnt);
#pragma unroll
                    for (int i = 1; i < N; i++) sh[i] = __funnelshift_lc(res[i - 1], res[i], cnt);
                    sh[N] = __funnelshift_lc(res[N - 1], 0u, cnt);
                    acc_add<N + 1, N + 2>(acc, sh);      // < 2^33 p
                    F::reduce_small(res, acc, f);
#pragma unroll
                    for (int i = 0; i < N; i++) wacc[i] = 0;
                }
            }
            if (b == nblk - 1) {                         // the last group ended with the row's last column
                stg_elem<L>(out + row * L, res);
                zero_n<N>(res);
            }
        }
        if (++cstage == C::STAGES) cstage = 0;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------------------
// k_conv2d: Y[i, j, y, x] = B[j] + sum_{l < r} sum_{dy, dx < s} X[i, l, y+dy-s2, x+dx-s2] * W[j, l, dy, dx]  (mod p),
// s odd, s2 = (s-1)/2, zero outside the image -- what np_cnnmnist's convolvetensor builds from np.correlate(.., 'same')
// row by row (demos/np_cnnmnist.py:69-81).  Work item = (i, j, tile of 256 output pixels); the r*s*s filter taps of
// output channel j sit in shared memory in table form, every thread accumulates its pixel's r*s*s products lazily and
// reduces once.  Integer-issue bound; X is re-read s*s times per input channel through L1/L2.
// ---------------------------------------------------------------------------------------

template <int L, int KIND>
__global__ void MPYC_LB
k_conv2d(FieldParams f, const u64* __restrict__ X, const u64* __restrict__ W, const u64* __restrict__ B, u64* __restrict__ Y,
         int k, int r, int m, int n, int v, int s) {
    typedef Fp<L, KIND> F;
    constexpr int N = 2 * L;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u32* sW = reinterpret_cast<u32*>(smem_raw);          // [r*s*s][N], table form
    const int taps = r * s * s, s2 = (s - 1) / 2;
    const size_t pix = (size_t)m * n;
    const size_t ptiles = (pix + MPYC_THREADS - 1) / MPYC_THREADS;
    const size_t items = (size_t)k * v * ptiles;
    int staged_j = -1;
    for (size_t w = blockIdx.x; w < items; w += gridDim.x) {
        const size_t pt = w % ptiles;
        const int j = (int)((w / ptiles) % v), i = (int)(w / (ptiles * v));
        if (j != staged_j) {
            __syncthreads();
            for (int idx = threadIdx.x; idx < taps; idx += MPYC_THREADS) {
                u32 x[N];
                load_limbs<L, false>(x, W + ((size_t)j * taps + idx) * L);
                F::to_dom(x, x, f);
#pragma unroll
                for (int q = 0; q < N; q++) sW[idx * N + q] = x[q];
            }
            __syncthreads();
            staged_j = j;
        }
        const size_t px = pt * MPYC_THREADS + threadIdx.x;
        if (px >= pix) continue;
        const int y = (int)(px / n), x0 = (int)(px % n);
        u32 acc[F::WACC];
        zero_n<F::WACC>(acc);
        for (int l = 0; l < r; l++) {
            const u64* Xc = X + ((size_t)i * r + l) * pix * L;
            for (int dy = 0; dy < s; dy++) {
                const int yy = y + dy - s2;
                if (yy < 0 || yy >= m) continue;
                for (int dx = 0; dx < s; dx++) {
                    const int xx = x0 + dx - s2;
                    if (xx < 0 || xx >= n) continue;
                    u32 a[N], wt[N];
                    const u64* src = Xc + ((size_t)yy * n + xx) * L;
#pragma unroll
                    for (int q = 0; q < L; q++) {
                        const u64 word = __ldg(src + q);
                        a[2 * q] = (u32)word;
                        a[2 * q + 1] = (u32)(word >> 32);
                    }
                    const u32* ws = sW + ((l * s + dy) * s + dx) * N;
#pragma unroll
                    for (int q = 0; q < N; q++) wt[q] = ws[q];
                    F::mac(acc, a, wt);
                }
            }
        }
        u32 res[N], bias[N];
        F::finish(res, acc, f);
        load_limbs<L, false>(bias, B + (size_t)j * L);
        F::add(res, res, bias, f);
        store_limbs<L, false>(Y + (((size_t)i * v + j) * pix + px) * L, res);
    }
}

// ---------------------------------------------------------------------------------------
// (R, C) matrices of elements: transpose, running sum down the rows, row-vector broadcast -- the (l, n) bit-matrix
// algebra of np_sgn (runtime.py:3659-3672): `r_bits.T`, `np.cumsum(np.vstack((zeros, Xor)), axis=0)`,
// `s_sign - np.vstack((c_bits - r_bits, ones)) + 3*SumXors`.
// ---------------------------------------------------------------------------------------

// out (C, R) = in (R, C)^T: 32 x 32 element tiles through shared memory, both sides coalesced along their rows.
// L <= 3: a lane moves one element (L words) and the tile is element-major.  L = 4: that layout puts the lanes of a warp
// 8 banks apart (0.36 of the copy peak); there a warp moves the 32 elements of a row segment as 128 consecutive 64-bit
// words and the tile is limb-planar, tile[limb][row][col], with the planes offset by 32 / L banks -- fill and drain
// conflict-free (0.58).  Measured at np_sgn's shape (n x 38 matrices: the second column tile is 6/32 full).
template <int L>
__global__ void MPYC_LB
k_transpose(const u64* __restrict__ in, u64* __restrict__ out, size_t R, size_t C) {
    constexpr bool PLANAR = (L == 4);
    constexpr int PLANE = 32 * 33 + 16 / L;
    __shared__ u64 tile[PLANAR ? L * PLANE : 32 * 33 * L];
    const size_t tc = (C + 31) / 32, tr = (R + 31) / 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8 threads
    for (size_t w = blockIdx.x; w < tc * tr; w += gridDim.x) {
        const size_t r0 = (w / tc) * 32, c0 = (w % tc) * 32;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const size_t r = r0 + ty + 8 * k;                    // input row
            if (r < R) {
                const u64* src = in + (r * C + c0) * L;
#pragma unroll
                for (int q = 0; q < L; q++) {
                    if constexpr (PLANAR) {
                        const int idx = tx + 32 * q, e = idx / L, lb = idx % L;
                        if (c0 + e < C) tile[lb * PLANE + (ty + 8 * k) * 33 + e] = src[idx];
                    } else {
                        if (c0 + tx < C) tile[(ty + 8 * k) * 33 * L + tx * L + q] = src[tx * L + q];
                    }
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const size_t c = c0 + ty + 8 * k;                    // output row = input column
            if (c < C) {
                u64* dst = out + (c * R + r0) * L;
#pragma unroll
                for (int q = 0; q < L; q++) {
                    if constexpr (PLANAR) {
                        const int idx = tx + 32 * q, e = idx / L, lb = idx % L;
                        if (r0 + e < R) dst[idx] = tile[lb * PLANE + e * 33 + (ty + 8 * k)];
                    } else {
                        if (r0 + tx < R) dst[tx * L + q] = tile[tx * 33 * L + (ty + 8 * k) * L + q];
                    }
                }
            }
        }
    }
}

// out[j][i] = a[j][i] (op) b[i], or b[i] (op) a[j][i] when REFLECT; a: (R, C), b: (C).  A thread owns a column (b[i] is
// loaded once) and walks down the rows, which are coalesced across the warp; ROWS_PER rows are in flight per trip.
template <int L, int KIND, int OP, bool REFLECT>
__global__ void MPYC_LB
k_binop_rows(FieldParams f, const u64* __restrict__ a, const u64* __restrict__ b, u64* __restrict__ out, size_t R, size_t C) {
    constexpr int N = 2 * L;
    constexpr int ROWS_PER = 4;
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < C; i += nth) {
        u32 y[N];
        ldg_elem<L>(y, b + i * L);
        size_t j = 0;
        for (; j + ROWS_PER <= R; j += ROWS_PER) {
            u32 x[ROWS_PER][N];
#pragma unroll
            for (int q = 0; q < ROWS_PER; q++) ldg_elem<L>(x[q], a + ((j + q) * C + i) * L);
#pragma unroll
            for (int q = 0; q < ROWS_PER; q++) {
                u32 r[N];
                if constexpr (REFLECT) apply_op<L, KIND, OP>(r, y, x[q], f);
                else apply_op<L, KIND, OP>(r, x[q], y, f);
                stg_elem<L>(out + ((j + q) * C + i) * L, r);
            }
        }
        for (; j < R; j++) {
            u32 x[N], r[N];
            ldg_elem<L>(x, a + (j * C + i) * L);
            if constexpr (REFLECT) apply_op<L, KIND, OP>(r, y, x, f);
            else apply_op<L, KIND, OP>(r, x, y, f);
            stg_elem<L>(out + (j * C + i) * L, r);
        }
    }
}
