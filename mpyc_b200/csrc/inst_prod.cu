// K13's launcher (prod.cuh): the columns form for I >= 32 and for rows too short to fill one warp step (R * I < 32,
// where the rows form would leave most lanes idle), the rows form otherwise; K7's 16-byte path for even L on 16-byte
// aligned arrays.  R is split into slices when the shape's work items cannot fill two CTAs per SM (prod_plan); the slice
// partials (S, O, I) live in stream-ordered scratch and are combined by a second pass of the same kernels on (1, S, O*I).
#include "launch_impl.cuh"
#include "prod.cuh"

namespace {

bool cols_form(size_t R, size_t I) { return I >= 32 || R * I < 32; }

// As K7's axis_plan, but for two CTAs per SM in both forms: a product thread holds more registers than a sum thread.
// Slices keep >= 64 rows (columns) / >= 1024 elements (rows form).
AxisPlan prod_plan(size_t O, size_t R, size_t I) {
    const bool cols = cols_form(R, I);
    const size_t want = (size_t)mpyc_sm_count() * 2 * MPYC_THREADS;       // threads
    const size_t items = cols ? O * I : O * 32;
    const size_t most = cols ? R / 64 : R * I / 1024;
    size_t S = items < want ? std::min((want + items - 1) / items, most) : 1;
    if (S < 2) return AxisPlan{1, R};
    const size_t rs = (R + S - 1) / S;
    return AxisPlan{(R + rs - 1) / rs, rs};
}

bool vec_ok(int L, const void* in, const void* out) { return L % 2 == 0 && aligned16(in) && aligned16(out); }

template <int L, int KIND, bool VEC>
cudaError_t prod_pass_k(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                        const ScalarParam& init, int mul_init, cudaStream_t st) {
    if (cols_form(R, I)) return launch_kernel(k_prod_cols<L, KIND, VEC>, S * O * I, 0, st, fp, in, out, O, R, I, rs, S, init, mul_init);
    return launch_kernel(k_prod_rows<L, KIND, VEC>, S * O * 32, 0, st, fp, in, out, O, R, I, rs, S, init, mul_init);
}

template <int L, int KIND, bool VEC>
cudaError_t cumprod_pass_k(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                           const u64* carry, int inc, cudaStream_t st) {
    if (cols_form(R, I)) return launch_kernel(k_cumprod_cols<L, KIND, VEC>, S * O * I, 0, st, fp, in, out, O, R, I, rs, S, carry, inc);
    return launch_kernel(k_cumprod_rows<L, KIND, VEC>, S * O * 32, 0, st, fp, in, out, O, R, I, rs, S, carry, inc);
}

template <int L, bool VEC, bool ANY>
cudaError_t allany_pass_k(const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs, cudaStream_t st) {
    if (cols_form(R, I)) return launch_kernel(k_allany_cols<L, VEC, ANY>, S * O * I, 0, st, in, out, O, R, I, rs, S);
    return launch_kernel(k_allany_rows<L, VEC, ANY>, S * O * 32, 0, st, in, out, O, R, I, rs, S);
}

template <int L>
cudaError_t prod_pass(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                      const ScalarParam& init, int mul_init, cudaStream_t st) {
    if constexpr (L % 2 == 0) {
        if (vec_ok(L, in, out)) {
#define M(K) return prod_pass_k<L, K, true>(fp, in, out, O, R, I, S, rs, init, mul_init, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return prod_pass_k<L, K, false>(fp, in, out, O, R, I, S, rs, init, mul_init, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t cumprod_pass(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs,
                         const u64* carry, int inc, cudaStream_t st) {
    if constexpr (L % 2 == 0) {
        if (vec_ok(L, in, out)) {
#define M(K) return cumprod_pass_k<L, K, true>(fp, in, out, O, R, I, S, rs, carry, inc, st)
            KIND_SWITCH(fp.kind, M)
#undef M
        }
    }
#define M(K) return cumprod_pass_k<L, K, false>(fp, in, out, O, R, I, S, rs, carry, inc, st)
    KIND_SWITCH(fp.kind, M)
#undef M
    return cudaErrorInvalidValue;
}

template <int L>
cudaError_t allany_pass(bool any, const u64* in, u64* out, size_t O, size_t R, size_t I, size_t S, size_t rs, cudaStream_t st) {
    if constexpr (L % 2 == 0) {
        if (vec_ok(L, in, out))
            return any ? allany_pass_k<L, true, true>(in, out, O, R, I, S, rs, st) : allany_pass_k<L, true, false>(in, out, O, R, I, S, rs, st);
    }
    return any ? allany_pass_k<L, false, true>(in, out, O, R, I, S, rs, st) : allany_pass_k<L, false, false>(in, out, O, R, I, S, rs, st);
}

template <int L>
cudaError_t prod_l(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, const ScalarParam& init,
                   int mul_init, cudaStream_t st) {
    if (O * I == 0) return cudaSuccess;
    const AxisPlan pl = prod_plan(O, R, I);
    if (pl.S == 1) return prod_pass<L>(fp, in, out, O, R, I, 1, R, init, mul_init, st);
    u64* part = nullptr;                                 // (S, O, I) slice products, stream-ordered scratch
    cudaError_t e = mpyc_scratch_alloc(&part, pl.S * O * I * L * sizeof(u64), st);
    if (e != cudaSuccess) return e;
    e = prod_pass<L>(fp, in, part, O, R, I, pl.S, pl.rs, init, 0, st);
    if (e == cudaSuccess) e = prod_l<L>(fp, part, out, 1, pl.S, O * I, init, mul_init, st);
    cudaFreeAsync(part, st);
    return e;
}

// Split R: the slice products (S, O, I), their running products along S (slice s's carry-in is entry s - 1: the exclusive
// scan), then every slice rescanned from its carry-in.  Three launches in stream order; the input is read twice.
template <int L>
cudaError_t cumprod_l(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, int inc, cudaStream_t st) {
    if (O * I == 0) return cudaSuccess;
    const AxisPlan pl = prod_plan(O, R, I);
    if (pl.S == 1) return cumprod_pass<L>(fp, in, out, O, R, I, 1, R, nullptr, inc, st);
    const size_t count = pl.S * O * I;
    u64* part = nullptr;                                 // slice products, then their running products
    cudaError_t e = mpyc_scratch_alloc(&part, 2 * count * L * sizeof(u64), st);
    if (e != cudaSuccess) return e;
    const ScalarParam none = {};
    e = prod_pass<L>(fp, in, part, O, R, I, pl.S, pl.rs, none, 0, st);
    if (e == cudaSuccess) e = cumprod_l<L>(fp, part, part + count * L, 1, pl.S, O * I, 0, st);
    if (e == cudaSuccess) e = cumprod_pass<L>(fp, in, out, O, R, I, pl.S, pl.rs, part + count * L, inc, st);
    cudaFreeAsync(part, st);
    return e;
}

// Split R: every slice's 0 / 1 (all of the slice / any of it), then the same test along S.
template <int L>
cudaError_t allany_l(bool any, const u64* in, u64* out, size_t O, size_t R, size_t I, cudaStream_t st) {
    if (O * I == 0) return cudaSuccess;
    const AxisPlan pl = prod_plan(O, R, I);
    if (pl.S == 1) return allany_pass<L>(any, in, out, O, R, I, 1, R, st);
    u64* part = nullptr;
    cudaError_t e = mpyc_scratch_alloc(&part, pl.S * O * I * L * sizeof(u64), st);
    if (e != cudaSuccess) return e;
    e = allany_pass<L>(any, in, part, O, R, I, pl.S, pl.rs, st);
    if (e == cudaSuccess) e = allany_l<L>(any, part, out, 1, pl.S, O * I, st);
    cudaFreeAsync(part, st);
    return e;
}

}  // namespace

cudaError_t launch_prod_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, const u64* init,
                             cudaStream_t st) {
    ScalarParam sp = {};
    if (init)
        for (u32 i = 0; i < fp.L; i++) sp.v[i] = init[i];
    const int mul_init = init ? 1 : 0;
    switch (fp.L) {
        case 1: return prod_l<1>(fp, in, out, O, R, I, sp, mul_init, st);
        case 2: return prod_l<2>(fp, in, out, O, R, I, sp, mul_init, st);
        case 3: return prod_l<3>(fp, in, out, O, R, I, sp, mul_init, st);
        case 4: return prod_l<4>(fp, in, out, O, R, I, sp, mul_init, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_cumprod_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool inc,
                                cudaStream_t st) {
    const int c = inc ? 1 : 0;
    switch (fp.L) {
        case 1: return cumprod_l<1>(fp, in, out, O, R, I, c, st);
        case 2: return cumprod_l<2>(fp, in, out, O, R, I, c, st);
        case 3: return cumprod_l<3>(fp, in, out, O, R, I, c, st);
        case 4: return cumprod_l<4>(fp, in, out, O, R, I, c, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_all_any_axis(const FieldParams& fp, const u64* in, u64* out, size_t O, size_t R, size_t I, bool any,
                                cudaStream_t st) {
    switch (fp.L) {
        case 1: return allany_l<1>(any, in, out, O, R, I, st);
        case 2: return allany_l<2>(any, in, out, O, R, I, st);
        case 3: return allany_l<3>(any, in, out, O, R, I, st);
        case 4: return allany_l<4>(any, in, out, O, R, I, st);
    }
    return cudaErrorInvalidValue;
}
