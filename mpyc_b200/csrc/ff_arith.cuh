// Multi-limb prime-field arithmetic for sm_90a (and, for table preparation and algorithm
// tests, the host).  Elements are L little-endian 64-bit limbs in memory (L in {1,2,3,4}); in
// registers they are handled as N = 2L 32-bit limbs, because the native multiplier is
// IMAD.WIDE.U32 (32x32+64 with carry in/out): every mad.lo.cc.u32 / madc.hi.cc.u32 pair below is
// one such instruction, and products are accumulated in two interleaved carry chains (even and
// odd columns) so that no extra additions are spent on carries.
//
// Two reduction families, chosen per modulus when the field context is created:
//   * pseudo-Mersenne p = 2^k - c with c < 2^16 and k >= 56  (MPyC's default primes from
//     finfields.find_prime_root, reference mpyc/finfields.py:325-331: 2^61-1, 2^64-189,
//     2^69-93, 2^128-173, 2^256-189): fold the high part down with a multiply by c.
//       KIND_PM_ALIGNED  k == 64 L     (fold at a limb boundary)
//       KIND_PM_SHIFT    k % 64 != 0   (fold at bit k with funnel shifts)
//   * KIND_GENERIC: any odd p < 2^(64 L).
//       - lazily accumulated sums of full products against per-call constants: Montgomery reduction
//         with ONE GUARD LIMB, R' = 2^(64 (L+1)), so that up to 2^20 products (< K p^2 < p R') reduce
//         with a single REDC and one conditional subtraction.  Constants ("table form") are
//         pre-multiplied by R' on the host, data stays canonical:
//         REDC(sum_i lambda_i R' * share_i) = sum_i lambda_i share_i mod p.
//       - canonical * canonical and (L+1)-limb sums of 64-bit-constant products: Barrett reduction
//         (quotient estimated from the top limbs with a precomputed reciprocal; at most 3 too small).
//
// Everything at the kernel boundary is a canonical residue in [0, p); Montgomery form never
// leaves a kernel.  The arithmetic replaces the reference's Python-int `(a op b) % p` inside
// NumPy object loops (mpyc/finfields.py:717-725,1056-1124; mpyc/thresha.py:63,129).
#pragma once
#include <stdint.h>

typedef unsigned long long u64;
typedef unsigned int u32;

#if defined(__CUDACC__)
#define FF_HD __host__ __device__ __forceinline__
#else
#define FF_HD inline
#endif

enum { KIND_GENERIC = 0, KIND_PM_ALIGNED = 1, KIND_PM_SHIFT = 2 };

// Upper bound on the number of full-width products that may be accumulated lazily
// (in a 2L+1 limb accumulator) before a reduction is required.
#define FF_MAX_LAZY_TERMS (1u << 20)

struct FieldParams {
    u64 p[4];    // modulus
    u64 r1[4];   // GENERIC: R' mod p      (table form of 1)
    u64 r2[4];   // GENERIC: R'^2 mod p
    u64 pinv;    // GENERIC: -p^-1 mod 2^64
    u64 c;       // PM: 2^k - p
    u32 k;       // bit length of p (PM: the exponent)
    u32 s;       // k % 64
    u32 L;       // 64-bit limbs
    u32 kind;
    // GENERIC, Barrett reductions of canonical data (quotient estimate from the top bits, <= 3 too small):
    u64 p2[5];   //   2p
    u64 mus;     //   floor(2^(k+64) / p) - 2^64            (64-bit quotients: (L+1)-limb values)
    u64 pn[4];   //   p << nsh: the modulus normalised to 64L bits
    u64 pn2[5];  //   2 pn
    u64 muf[4];  //   floor(2^(128L) / pn) - 2^(64L)        (full-width quotients: products)
    u32 nsh;     //   64L - k
    u32 mus32;   //   floor(2^(k+32) / p) - 2^32            (32-bit quotients: values < 2^(k+31), barrett_small32)
    u32 q32;     //   per launch (set by the launcher, 0 in the field handle): every value handed to reduce_small is
    u32 pad_;    //   < 2^(k+31), so the 32-bit-quotient step applies
};

// 32-bit view of a little-endian u64 array (kernel parameters and tables are stored as u64)
FF_HD const u32* as32(const u64* x) { return reinterpret_cast<const u32*>(x); }

// ---------------------------------------------------------------------------------------
// n-limb primitives on 32-bit limbs.  Device: PTX carry chains, one instruction per asm statement,
// fully unrolled so limbs stay in registers.  Host: portable 64-bit arithmetic.
// ---------------------------------------------------------------------------------------

template <int N>
FF_HD u32 add_n(u32* r, const u32* a, const u32* b) {
#ifdef __CUDA_ARCH__
    asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
    for (int i = 1; i < N; i++)
        asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r[i]) : "r"(a[i]), "r"(b[i]));
    u32 cy;
    asm volatile("addc.u32 %0, 0, 0;" : "=r"(cy));
    return cy;
#else
    u64 acc = 0;
    for (int i = 0; i < N; i++) {
        acc += (u64)a[i] + b[i];
        r[i] = (u32)acc;
        acc >>= 32;
    }
    return (u32)acc;
#endif
}

// r = a - b, returns 1 on borrow
template <int N>
FF_HD u32 sub_n(u32* r, const u32* a, const u32* b) {
#ifdef __CUDA_ARCH__
    asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
    for (int i = 1; i < N; i++)
        asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r[i]) : "r"(a[i]), "r"(b[i]));
    u32 bw;
    asm volatile("subc.u32 %0, 0, 0;" : "=r"(bw));
    return bw & 1u;
#else
    u32 bw = 0;
    for (int i = 0; i < N; i++) {
        u64 d = (u64)a[i] - b[i] - bw;
        r[i] = (u32)d;
        bw = (u32)(d >> 32) & 1u;
    }
    return bw;
#endif
}

// acc[0..W) += x[0..NX)   (NX <= W; the carry is propagated to the top of acc)
template <int NX, int W>
FF_HD void acc_add(u32* acc, const u32* x) {
    static_assert(NX <= W, "accumulator too short");
#ifdef __CUDA_ARCH__
    asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(acc[0]) : "r"(x[0]));
#pragma unroll
    for (int i = 1; i < NX; i++) asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(acc[i]) : "r"(x[i]));
#pragma unroll
    for (int i = NX; i < W; i++) asm volatile("addc.cc.u32 %0, %0, 0;" : "+r"(acc[i]));
#else
    u64 cy = 0;
    for (int i = 0; i < W; i++) {
        cy += (u64)acc[i] + (i < NX ? x[i] : 0u);
        acc[i] = (u32)cy;
        cy >>= 32;
    }
#endif
}

// One carry chain: acc[i, i+1] += a[i] * b for i = I0, I0+2, ... < N, then the carry is added into
// the following limbs up to W.  Each (mad.lo.cc, madc.hi.cc) pair is one IMAD.WIDE.U32.
template <int N, int W, int I0>
FF_HD void mad_chain(u32* acc, const u32* a, u32 b) {
    if constexpr (I0 < N) {
#ifdef __CUDA_ARCH__
        asm volatile("mad.lo.cc.u32 %0, %1, %2, %0;" : "+r"(acc[I0]) : "r"(a[I0]), "r"(b));
        asm volatile("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(acc[I0 + 1]) : "r"(a[I0]), "r"(b));
#pragma unroll
        for (int i = I0 + 2; i < N; i += 2) {
            asm volatile("madc.lo.cc.u32 %0, %1, %2, %0;" : "+r"(acc[i]) : "r"(a[i]), "r"(b));
            asm volatile("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(acc[i + 1]) : "r"(a[i]), "r"(b));
        }
        constexpr int LAST = I0 + 2 * ((N - 1 - I0) / 2);   // last index multiplied
#pragma unroll
        for (int c = LAST + 2; c < W; c++) asm volatile("addc.cc.u32 %0, %0, 0;" : "+r"(acc[c]));
#else
        u64 cy = 0;
        int c = I0;
        for (int i = I0; i < N; i += 2) {
            u64 prod = (u64)a[i] * b;
            cy += (u64)acc[i] + (u32)prod;
            acc[i] = (u32)cy;
            cy >>= 32;
            cy += (u64)acc[i + 1] + (prod >> 32);
            acc[i + 1] = (u32)cy;
            cy >>= 32;
            c = i + 2;
        }
        for (; c < W; c++) {
            cy += acc[c];
            acc[c] = (u32)cy;
            cy >>= 32;
        }
#endif
    }
}

// acc[0..W) += a[0..N) * b  (b one 32-bit limb).  W >= N+1; a carry out of acc[W-1] must be
// impossible by construction (every caller's magnitude bound guarantees it).
template <int N, int W>
FF_HD void mac_small(u32* acc, const u32* a, u32 b) {
    static_assert(W >= N + 1, "accumulator too short");
    mad_chain<N, W, 0>(acc, a, b);
    mad_chain<N, W, 1>(acc, a, b);
}

// r[0..NA+NB) = a[0..NA) * b[0..NB): products accumulated in two interleaved accumulators (E: pairs
// starting at even columns, O: at odd columns), merged by one addition at the end.
template <int NA, int NB, int J>
FF_HD void mul_rows(u32* E, u32* O, const u32* a, const u32* b) {
    if constexpr (J < NB) {
        // row J: a[i]*b[J] lands in columns (i+J, i+J+1); the parity of i+J picks the accumulator.
        // The limb above each chain holds at most earlier carry bits, so one more limb suffices.
        constexpr int WE = ((NA - 1) / 2) * 2 + 3;            // even i: last i = 2*((NA-1)/2), + pair + carry
        constexpr int WO = ((NA - 2) / 2) * 2 + 1 + 3;        // odd  i: last i = 1 + 2*((NA-2)/2)
        if constexpr (J % 2 == 0) {
            mad_chain<NA, WE, 0>(E + J, a, b[J]);
            if constexpr (NA > 1) mad_chain<NA, WO, 1>(O + J, a, b[J]);
        } else {
            mad_chain<NA, WE, 0>(O + J, a, b[J]);
            if constexpr (NA > 1) mad_chain<NA, WO, 1>(E + J, a, b[J]);
        }
        mul_rows<NA, NB, J + 1>(E, O, a, b);
    }
}

template <int NA, int NB>
FF_HD void mul_fresh(u32* r, const u32* a, const u32* b) {
    u32 E[NA + NB + 2], O[NA + NB + 2];
#pragma unroll
    for (int i = 0; i < NA + NB + 2; i++) E[i] = O[i] = 0;
    mul_rows<NA, NB, 0>(E, O, a, b);
    add_n<NA + NB>(r, E, O);
}

// r[0..W) = a[0..NA) * b[0..NB) mod 2^(32 W): the partial products that land entirely at or above
// column W are skipped, the one straddling it contributes its low half only.
template <int NA, int NB, int W, int J>
FF_HD void mul_lo_rows(u32* E, u32* O, const u32* a, const u32* b) {
    if constexpr (J < NB && J < W) {
        constexpr int FIT = W - 1 - J;                 // a[i], i < FIT: both halves of a[i]*b[J] lie below column W
        constexpr int CNT = NA < FIT ? NA : FIT;
        u32* X0 = (J % 2 == 0) ? E : O;                // accumulator of the even-i pairs of this row
        u32* X1 = (J % 2 == 0) ? O : E;
        if constexpr (CNT >= 1) mad_chain<CNT, ((CNT - 1) / 2) * 2 + 3, 0>(X0 + J, a, b[J]);
        if constexpr (CNT >= 2) mad_chain<CNT, ((CNT - 2) / 2) * 2 + 1 + 3, 1>(X1 + J, a, b[J]);
        if constexpr (CNT < NA) X0[W - 1] += a[CNT] * b[J];   // low half into the top column, carry irrelevant
        mul_lo_rows<NA, NB, W, J + 1>(E, O, a, b);
    }
}

template <int NA, int NB, int W>
FF_HD void mul_lo(u32* r, const u32* a, const u32* b) {
    static_assert(W <= NA + NB, "nothing to truncate");
    u32 E[W + 3], O[W + 3];
#pragma unroll
    for (int i = 0; i < W + 3; i++) E[i] = O[i] = 0;
    mul_lo_rows<NA, NB, W, 0>(E, O, a, b);
    add_n<W>(r, E, O);
}

template <int N>
FF_HD void zero_n(u32* r) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = 0;
}

template <int N>
FF_HD void copy_n(u32* r, const u32* a) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = a[i];
}

template <int N>
FF_HD bool is_zero_n(const u32* a) {
    u32 t = 0;
#pragma unroll
    for (int i = 0; i < N; i++) t |= a[i];
    return t == 0;
}

// r = take ? t : r
template <int N>
FF_HD void select_n(u32* r, const u32* t, bool take) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = take ? t[i] : r[i];
}

FF_HD u64 get64(const u32* x, int i) { return (u64)x[2 * i] | ((u64)x[2 * i + 1] << 32); }
FF_HD void set64(u32* x, int i, u64 v) {
    x[2 * i] = (u32)v;
    x[2 * i + 1] = (u32)(v >> 32);
}

// ---------------------------------------------------------------------------------------
// Field<L, KIND>: all element arguments are N = 2L 32-bit limbs
// ---------------------------------------------------------------------------------------

template <int L, int KIND>
struct Fp {
    static constexpr int N = 2 * L;          // 32-bit limbs per element
    static constexpr int WACC = 2 * N + 2;   // lazy accumulator of full products   (2L+1 64-bit limbs)
    static constexpr int WSM = N + 2;        // lazy accumulator of element * 64-bit constants (L+1)

    // a in [0, 2p) (N limbs plus an explicit carry `hi`)  ->  [0, p)
    static FF_HD void csub(u32* a, u32 hi, const FieldParams& f) {
        u32 t[N];
        u32 bw = sub_n<N>(t, a, as32(f.p));
        select_n<N>(a, t, (hi != 0) | (bw == 0));
    }

    static FF_HD void add(u32* r, const u32* a, const u32* b, const FieldParams& f) {
        u32 cy = add_n<N>(r, a, b);
        csub(r, cy, f);
    }

    static FF_HD void sub(u32* r, const u32* a, const u32* b, const FieldParams& f) {
        u32 t[N];
        u32 bw = sub_n<N>(r, a, b);
        add_n<N>(t, r, as32(f.p));
        select_n<N>(r, t, bw != 0);
    }

    static FF_HD void neg(u32* r, const u32* a, const FieldParams& f) {
        u32 t[N];
        bool z = is_zero_n<N>(a);
        sub_n<N>(t, as32(f.p), a);
        zero_n<N>(r);
        select_n<N>(r, t, !z);
    }

    // ---- pseudo-Mersenne: true reduction of a W-limb value (W 32-bit limbs) ------------------
    // Precondition (met by every caller in this library): x < 2^(2k+20), k = bit length of p
    // (covers products < p^2, lazy sums of < 2^20 products, and 64-bit-constant sums < 2^64 p).
    template <int W>
    static FF_HD void pm_reduce(u32* r, const u32* x, const FieldParams& f) {
        static_assert(W == N + 2 || W == 2 * N || W == 2 * N + 2, "unsupported width");
        const u32 c = (u32)f.c;
        // number of 32-bit limbs of the part above the fold point that can be non-zero
        constexpr int HM = (W == N + 2) ? 2 : (W == 2 * N ? N : N + 1);
        u32 r1[N + 2];
        if constexpr (KIND == KIND_PM_ALIGNED && W == N + 2 && L >= 2) {
            // (L+1)-limb sum of 64-bit-constant products: the limb above the fold point times c is
            // < 2^80 and fits the element width, so one pass suffices: r = lo + top*c (+ c on carry).
            const u64 t0 = (u64)x[N] * c, t1 = (u64)x[N + 1] * c;
            const u64 a = t0 + (t1 << 32);
            u32 uu[N];
            zero_n<N>(uu);
            uu[0] = (u32)a;
            uu[1] = (u32)(a >> 32);
            uu[2] = (u32)(t1 >> 32) + (a < t0 ? 1u : 0u);
            u32 cy = add_n<N>(r, x, uu);
            if (cy) {                                    // 2^(64L) = c (mod p); cannot carry again.  Rare.
                zero_n<N>(uu);
                uu[0] = c;
                add_n<N>(r, r, uu);
            }
            csub(r, 0, f);
        } else if constexpr (KIND == KIND_PM_ALIGNED) {
            copy_n<N>(r1, x);
            r1[N] = r1[N + 1] = 0;
            mac_small<HM, N + 2>(r1, x + N, c);
            const u64 u = get64(r1, L) * c;              // < 2^64 by the precondition
            u32 uu[N];
            zero_n<N>(uu);
            uu[0] = (u32)u;
            uu[1] = (u32)(u >> 32);
            u32 cy = add_n<N>(r, r1, uu);
            if (cy) {                                    // 2^(64L) = c (mod p); cannot carry again.  Rare.
                zero_n<N>(uu);
                uu[0] = c;
                add_n<N>(r, r, uu);
            }
            csub(r, 0, f);
        } else {
            const u32 s = f.s;                           // 1..63, p = 2^(64(L-1)+s) - c
            const u64 mask = (1ull << s) - 1;
            u32 hi[N + 2];
#pragma unroll
            for (int i = 0; i <= L; i++) {
                u64 lo_part = (2 * (L - 1 + i) < W) ? (get64(x, L - 1 + i) >> s) : 0;
                u64 hi_part = (2 * (L + i) < W) ? (get64(x, L + i) << (64 - s)) : 0;
                set64(hi, i, lo_part | hi_part);
            }
            copy_n<N>(r1, x);
            set64(r1, L - 1, get64(r1, L - 1) & mask);
            r1[N] = r1[N + 1] = 0;
            mac_small<HM, N + 2>(r1, hi, c);
            const u64 top = (get64(r1, L - 1) >> s) | (get64(r1, L) << (64 - s));
            set64(r1, L - 1, get64(r1, L - 1) & mask);
            const u64 u = top * c;
            u32 uu[N];
            zero_n<N>(uu);
            uu[0] = (u32)u;
            uu[1] = (u32)(u >> 32);
            add_n<N>(r, r1, uu);
            csub(r, 0, f);
        }
    }

    // ---- generic: Montgomery REDC with guard limb: returns x / R' mod p, canonical -----------
    // Precondition: x < p * R'  (R' = 2^(64(L+1))).  One round per 64-bit limb.
    template <int I>
    static FF_HD void redc_rounds(u32* T, const FieldParams& f) {
        if constexpr (I <= L) {
            const u64 m = get64(T, I) * f.pinv;
            u32 m32[2] = {(u32)m, (u32)(m >> 32)};
            u32 P[N + 2];
            mul_fresh<N, 2>(P, as32(f.p), m32);
            acc_add<N + 2, 2 * N + 4 - 2 * I>(T + 2 * I, P);
            redc_rounds<I + 1>(T, f);
        }
    }

    template <int W>
    static FF_HD void redc(u32* r, const u32* x, const FieldParams& f) {
        static_assert(W >= 1 && W <= 2 * N + 2, "unsupported width");
        u32 T[2 * N + 4];
#pragma unroll
        for (int i = 0; i < 2 * N + 4; i++) T[i] = i < W ? x[i] : 0;
        redc_rounds<0>(T, f);
        copy_n<N>(r, T + N + 2);          // result = T[N+2 .. 2N+4) < 2p
        csub(r, T[2 * N + 2], f);
    }

    // acc (WACC limbs) += a * tab        (tab: N limbs, table form)
    static FF_HD void mac(u32* acc, const u32* a, const u32* tab) {
        u32 P[2 * N];
        mul_fresh<N, N>(P, a, tab);
        acc_add<2 * N, WACC>(acc, P);
    }

    // acc (WSM limbs) += a * v   for a plain 64-bit constant v (pseudo-Mersenne fields)
    static FF_HD void mac_const(u32* acc, const u32* a, u64 v) {
        mac_small<N, WSM>(acc, a, (u32)v);
        const u32 vh = (u32)(v >> 32);
        if (vh) mac_small<N, WSM - 1>(acc + 1, a, vh);   // table entries are warp-uniform
    }

    // r = lazily accumulated sum, reduced.  GENERIC: the table-form factor R' is divided out.
    static FF_HD void finish(u32* r, const u32* acc, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) redc<WACC>(r, acc, f);
        else pm_reduce<WACC>(r, acc, f);
    }

    // "domain" multiplication: PM: plain modular product.  GENERIC: Montgomery product ab/R'.
    static FF_HD void dmul(u32* r, const u32* a, const u32* b, const FieldParams& f) {
        u32 x[2 * N];
        mul_fresh<N, N>(x, a, b);
        if constexpr (KIND == KIND_GENERIC) redc<2 * N>(r, x, f);
        else pm_reduce<2 * N>(r, x, f);
    }

    static FF_HD void to_dom(u32* r, const u32* a, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) dmul(r, a, as32(f.r2), f);
        else copy_n<N>(r, a);
    }

    static FF_HD void from_dom(u32* r, const u32* a, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) redc<N>(r, a, f);
        else copy_n<N>(r, a);
    }

    static FF_HD void dom_one(u32* r, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) copy_n<N>(r, as32(f.r1));
        else {
            zero_n<N>(r);
            r[0] = 1;
        }
    }

    // ---- generic: Barrett reductions of canonical data (no domain change) ---------------------
    // d (N+1 limbs) in [0, 4m) -> [0, m) in r (N limbs); m2 = 2m (N+1 limbs)
    static FF_HD void barrett_fix(u32* r, u32* d, const u32* m, const u32* m2) {
        u32 t[N + 1];
        u32 bw = sub_n<N + 1>(t, d, m2);
        select_n<N + 1>(d, t, bw == 0);                 // now d < 2m
        bw = sub_n<N>(t, d, m);
        copy_n<N>(r, d);
        select_n<N>(r, t, (d[N] != 0) | (bw == 0));
    }

    // x < 2^(k+64) in WSM limbs -> x mod p.  Quotient estimate q^ = x1 + floor(x1 * mus / 2^64) with
    // x1 = floor(x / 2^k) < 2^64 and 2^64 + mus = floor(2^(k+64) / p):  q - 3 <= q^ <= q < 2^65.
    static FF_HD void barrett_small(u32* r, const u32* x, const FieldParams& f) {
        const u64 lo = get64(x, L - 1), hi = get64(x, L);
        const u64 x1 = f.s ? ((lo >> f.s) | (hi << (64 - f.s))) : hi;
        const u32 x32[2] = {(u32)x1, (u32)(x1 >> 32)};
        u32 P[4], q[3];
        mul_fresh<2, 2>(P, x32, as32(&f.mus));
        q[2] = add_n<2>(q, x32, P + 2);
        u32 T[N + 1], d[N + 1];
        mul_lo<N, 3, N + 1>(T, as32(f.p), q);
        sub_n<N + 1>(d, x, T);                          // x - q^ p in [0, 4p), exact mod 2^(32(N+1))
        barrett_fix(r, d, as32(f.p), as32(f.p2));
    }

    // x < 2^(k+31) in WSM limbs -> x mod p, with a ONE-limb quotient: x1 = floor(x / 2^k) < 2^31,
    // q^ = x1 + floor(x1 * mus32 / 2^32) with 2^32 + mus32 = floor(2^(k+32) / p):  q - 3 <= q^ <= q < 2^32
    // (x/p - q^ = frac(x1 M / 2^32) + x1 eps / 2^32 + x0 / p < 1 + 1 + 2).  One IMAD.HI for the estimate and N
    // IMAD.WIDE for q^ p, against 4 + 3N for barrett_small: share generation multiplies by (i+1)^j only, so its
    // sums are < (1 + m + ... + m^t) p and the quotient is tiny (launch_impl.cuh: split_q32).
    static FF_HD void barrett_small32(u32* r, const u32* x, const FieldParams& f) {
        const u64 lo = get64(x, L - 1), hi = get64(x, L);
        const u32 x1 = (u32)(f.s ? ((lo >> f.s) | (hi << (64 - f.s))) : hi);
        const u32 q = x1 + (u32)(((u64)x1 * f.mus32) >> 32);        // q^ <= q = floor(x / p) < 2^(k+31) / 2^(k-1) = 2^32
        u32 T[N + 2], d[N + 1];
        zero_n<N + 2>(T);
        mac_small<N, N + 2>(T, as32(f.p), q);
        sub_n<N + 1>(d, x, T);                          // x - q^ p in [0, 4p), exact mod 2^(32(N+1))
        barrett_fix(r, d, as32(f.p), as32(f.p2));
    }

    // canonical a, b -> a b mod p.  The product is taken against b << nsh so that the modulus is the
    // normalised pn = p << nsh (top bit of N limbs set): x' = a b 2^nsh < 2^(32N) pn, x1 = its high N
    // limbs, q^ = x1 + floor(x1 * muf / 2^(32N)) with 2^(32N) + muf = floor(2^(64N) / pn);
    // q' - 3 <= q^ <= q' = floor(x' / pn) < p.  r = (x' - q^ pn) mod pn, shifted back.
    static FF_HD void barrett_mul(u32* r, const u32* a, const u32* b, const FieldParams& f) {
        const u32 sh = f.nsh;                           // 0..63, warp-uniform
        u32 bs[N];
#pragma unroll
        for (int i = L - 1; i >= 0; i--) {
            const u64 cur = get64(b, i), below = i ? get64(b, i - 1) : 0;
            set64(bs, i, sh ? ((cur << sh) | (below >> (64 - sh))) : cur);
        }
        u32 X[2 * N], H[2 * N], q[N];
        mul_fresh<N, N>(X, a, bs);
        mul_fresh<N, N>(H, X + N, as32(f.muf));
        add_n<N>(q, X + N, H + N);
        u32 T[N + 1], d[N + 1];
        mul_lo<N, N, N + 1>(T, as32(f.pn), q);
        sub_n<N + 1>(d, X, T);
        u32 rs[N];
        barrett_fix(rs, d, as32(f.pn), as32(f.pn2));
#pragma unroll
        for (int i = 0; i < L; i++) {
            const u64 cur = get64(rs, i), above = i + 1 < L ? get64(rs, i + 1) : 0;
            set64(r, i, sh ? ((cur >> sh) | (above << (64 - sh))) : cur);
        }
    }

    // canonical * canonical -> canonical
    static FF_HD void mul(u32* r, const u32* a, const u32* b, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) barrett_mul(r, a, b, f);
        else dmul(r, a, b, f);
    }

    // true reduction of an (L+1)-limb value x < 2^(k+64)  (WSM 32-bit limbs)
    static FF_HD void reduce_small(u32* r, const u32* x, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) barrett_small(r, x, f);
        else pm_reduce<WSM>(r, x, f);
    }

    // the same when the launcher has established x < 2^(k+31) for every value of this launch (f.q32, warp-uniform)
    static FF_HD void reduce_small_q32(u32* r, const u32* x, const FieldParams& f) {
        if constexpr (KIND == KIND_GENERIC) {
            if (f.q32) barrett_small32(r, x, f);
            else barrett_small(r, x, f);
        } else if constexpr (KIND == KIND_PM_ALIGNED && L == 1) {
            if (f.q32) {
                // p = 2^64 - c, x = lo + hi 2^64 with hi < 2^31: x = lo + hi c (mod p), hi c < 2^47 -- one IMAD.WIDE,
                // one 64-bit add, a rare second fold of the carry, one conditional subtraction (the general fold
                // multiplies the two-limb top part by c and folds twice)
                const u64 lo = get64(x, 0);
                const u64 t = (u64)x[2] * (u32)f.c;
                u64 v = lo + t;
                if (v < t) v += f.c;                     // carry: 2^64 = c (mod p); cannot carry again (v < 2^48 + c)
                set64(r, 0, v);
                csub(r, 0, f);
            } else {
                pm_reduce<WSM>(r, x, f);
            }
        } else {
            pm_reduce<WSM>(r, x, f);
        }
    }

    // r = a^e in the domain; e = little-endian 64-bit limbs, ebits = bit length of e (>= 0).
    // Branch-free in the exponent (per-thread exponents).
    static FF_HD void dpow(u32* r, const u32* a, const u64* e, int ebits, const FieldParams& f) {
        u32 acc[N];
        dom_one(acc, f);
        for (int i = ebits - 1; i >= 0; i--) {
            u32 sq[N], mu[N];
            dmul(sq, acc, acc, f);
            dmul(mu, sq, a, f);
            bool bit = (e[i >> 6] >> (i & 63)) & 1;
            copy_n<N>(acc, sq);
            select_n<N>(acc, mu, bit);
        }
        copy_n<N>(r, acc);
    }

    // same, for an exponent that is identical for every thread (public: p-2, (p+1)/4, ...):
    // the branch on the exponent bit is warp-uniform, so zero bits cost one squaring only.
    static FF_HD void dpow_uniform(u32* r, const u32* a, const u64* e, int ebits, const FieldParams& f) {
        u32 acc[N];
        dom_one(acc, f);
        for (int i = ebits - 1; i >= 0; i--) {
            dmul(acc, acc, acc, f);
            if ((e[i >> 6] >> (i & 63)) & 1) dmul(acc, acc, a, f);
        }
        copy_n<N>(r, acc);
    }
};
