// C-ABI of the mpyc_b200 engine (see include/mpyc_b200.h for the contract and the reference
// interfaces each entry point replaces).  This translation unit holds the host logic: field
// context construction (reduction-kind selection, Montgomery constants), Vandermonde / Lagrange
// table preparation and caching, argument checking, and the chunked host-buffer pipelines.
// Kernels live in kernels.cuh / gf256.cuh and are instantiated per limb count in inst_L*.cu.
#include <cuda_runtime.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <vector>

#include "../../include/mpyc_b200.h"
#include "field_setup.h"
#include "gf256.cuh"
#include "launch.h"
#include "prf_reduce.cuh"
#include "shake128.h"
#include "shake128_x8.h"

#define MPYC_API extern "C" __attribute__((visibility("default")))

std::atomic<unsigned long long> g_mpyc_launches{0};

static thread_local char tl_error[512] = "";

static int cuda_fail(cudaError_t e, const char* what) {
    snprintf(tl_error, sizeof tl_error, "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
    cudaGetLastError();   // clear the sticky-less error state
    if (e == cudaErrorMemoryAllocation) return MPYC_B200_ENOMEM;
    if (e == cudaErrorMisalignedAddress) {
        snprintf(tl_error, sizeof tl_error, "%s: buffers must be 16-byte aligned", what);
        return MPYC_B200_EINVAL;
    }
    return MPYC_B200_ECUDA;
}
#define CU(call)                                              \
    do {                                                      \
        cudaError_t e__ = (call);                             \
        if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
    } while (0)

static int fail(int code, const char* msg) {
    snprintf(tl_error, sizeof tl_error, "%s", msg);
    return code;
}

// ---------------------------------------------------------------------------------------
// grid sizing
// ---------------------------------------------------------------------------------------

int mpyc_grid_size(const void* kernel, size_t items, size_t dyn_smem) {
    static std::mutex mu;
    static std::map<std::tuple<const void*, int, size_t>, int> wave;   // (kernel, device, dynamic smem) -> CTAs per full wave
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    int w;
    {
        std::lock_guard<std::mutex> g(mu);
        auto key = std::make_tuple(kernel, dev, dyn_smem);
        auto it = wave.find(key);
        if (it == wave.end()) {
            int sms = 0, occ = 0;
            if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, MPYC_THREADS, dyn_smem) != cudaSuccess)
                return -1;
            if (occ < 1) occ = 1;
            w = sms * occ;
            wave[key] = w;
        } else {
            w = it->second;
        }
    }
    size_t need = (items + MPYC_THREADS - 1) / MPYC_THREADS;
    if (need < 1) need = 1;
    return (int)std::min<size_t>(need, (size_t)w);
}

int mpyc_sm_count() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return 132;
    return sms > 0 ? sms : 132;
}

// Scratch for split partials (K13, K14), from a pool of the library's own that keeps its memory between calls: the device's
// default pool returns freed memory at every synchronisation, and a fresh allocation cost a split call about 0.2 ms.
// The partials take at most a few MB (about two waves of threads' worth of elements).
cudaError_t mpyc_scratch_alloc(u64** p, size_t bytes, cudaStream_t st) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    {
        std::lock_guard<std::mutex> lock(mu);
        if (!pools[dev]) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            cudaMemPool_t pool = nullptr;
            e = cudaMemPoolCreate(&pool, &props);
            if (e != cudaSuccess) return e;
            uint64_t keep = UINT64_MAX;
            e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
            if (e != cudaSuccess) {
                cudaMemPoolDestroy(pool);
                return e;
            }
            pools[dev] = pool;
        }
    }
    return cudaMallocFromPoolAsync(reinterpret_cast<void**>(p), bytes, pools[dev], st);
}

// ---------------------------------------------------------------------------------------
// field handle
// ---------------------------------------------------------------------------------------

struct DevTable {
    u64* d = nullptr;
    u32 bytes = 0;
    bool full = false;
    u32 aux = 0;        // builder-defined (recombination tables: 1 = every row's sum of |lambda| is <= 2^31, see q32)
};

static thread_local u32 tl_table_aux = 0;   // set by a table builder, copied into DevTable::aux by get_table

struct mpyc_b200_field {
    FieldParams fp;
    int kind;           // MPYC_B200_KIND_*
    u32 gf_poly;        // GF(2^8): modulus polynomial (9 bits)
    std::mutex mu;
    std::map<std::string, DevTable> tables;   // key includes the device ordinal
};

template <int L, class Fn>
static int with_kind(const FieldParams& fp, Fn&& fn) {
    switch (fp.kind) {
        case KIND_GENERIC: return fn(std::integral_constant<int, L>(), std::integral_constant<int, KIND_GENERIC>());
        case KIND_PM_ALIGNED: return fn(std::integral_constant<int, L>(), std::integral_constant<int, KIND_PM_ALIGNED>());
        case KIND_PM_SHIFT: return fn(std::integral_constant<int, L>(), std::integral_constant<int, KIND_PM_SHIFT>());
    }
    return MPYC_B200_EINVAL;
}
// calls fn(L_constant, KIND_constant) on the host with the field's compile-time parameters
template <class Fn>
static int with_field(const FieldParams& fp, Fn&& fn) {
    switch (fp.L) {
        case 1: return with_kind<1>(fp, fn);
        case 2: return with_kind<2>(fp, fn);
        case 3: return with_kind<3>(fp, fn);
        case 4: return with_kind<4>(fp, fn);
    }
    return MPYC_B200_EINVAL;
}
template <class Fn>
static int with_limbs(int L, Fn&& fn) {
    switch (L) {
        case 1: return fn(std::integral_constant<int, 1>());
        case 2: return fn(std::integral_constant<int, 2>());
        case 3: return fn(std::integral_constant<int, 3>());
        case 4: return fn(std::integral_constant<int, 4>());
    }
    return MPYC_B200_EINVAL;
}

MPYC_API int mpyc_b200_version(void) { return 100; }

MPYC_API const char* mpyc_b200_strerror(int status) {
    switch (status) {
        case MPYC_B200_OK: return "ok";
        case MPYC_B200_EINVAL: return "invalid argument";
        case MPYC_B200_EUNSUPPORTED: return "unsupported field or shape";
        case MPYC_B200_EZERODIV: return "inverse of zero";
        case MPYC_B200_ECUDA: return "CUDA error";
        case MPYC_B200_ENOMEM: return "out of memory";
    }
    return "unknown status";
}

MPYC_API const char* mpyc_b200_last_error(void) { return tl_error; }

MPYC_API uint64_t mpyc_b200_launch_count(void) { return g_mpyc_launches.load(); }

MPYC_API int mpyc_b200_device_count(int* count) {
    if (!count) return fail(MPYC_B200_EINVAL, "count is null");
    CU(cudaGetDeviceCount(count));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_field_create(const uint64_t* modulus, int nlimbs, mpyc_b200_field** out) {
    if (!modulus || !out || nlimbs < 1) return fail(MPYC_B200_EINVAL, "field_create: bad arguments");
    while (nlimbs > 1 && modulus[nlimbs - 1] == 0) nlimbs--;
    if (nlimbs > MPYC_B200_MAX_LIMBS) return fail(MPYC_B200_EUNSUPPORTED, "modulus wider than 256 bits");
    if (!(modulus[0] & 1) || (nlimbs == 1 && modulus[0] < 3))
        return fail(MPYC_B200_EUNSUPPORTED, "modulus must be an odd prime >= 3");
    mpyc_b200_field* f = new (std::nothrow) mpyc_b200_field();
    if (!f) return fail(MPYC_B200_ENOMEM, "field_create: allocation failed");
    FieldParams& fp = f->fp;
    field_params_init(modulus, nlimbs, &fp);
    f->kind = fp.kind;
    f->gf_poly = 0;
    *out = f;
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_field_create_gf256(uint32_t modulus_poly, mpyc_b200_field** out) {
    if (!out) return fail(MPYC_B200_EINVAL, "out is null");
    if ((modulus_poly >> 8) != 1) return fail(MPYC_B200_EUNSUPPORTED, "modulus polynomial must have degree 8");
    // irreducibility check: x^(2^8) == x (mod f) and gcd conditions reduce, for degree 8, to
    // "no root and no factor of degree <= 4": test by trial division over all polynomials of degree 1..4
    for (u32 g = 2; g < 32; g++) {
        u32 a = modulus_poly;
        int dg = 31 - __builtin_clz(g);
        while (a && (31 - __builtin_clz(a)) >= dg) a ^= g << ((31 - __builtin_clz(a)) - dg);
        if (a == 0) return fail(MPYC_B200_EUNSUPPORTED, "modulus polynomial is reducible");
    }
    mpyc_b200_field* f = new (std::nothrow) mpyc_b200_field();
    if (!f) return fail(MPYC_B200_ENOMEM, "field_create: allocation failed");
    memset(&f->fp, 0, sizeof f->fp);
    f->kind = MPYC_B200_KIND_GF256;
    f->gf_poly = modulus_poly;
    f->fp.k = 8;
    *out = f;
    return MPYC_B200_OK;
}

MPYC_API void mpyc_b200_field_destroy(mpyc_b200_field* f) {
    if (!f) return;
    for (auto& kv : f->tables)
        if (kv.second.d) cudaFree(kv.second.d);
    delete f;
}

MPYC_API int mpyc_b200_field_info(const mpyc_b200_field* f, int* nlimbs, int* kind, int* bits, size_t* elem_bytes) {
    if (!f) return fail(MPYC_B200_EINVAL, "field is null");
    const bool gf = f->kind == MPYC_B200_KIND_GF256;
    if (nlimbs) *nlimbs = gf ? 0 : (int)f->fp.L;
    if (kind) *kind = f->kind;
    if (bits) *bits = (int)f->fp.k;
    if (elem_bytes) *elem_bytes = gf ? 1 : 8 * (size_t)f->fp.L;
    return MPYC_B200_OK;
}

// ---------------------------------------------------------------------------------------
// host-side field helpers (table preparation)
// ---------------------------------------------------------------------------------------

// canonical limbs of (v mod p) for a signed 64-bit integer v
template <int L, int KIND>
static void h_from_int(u32* r, int64_t v, const FieldParams& fp) {
    u64 mag = v < 0 ? (u64)(-(v + 1)) + 1 : (u64)v;
    zero_n<2 * L>(r);
    if (L == 1) mag %= fp.p[0];
    set64(r, 0, mag);   // L > 1: p >= 2^64 > mag
    if (v < 0) Fp<L, KIND>::neg(r, r, fp);
}

// canonical inverse by Fermat; returns false for zero
template <int L, int KIND>
static bool h_inv(u32* r, const u32* a, const FieldParams& fp) {
    constexpr int N = 2 * L;
    if (is_zero_n<N>(a)) return false;
    u32 e32[N], two[N];
    zero_n<N>(two);
    two[0] = 2;
    sub_n<N>(e32, as32(fp.p), two);
    u64 e[L];
    for (int i = 0; i < L; i++) e[i] = get64(e32, i);
    u32 x[N];
    Fp<L, KIND>::to_dom(x, a, fp);
    Fp<L, KIND>::dpow_uniform(x, x, e, (int)fp.k, fp);
    Fp<L, KIND>::from_dom(r, x, fp);
    return true;
}

static inline u32* w32(u64* x) { return reinterpret_cast<u32*>(x); }

static int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}

// look up or build a device table; `build` fills a host vector of u64 (already in final form)
template <class Build>
static int get_table(mpyc_b200_field* f, const std::string& key, DevTable* out, Build&& build) {
    std::lock_guard<std::mutex> g(f->mu);
    auto it = f->tables.find(key);
    if (it != f->tables.end()) {
        *out = it->second;
        return MPYC_B200_OK;
    }
    std::vector<u64> host;
    bool full = false;
    tl_table_aux = 0;
    int rc = build(host, full);
    if (rc != MPYC_B200_OK) return rc;
    if (host.size() % 2) host.push_back(0);   // bulk copies move multiples of 16 bytes
    if (host.empty()) host.assign(2, 0);
    DevTable t;
    t.bytes = (u32)(host.size() * sizeof(u64));
    t.full = full;
    t.aux = tl_table_aux;
    CU(cudaMalloc(&t.d, t.bytes));
    cudaError_t e = cudaMemcpy(t.d, host.data(), t.bytes, cudaMemcpyHostToDevice);
    // cudaMemcpy from PAGEABLE host memory returns once the data sits in the driver's staging buffer -- the DMA into
    // t.d may still be in flight -- and it runs on the legacy default stream, which the library's non-blocking
    // streams do not order against: a kernel launched right after could stage a half-written table.  With the GPU to
    // itself the DMA always won that race; with three MPyC parties time-slicing one GPU it lost it on the first use
    // of a table (round 2: wrong reshare results in real -M3 runs).  Wait for the copy before publishing the table.
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(t.d);
        return cuda_fail(e, "table upload");
    }
    f->tables[key] = t;
    *out = t;
    return MPYC_B200_OK;
}

#define MAX_SMEM_TABLE (40u * 1024u)   // tables are staged in the default 48 KB dynamic shared memory window

// Vandermonde table for share generation: row i, column j = (i+1)^j
static int build_split_table(const FieldParams& fp, int t, int m, std::vector<u64>& host, bool& full) {
    // 64-bit-constant form when m^t < 2^59 (t <= 8 keeps the (L+1)-limb sum below 2^(k+64))
    bool small = t <= 8;
    if (small) {
        long double lim = 1;
        for (int j = 0; j < t; j++) lim *= m;
        if (lim >= 576460752303423488.0L) small = false;   // 2^59
    }
    full = !small;
    if (small) {
        host.resize((size_t)m * (t + 1));
        for (int i = 0; i < m; i++) {
            u64 x = 1;
            for (int j = 0; j <= t; j++) {
                host[(size_t)i * (t + 1) + j] = x;
                x *= (u64)(i + 1);
            }
        }
        return MPYC_B200_OK;
    }
    return with_field(fp, [&](auto Lc, auto Kc) {
        constexpr int L = decltype(Lc)::value;
        constexpr int K = decltype(Kc)::value;
        host.resize((size_t)m * (t + 1) * L);
        for (int i = 0; i < m; i++) {
            u32 pt[2 * L], x[2 * L];
            h_from_int<L, K>(pt, i + 1, fp);
            h_from_int<L, K>(x, 1, fp);
            for (int j = 0; j <= t; j++) {
                u32 tf[2 * L];
                Fp<L, K>::to_dom(tf, x, fp);
                for (int l = 0; l < L; l++) host[((size_t)i * (t + 1) + j) * L + l] = get64(tf, l);
                Fp<L, K>::mul(x, x, pt, fp);
            }
        }
        return MPYC_B200_OK;
    });
}

// lambda[r][i] (canonical) for x-coordinates xs and recombination points x_rs
static int compute_lambda(const FieldParams& fp, const int64_t* xs, int k, const int64_t* x_rs, int width,
                          std::vector<u64>& lam) {
    return with_field(fp, [&](auto Lc, auto Kc) {
        constexpr int L = decltype(Lc)::value;
        constexpr int K = decltype(Kc)::value;
        typedef Fp<L, K> F;
        constexpr int N = 2 * L;
        lam.assign((size_t)width * k * L, 0);
        std::vector<u64> X((size_t)k * L);
        for (int i = 0; i < k; i++) h_from_int<L, K>(w32(&X[(size_t)i * L]), xs[i], fp);
        for (int r = 0; r < width; r++) {
            u32 xr[N];
            h_from_int<L, K>(xr, x_rs[r], fp);
            for (int i = 0; i < k; i++) {
                u32 num[N], den[N], d[N];
                h_from_int<L, K>(num, 1, fp);
                h_from_int<L, K>(den, 1, fp);
                for (int j = 0; j < k; j++) {
                    if (j == i) continue;
                    F::sub(d, xr, w32(&X[(size_t)j * L]), fp);
                    F::mul(num, num, d, fp);
                    F::sub(d, w32(&X[(size_t)i * L]), w32(&X[(size_t)j * L]), fp);
                    F::mul(den, den, d, fp);
                }
                u32 inv[N];
                if (!h_inv<L, K>(inv, den, fp)) return fail(MPYC_B200_EZERODIV, "recombination: repeated x-coordinate");
                F::mul(w32(&lam[((size_t)r * k + i) * L]), num, inv, fp);
            }
        }
        return MPYC_B200_OK;
    });
}

static void to_table_form(const FieldParams& fp, std::vector<u64>& v) {
    with_field(fp, [&](auto Lc, auto Kc) {
        constexpr int L = decltype(Lc)::value;
        constexpr int K = decltype(Kc)::value;
        for (size_t i = 0; i + L <= v.size(); i += L) Fp<L, K>::to_dom(w32(&v[i]), w32(&v[i]), fp);
        return 0;
    });
}

static std::string key_of(const char* tag, int dev, const int64_t* a, int na, const int64_t* b, int nb) {
    std::string s = tag;
    s += ":" + std::to_string(dev) + ":";
    for (int i = 0; i < na; i++) s += std::to_string(a[i]) + ",";
    s += "|";
    for (int i = 0; i < nb; i++) s += std::to_string(b[i]) + ",";
    return s;
}

#define REQUIRE_PRIME(f, what) \
    if ((f)->kind == MPYC_B200_KIND_GF256) return fail(MPYC_B200_EUNSUPPORTED, what ": not defined for GF(2^8)")

// ---------------------------------------------------------------------------------------
// elementwise
// ---------------------------------------------------------------------------------------

static int launch_status(cudaError_t e, const char* what) { return e == cudaSuccess ? MPYC_B200_OK : cuda_fail(e, what); }

static int binop_impl(const mpyc_b200_field* f, int op, const void* a, const void* b, const uint64_t* scal, void* out,
                      size_t n, void* stream) {
    if (!f || (n && (!a || !out))) return fail(MPYC_B200_EINVAL, "ff_binop: null argument");
    if (op < 0 || op > 3) return fail(MPYC_B200_EINVAL, "ff_binop: unknown op");
    if (n && op != OP_NEG && !b && !scal) return fail(MPYC_B200_EINVAL, "ff_binop: second operand missing");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256)
        return launch_status(gf256_binop(f->gf_poly, op, (const unsigned char*)a, (const unsigned char*)b,
                                         scal ? (int)(scal[0] & 0xFF) : -1, (unsigned char*)out, n, st),
                             "gf256 binop");
    if (scal && bit_length((const u64*)scal, (int)f->fp.L) > (int)f->fp.k)
        return fail(MPYC_B200_EINVAL, "ff_binop_scalar: scalar is not a canonical residue");
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::binop(f->fp, op, (const u64*)a, (const u64*)b, (const u64*)scal, (u64*)out, n, st),
                             "ff_binop launch");
    });
}

MPYC_API int mpyc_b200_ff_binop(const mpyc_b200_field* f, int op, const void* d_a, const void* d_b, void* d_out,
                                  size_t n, void* stream) {
    if (op < 0 || op > 2) return fail(MPYC_B200_EINVAL, "ff_binop: op must be ADD, SUB or MUL");
    return binop_impl(f, op, d_a, d_b, nullptr, d_out, n, stream);
}

MPYC_API int mpyc_b200_ff_binop_scalar(const mpyc_b200_field* f, int op, const void* d_a, const uint64_t* h_scalar,
                                         void* d_out, size_t n, void* stream) {
    if (op < 0 || op > 2 || !h_scalar) return fail(MPYC_B200_EINVAL, "ff_binop_scalar: bad arguments");
    return binop_impl(f, op, d_a, nullptr, h_scalar, d_out, n, stream);
}

MPYC_API int mpyc_b200_ff_neg(const mpyc_b200_field* f, const void* d_a, void* d_out, size_t n, void* stream) {
    return binop_impl(f, OP_NEG, d_a, nullptr, nullptr, d_out, n, stream);
}

// ---- pow family ------------------------------------------------------------------------------

// tiny host helpers on little-endian u64 arrays (exponent arithmetic)
static void wide_copy(u64* r, const u64* a, int n) { for (int i = 0; i < n; i++) r[i] = a[i]; }
static void wide_add(u64* r, const u64* a, int n) {
    unsigned __int128 cy = 0;
    for (int i = 0; i < n; i++) { cy += (unsigned __int128)r[i] + a[i]; r[i] = (u64)cy; cy >>= 64; }
}
static void wide_add_small(u64* r, int n, u64 v) {
    unsigned __int128 cy = v;
    for (int i = 0; i < n; i++) { cy += r[i]; r[i] = (u64)cy; cy >>= 64; }
}
static void wide_sub_small(u64* r, int n, u64 v) {
    for (int i = 0; i < n; i++) {
        u64 before = r[i];
        r[i] = before - v;
        v = before < v ? 1 : 0;
        if (!v) break;
    }
}

// "saw a zero" flag of the inverse family: one device int per (host thread, device), allocated on first use and
// kept (cudaMalloc / cudaFree per call cost more than the kernel at the demos' array sizes and synchronise the
// device).  acquire() returns it cleared on `st`; calls are one per thread per stream, so there is no sharing.
struct ZeroFlag {
    int* d = nullptr;
    int acquire(cudaStream_t st) {
        thread_local int* cache[16] = {nullptr};
        int dev = 0;
        CU(cudaGetDevice(&dev));
        if (dev < 0 || dev >= 16) return fail(MPYC_B200_EINVAL, "device ordinal out of range");
        if (!cache[dev]) CU(cudaMalloc(&cache[dev], sizeof(int)));
        d = cache[dev];
        CU(cudaMemsetAsync(d, 0, sizeof(int), st));
        return MPYC_B200_OK;
    }
};

static int pow_impl(const mpyc_b200_field* f, const void* d_a, const u64* e, int elimbs, int mode, bool check_zero,
                    void* d_out, unsigned char* d_out8, size_t n, cudaStream_t st) {
    ExpParams ex;
    memset(&ex, 0, sizeof ex);
    if (elimbs > 8) return fail(MPYC_B200_EUNSUPPORTED, "exponent wider than 512 bits");
    for (int i = 0; i < elimbs; i++) ex.e[i] = e[i];
    ex.ebits = bit_length(ex.e, 8);
    ZeroFlag zf;
    if (check_zero) {
        if (int zrc = zf.acquire(st)) return zrc;
    }
    int rc = with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::pow(f->fp, ex, mode, (const u64*)d_a, (u64*)d_out, d_out8, zf.d, n, st), "ff_pow launch");
    });
    if (rc != MPYC_B200_OK) return rc;
    if (check_zero) {
        int flag = 0;
        CU(cudaMemcpyAsync(&flag, zf.d, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (flag) return fail(MPYC_B200_EZERODIV, "inverse of zero");
    }
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_ff_pow(const mpyc_b200_field* f, const void* d_a, const uint64_t* h_exponent, int exp_nlimbs,
                                void* d_out, size_t n, void* stream) {
    if (!f || !h_exponent || exp_nlimbs < 1 || (n && (!d_a || !d_out))) return fail(MPYC_B200_EINVAL, "ff_pow: bad arguments");
    if (f->kind == MPYC_B200_KIND_GF256) {
        u64 e = h_exponent[0];
        for (int i = 1; i < exp_nlimbs; i++)
            if (h_exponent[i]) return fail(MPYC_B200_EUNSUPPORTED, "gf256 pow: reduce the exponent mod 255 first");
        return launch_status(gf256_pow(f->gf_poly, (const unsigned char*)d_a, e, (unsigned char*)d_out, nullptr, n,
                                       (cudaStream_t)stream), "gf256 pow");
    }
    return pow_impl(f, d_a, (const u64*)h_exponent, exp_nlimbs, 0, false, d_out, nullptr, n, (cudaStream_t)stream);
}

MPYC_API int mpyc_b200_ff_inv(const mpyc_b200_field* f, const void* d_a, void* d_out, size_t n, void* stream) {
    if (!f || (n && (!d_a || !d_out))) return fail(MPYC_B200_EINVAL, "ff_inv: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256) {
        ZeroFlag zf;
        if (int zrc = zf.acquire(st)) return zrc;
        int rc = launch_status(gf256_pow(f->gf_poly, (const unsigned char*)d_a, 254, (unsigned char*)d_out, zf.d, n, st), "gf256 inv");
        if (rc) return rc;
        int flag = 0;
        CU(cudaMemcpyAsync(&flag, zf.d, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        return flag ? fail(MPYC_B200_EZERODIV, "inverse of zero") : MPYC_B200_OK;
    }
    u64 e[4];
    wide_copy(e, f->fp.p, 4);
    wide_sub_small(e, 4, 2);   // p - 2
    if (d_a == d_out || n == 0) return pow_impl(f, d_a, e, 4, 0, true, d_out, nullptr, n, st);   // in place: per-element Fermat
    // Montgomery's trick: running products in d_out, one exponentiation per batch (k_inv_batch)
    ExpParams ex;
    memset(&ex, 0, sizeof ex);
    for (int i = 0; i < 4; i++) ex.e[i] = e[i];
    ex.ebits = bit_length(ex.e, 8);
    ZeroFlag zf;
    if (int zrc = zf.acquire(st)) return zrc;
    int rc = with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::inv_batch(f->fp, ex, (const u64*)d_a, (u64*)d_out, zf.d, n, st), "ff_inv launch");
    });
    if (rc != MPYC_B200_OK) return rc;
    int flag = 0;
    CU(cudaMemcpyAsync(&flag, zf.d, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return flag ? fail(MPYC_B200_EZERODIV, "inverse of zero") : MPYC_B200_OK;
}

MPYC_API int mpyc_b200_ff_sqrt(const mpyc_b200_field* f, const void* d_a, int inverse, void* d_out, size_t n, void* stream) {
    if (!f || (n && (!d_a || !d_out))) return fail(MPYC_B200_EINVAL, "ff_sqrt: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256) {
        // finfields.py:1552-1563: a^(q/2), inverse: a^(q/2 - 1)
        ZeroFlag zf;
        if (inverse) {
            if (int zrc = zf.acquire(st)) return zrc;
        }
        int rc = launch_status(gf256_pow(f->gf_poly, (const unsigned char*)d_a, inverse ? 127 : 128, (unsigned char*)d_out, zf.d, n, st), "gf256 sqrt");
        if (rc || !inverse) return rc;
        int flag = 0;
        CU(cudaMemcpyAsync(&flag, zf.d, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        return flag ? fail(MPYC_B200_EZERODIV, "no inverse sqrt of 0") : MPYC_B200_OK;
    }
    if ((f->fp.p[0] & 3) != 3) return fail(MPYC_B200_EUNSUPPORTED, "ff_sqrt: batched path needs a Blum prime (p % 4 == 3)");
    // e = (p+1)/4, or (3p-5)/4 for the inverse square root; up to 258 bits -> 5 limbs
    u64 e[8] = {0}, t[5] = {f->fp.p[0], f->fp.p[1], f->fp.p[2], f->fp.p[3], 0};
    if (!inverse) {
        wide_add_small(t, 5, 1);
    } else {
        u64 pp[5];
        wide_copy(pp, t, 5);
        wide_add(t, pp, 5);
        wide_add(t, pp, 5);        // 3p
        wide_sub_small(t, 5, 5);   // 3p - 5
    }
    for (int i = 0; i < 5; i++) e[i] = (t[i] >> 2) | (i < 4 ? (t[i + 1] << 62) : 0);
    return pow_impl(f, d_a, e, 5, 0, inverse != 0, d_out, nullptr, n, st);
}

MPYC_API int mpyc_b200_ff_is_sqr(const mpyc_b200_field* f, const void* d_a, uint8_t* d_out_u8, size_t n, void* stream) {
    if (!f || (n && (!d_a || !d_out_u8))) return fail(MPYC_B200_EINVAL, "ff_is_sqr: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256) {   // every element of GF(2^8) is a square
        CU(cudaMemsetAsync(d_out_u8, 1, n, st));
        return MPYC_B200_OK;
    }
    u64 e[4];
    for (int i = 0; i < 4; i++) e[i] = (f->fp.p[i] >> 1) | (i < 3 ? (f->fp.p[i + 1] << 63) : 0);   // (p-1)/2
    return pow_impl(f, d_a, e, 4, 1, false, nullptr, d_out_u8, n, st);
}

MPYC_API int mpyc_b200_ff_matmul(const mpyc_b200_field* f, const void* d_a, const void* d_b, void* d_c, size_t r,
                                 size_t k, size_t c, void* stream) {
    if (!f) return fail(MPYC_B200_EINVAL, "ff_matmul: field is null");
    if (r == 0 || c == 0) return MPYC_B200_OK;
    if (!d_c || (k && (!d_a || !d_b))) return fail(MPYC_B200_EINVAL, "ff_matmul: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256)
        return launch_status(gf256_matmul(f->gf_poly, (const unsigned char*)d_a, (const unsigned char*)d_b,
                                          (unsigned char*)d_c, r, k, c, st), "gf256 matmul");
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        return launch_status(Launch<LL>::matmul(f->fp, (const u64*)d_a, (const u64*)d_b, (u64*)d_c, r, k, c, st),
                             "ff_matmul launch");
    });
}

// ---------------------------------------------------------------------------------------
// K6: protocol-local algebra on raw share values (local.cuh; prime fields)
// ---------------------------------------------------------------------------------------

static int prime_only(const mpyc_b200_field* f, const char* what) {
    if (!f) return fail(MPYC_B200_EINVAL, what);
    if (f->kind == MPYC_B200_KIND_GF256) return fail(MPYC_B200_EUNSUPPORTED, "protocol-local kernels cover prime fields only");
    return MPYC_B200_OK;
}

static bool canonical(const mpyc_b200_field* f, const uint64_t* x) {
    for (int i = (int)f->fp.L - 1; i >= 0; i--) {
        if (x[i] < f->fp.p[i]) return true;
        if (x[i] > f->fp.p[i]) return false;
    }
    return false;
}

MPYC_API int mpyc_b200_ff_fma(const mpyc_b200_field* f, const void* d_a, const void* d_b, const void* d_c, void* d_out,
                              size_t n, void* stream) {
    if (int rc = prime_only(f, "ff_fma: field is null")) return rc;
    if (n && (!d_a || !d_c || !d_out)) return fail(MPYC_B200_EINVAL, "ff_fma: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::fma(f->fp, d_b == nullptr, (const u64*)d_a, (const u64*)d_b, (const u64*)d_c,
                                            (u64*)d_out, n, st), "ff_fma launch");
    });
}

MPYC_API int mpyc_b200_ff_axpb(const mpyc_b200_field* f, const void* d_a, const uint64_t* h_s, const uint64_t* h_t,
                               void* d_out, size_t n, void* stream) {
    if (int rc = prime_only(f, "ff_axpb: field is null")) return rc;
    if (!h_s || !h_t || (n && (!d_a || !d_out))) return fail(MPYC_B200_EINVAL, "ff_axpb: null argument");
    if (!canonical(f, h_s) || !canonical(f, h_t)) return fail(MPYC_B200_EINVAL, "ff_axpb: scalars must be canonical residues");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::axpb(f->fp, (const u64*)d_a, (const u64*)h_s, (const u64*)h_t, (u64*)d_out, n, st),
                             "ff_axpb launch");
    });
}

MPYC_API int mpyc_b200_ff_low_bits(const mpyc_b200_field* f, const void* d_a, int nbits, void* d_out, size_t n, void* stream) {
    if (int rc = prime_only(f, "ff_low_bits: field is null")) return rc;
    if (nbits < 0 || (n && (!d_a || !d_out))) return fail(MPYC_B200_EINVAL, "ff_low_bits: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::low_bits(f->fp, (const u64*)d_a, nbits, (u64*)d_out, n, st), "ff_low_bits launch");
    });
}

MPYC_API int mpyc_b200_ff_nonzero(const mpyc_b200_field* f, const void* d_a, uint8_t* d_out_u8, uint64_t* d_count, size_t n,
                                  void* stream) {
    if (int rc = prime_only(f, "ff_nonzero: field is null")) return rc;
    if (!d_count || (n && !d_a)) return fail(MPYC_B200_EINVAL, "ff_nonzero: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    CU(cudaMemsetAsync(d_count, 0, sizeof(uint64_t), st));
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::nonzero(f->fp, (const u64*)d_a, d_out_u8, (unsigned long long*)d_count, n, st),
                             "ff_nonzero launch");
    });
}

MPYC_API int mpyc_b200_ff_bits_compose(const mpyc_b200_field* f, const void* d_bits, size_t n, int nbits, int descending,
                                       void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_bits_compose: field is null")) return rc;
    if (nbits < 1 || nbits > 4096 || (n && (!d_bits || !d_out))) return fail(MPYC_B200_EINVAL, "ff_bits_compose: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::bits_compose(f->fp, (const u64*)d_bits, (u64*)d_out, n, nbits, descending != 0, st),
                             "ff_bits_compose launch");
    });
}

MPYC_API int mpyc_b200_ff_bits_decompose(const mpyc_b200_field* f, const void* d_c, size_t n, int nbits, int descending,
                                         void* d_out, size_t out_stride, void* stream) {
    if (int rc = prime_only(f, "ff_bits_decompose: field is null")) return rc;
    if (nbits < 0 || out_stride < n || (n && nbits && (!d_c || !d_out)))
        return fail(MPYC_B200_EINVAL, "ff_bits_decompose: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (nbits == 0) return MPYC_B200_OK;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::bits_decompose(f->fp, (const u64*)d_c, (u64*)d_out, out_stride, n, nbits, descending != 0, st),
                             "ff_bits_decompose launch");
    });
}

MPYC_API int mpyc_b200_ff_transpose(const mpyc_b200_field* f, const void* d_in, size_t rows, size_t cols, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_transpose: field is null")) return rc;
    if (rows && cols && (!d_in || !d_out)) return fail(MPYC_B200_EINVAL, "ff_transpose: null buffer");
    if (d_in == d_out && rows > 1 && cols > 1) return fail(MPYC_B200_EINVAL, "ff_transpose: in place is not supported");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::transpose(f->fp, (const u64*)d_in, (u64*)d_out, rows, cols, st), "ff_transpose launch");
    });
}

MPYC_API int mpyc_b200_ff_cumsum_rows(const mpyc_b200_field* f, const void* d_in, size_t rows, size_t cols, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_cumsum_rows: field is null")) return rc;
    if (rows && cols && (!d_in || !d_out)) return fail(MPYC_B200_EINVAL, "ff_cumsum_rows: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::scan_axis(f->fp, (const u64*)d_in, (u64*)d_out, 1, rows, cols, false, st), "ff_cumsum_rows launch");
    });
}

// ---------------------------------------------------------------------------------------
// K7: sums and running sums along an axis (reduce.cuh; prime fields)
// ---------------------------------------------------------------------------------------

// outer * rows * inner elements of L limbs, addressable in bytes
static bool axis_size_ok(const mpyc_b200_field* f, size_t outer, size_t rows, size_t inner) {
    size_t n = 0;
    return !__builtin_mul_overflow(outer, rows, &n) && !__builtin_mul_overflow(n, inner, &n) &&
           !__builtin_mul_overflow(n, (size_t)f->fp.L * sizeof(u64), &n);
}

MPYC_API int mpyc_b200_ff_sum_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                                   const uint64_t* initial, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_sum_axis: field is null")) return rc;
    if (!axis_size_ok(f, outer, len, inner) || !axis_size_ok(f, outer, 1, inner)) return fail(MPYC_B200_EINVAL, "ff_sum_axis: size overflow");
    if (outer == 0 || inner == 0) return MPYC_B200_OK;
    if (!d_out || (len && !d_in)) return fail(MPYC_B200_EINVAL, "ff_sum_axis: null buffer");
    if (initial && !canonical(f, initial)) return fail(MPYC_B200_EINVAL, "ff_sum_axis: initial must be a canonical residue");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::sum_axis(f->fp, (const u64*)d_in, (u64*)d_out, outer, len, inner, (const u64*)initial, st),
                             "ff_sum_axis launch");
    });
}

MPYC_API int mpyc_b200_ff_cumsum_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                                      int include_initial, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_cumsum_axis: field is null")) return rc;
    const size_t inc = include_initial ? 1 : 0;
    if (len > SIZE_MAX - inc || !axis_size_ok(f, outer, len + inc, inner)) return fail(MPYC_B200_EINVAL, "ff_cumsum_axis: size overflow");
    if (outer == 0 || inner == 0 || len + inc == 0) return MPYC_B200_OK;
    if (!d_out || (len && !d_in)) return fail(MPYC_B200_EINVAL, "ff_cumsum_axis: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::scan_axis(f->fp, (const u64*)d_in, (u64*)d_out, outer, len, inner, inc != 0, st),
                             "ff_cumsum_axis launch");
    });
}

// ---------------------------------------------------------------------------------------
// K8: strided views, joins and broadcast arithmetic (layout.cuh)
// ---------------------------------------------------------------------------------------

// A view's element count (0 if empty) after checking its shape and that every element lies in [0, len): the lowest and
// highest offsets are offset + the sum over axes of the extreme o_k * stride[k].  Returns -1 on a bad view.
static long long view_check(const mpyc_b200_view* v, size_t len, bool allow_index) {
    if (!v || v->rank < 0 || v->rank > MPYC_B200_VIEW_RANK) return -1;
    if (v->index_axis != -1 && (!allow_index || v->index_axis < 0 || v->index_axis >= v->rank || !v->index)) return -1;
    long long n = 1;
    for (int k = 0; k < v->rank; k++) {
        if (v->extent[k] < 0 || __builtin_mul_overflow(n, v->extent[k], &n)) return -1;
    }
    if (n == 0) return 0;
    __int128 lo = v->offset, hi = v->offset;
    for (int k = 0; k < v->rank; k++) {
        int64_t omin = 0, omax = v->extent[k] - 1;
        if (k == v->index_axis) {
            omin = omax = v->index[0];
            for (int64_t c = 1; c < v->extent[k]; c++) omin = std::min(omin, v->index[c]), omax = std::max(omax, v->index[c]);
        }
        const __int128 a = (__int128)omin * v->stride[k], b = (__int128)omax * v->stride[k];
        lo += std::min(a, b);
        hi += std::max(a, b);
    }
    if (lo < 0 || hi >= (__int128)len) return -1;
    return n;
}

static bool bytes_overlap(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return na && nb && x < y + nb && y < x + na;
}

static bool same_extents(const mpyc_b200_view* a, const mpyc_b200_view* b) {
    if (a->rank != b->rank) return false;
    for (int k = 0; k < a->rank; k++)
        if (a->extent[k] != b->extent[k]) return false;
    return true;
}

MPYC_API int mpyc_b200_copy_view(size_t elem_bytes, const void* d_src, size_t src_len, const mpyc_b200_view* src, void* d_dst,
                                 size_t dst_len, const mpyc_b200_view* dst, void* stream) {
    if (elem_bytes != 1 && elem_bytes != 8 && elem_bytes != 16 && elem_bytes != 24 && elem_bytes != 32)
        return fail(MPYC_B200_EINVAL, "copy_view: element size must be 1, 8, 16, 24 or 32 bytes");
    size_t sb = 0, db = 0;
    if (__builtin_mul_overflow(src_len, elem_bytes, &sb) || __builtin_mul_overflow(dst_len, elem_bytes, &db))
        return fail(MPYC_B200_EINVAL, "copy_view: buffer size overflow");
    const long long ns = view_check(src, src_len, true), nd = view_check(dst, dst_len, true);
    if (ns < 0 || nd < 0) return fail(MPYC_B200_EINVAL, "copy_view: bad view (rank > 6, negative extent or outside its buffer)");
    if (!same_extents(src, dst)) return fail(MPYC_B200_EINVAL, "copy_view: views of different extents");
    if (ns == 0) return MPYC_B200_OK;
    if (!d_src || !d_dst) return fail(MPYC_B200_EINVAL, "copy_view: null buffer");
    if (bytes_overlap(d_src, sb, d_dst, db)) return fail(MPYC_B200_EINVAL, "copy_view: source and destination overlap");
    CopyPlan p = {};
    p.rank = src->rank;
    p.six = src->index_axis, p.dix = dst->index_axis;
    p.soff = src->offset, p.doff = dst->offset;
    for (int k = 0; k < p.rank; k++) p.ext[k] = src->extent[k], p.sstr[k] = src->stride[k], p.dstr[k] = dst->stride[k];
    cudaStream_t st = (cudaStream_t)stream;
    // index tables: uploaded into stream-ordered scratch, freed after the copy
    const size_t ni = p.six >= 0 ? (size_t)p.ext[p.six] : 0, nj = p.dix >= 0 ? (size_t)p.ext[p.dix] : 0;
    long long* tab = nullptr;
    if (ni + nj) {
        CU(cudaMallocAsync(&tab, (ni + nj) * sizeof(long long), st));
        cudaError_t e = cudaSuccess;
        if (ni) e = cudaMemcpyAsync(tab, src->index, ni * sizeof(long long), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess && nj) e = cudaMemcpyAsync(tab + ni, dst->index, nj * sizeof(long long), cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) {
            cudaFreeAsync(tab, st);
            return cuda_fail(e, "copy_view: index upload");
        }
        p.sidx = ni ? tab : nullptr;
        p.didx = nj ? tab + ni : nullptr;
    }
    const cudaError_t e = launch_copy_view(p, elem_bytes, d_src, d_dst, st);
    if (tab) cudaFreeAsync(tab, st);
    return launch_status(e, "copy_view launch");
}

MPYC_API int mpyc_b200_ff_binop_view(const mpyc_b200_field* f, int op, const void* d_a, size_t a_len, const mpyc_b200_view* a,
                                     const void* d_b, size_t b_len, const mpyc_b200_view* b, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_binop_view: field is null")) return rc;
    if (op < 0 || op > 2) return fail(MPYC_B200_EINVAL, "ff_binop_view: op must be ADD, SUB or MUL");
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t ab = 0, bb = 0, ob = 0;
    if (__builtin_mul_overflow(a_len, E, &ab) || __builtin_mul_overflow(b_len, E, &bb))
        return fail(MPYC_B200_EINVAL, "ff_binop_view: buffer size overflow");
    const long long na = view_check(a, a_len, false), nb = view_check(b, b_len, false);
    if (na < 0 || nb < 0) return fail(MPYC_B200_EINVAL, "ff_binop_view: bad view (rank > 6, negative extent, index table or outside its buffer)");
    if (!same_extents(a, b)) return fail(MPYC_B200_EINVAL, "ff_binop_view: views of different extents");
    if (na == 0) return MPYC_B200_OK;
    if (__builtin_mul_overflow((size_t)na, E, &ob)) return fail(MPYC_B200_EINVAL, "ff_binop_view: size overflow");
    if (!d_a || !d_b || !d_out) return fail(MPYC_B200_EINVAL, "ff_binop_view: null buffer");
    if (bytes_overlap(d_out, ob, d_a, ab) || bytes_overlap(d_out, ob, d_b, bb))
        return fail(MPYC_B200_EINVAL, "ff_binop_view: out overlaps an operand");
    BinopPlan p = {};
    p.rank = a->rank;
    p.aoff = a->offset, p.boff = b->offset;
    for (int k = 0; k < p.rank; k++) p.ext[k] = a->extent[k], p.astr[k] = a->stride[k], p.bstr[k] = b->stride[k];
    if (p.rank == 0) p.rank = 1, p.ext[0] = 1;
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::binop_view(f->fp, op, p, (const u64*)d_a, (const u64*)d_b, (u64*)d_out, st),
                             "ff_binop_view launch");
    });
}

// ---------------------------------------------------------------------------------------
// K9: determinants, solves and inverses (linalg.cuh; prime fields)
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_ff_det(const mpyc_b200_field* f, const void* d_a, size_t batch, size_t n, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_det: field is null")) return rc;
    if (n == 0) return fail(MPYC_B200_EINVAL, "ff_det: n must be at least 1");
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t ab = 0, ob = 0;
    if (__builtin_mul_overflow(n, n, &ab) || __builtin_mul_overflow(ab, batch, &ab) || __builtin_mul_overflow(ab, E, &ab) ||
        __builtin_mul_overflow(batch, E, &ob))
        return fail(MPYC_B200_EINVAL, "ff_det: size overflow");
    if (batch == 0) return MPYC_B200_OK;
    if (!d_a || !d_out) return fail(MPYC_B200_EINVAL, "ff_det: null buffer");
    if (bytes_overlap(d_a, ab, d_out, ob)) return fail(MPYC_B200_EINVAL, "ff_det: out overlaps the matrices");
    return launch_status(launch_det(f->fp, (const u64*)d_a, batch, n, (u64*)d_out, (cudaStream_t)stream), "ff_det launch");
}

MPYC_API int mpyc_b200_ff_solve(const mpyc_b200_field* f, const void* d_a, size_t n, const void* d_b, size_t nrhs, void* d_x,
                                void* stream) {
    if (int rc = prime_only(f, "ff_solve: field is null")) return rc;
    if (n == 0) return fail(MPYC_B200_EINVAL, "ff_solve: n must be at least 1");
    if (!d_b && nrhs != n) return fail(MPYC_B200_EINVAL, "ff_solve: the identity right-hand side has n columns");
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t ab = 0, bb = 0, w = 0;
    if (__builtin_mul_overflow(n, n, &ab) || __builtin_mul_overflow(ab, E, &ab) || __builtin_mul_overflow(n, nrhs, &bb) ||
        __builtin_mul_overflow(bb, E, &bb) || __builtin_add_overflow(n, nrhs, &w) || __builtin_mul_overflow(w, n, &w) ||
        __builtin_mul_overflow(w, E, &w))
        return fail(MPYC_B200_EINVAL, "ff_solve: size overflow");
    if (!d_a || (nrhs && !d_x)) return fail(MPYC_B200_EINVAL, "ff_solve: null buffer");
    if (bytes_overlap(d_x, bb, d_a, ab) || (d_b && bytes_overlap(d_x, bb, d_b, bb)))
        return fail(MPYC_B200_EINVAL, "ff_solve: x overlaps an operand");
    int singular = 0;
    const int rc = launch_status(launch_solve(f->fp, (const u64*)d_a, n, (const u64*)d_b, nrhs, (u64*)d_x, &singular,
                                              (cudaStream_t)stream), "ff_solve launch");
    if (rc != MPYC_B200_OK) return rc;
    return singular ? fail(MPYC_B200_EZERODIV, "no inverse exists") : MPYC_B200_OK;
}

// ---------------------------------------------------------------------------------------
// K10: 1-D convolution (conv.cuh; prime fields)
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_ff_convolve(const mpyc_b200_field* f, const void* d_a, size_t m, const void* d_b, size_t n, size_t lo,
                                   size_t count, void* d_c, void* stream) {
    if (int rc = prime_only(f, "ff_convolve: field is null")) return rc;
    if (m == 0 || n == 0) return fail(MPYC_B200_EINVAL, "ff_convolve: empty operand");
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t full = 0, end = 0, ab = 0, bb = 0, cb = 0;
    if (__builtin_add_overflow(m, n - 1, &full) || __builtin_add_overflow(lo, count, &end) || __builtin_mul_overflow(m, E, &ab) ||
        __builtin_mul_overflow(n, E, &bb) || __builtin_mul_overflow(count, E, &cb) || full > (size_t)INT64_MAX / E)
        return fail(MPYC_B200_EINVAL, "ff_convolve: size overflow");
    if (end > full) return fail(MPYC_B200_EINVAL, "ff_convolve: window past the full result");
    if (count == 0) return MPYC_B200_OK;
    if (!d_a || !d_b || !d_c) return fail(MPYC_B200_EINVAL, "ff_convolve: null buffer");
    if (bytes_overlap(d_c, cb, d_a, ab) || bytes_overlap(d_c, cb, d_b, bb))
        return fail(MPYC_B200_EINVAL, "ff_convolve: c overlaps an operand");
    return launch_status(launch_convolve(f->fp, (const u64*)d_a, m, (const u64*)d_b, n, lo, count, (u64*)d_c, (cudaStream_t)stream),
                         "ff_convolve launch");
}

// ---------------------------------------------------------------------------------------
// K11: division (k_inv_batch with a numerator) and selection (select.cuh; prime fields)
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_ff_div(const mpyc_b200_field* f, const void* d_num, const void* d_den, void* d_out, size_t n,
                              void* stream) {
    if (int rc = prime_only(f, "ff_div: field is null")) return rc;
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t bytes = 0;
    if (__builtin_mul_overflow(n, E, &bytes) || bytes > (size_t)INT64_MAX) return fail(MPYC_B200_EINVAL, "ff_div: size overflow");
    if (n == 0) return MPYC_B200_OK;
    if (!d_num || !d_den || !d_out) return fail(MPYC_B200_EINVAL, "ff_div: null buffer");
    // the forward pass leaves prefix products in out, which the backward pass reads next to num and den
    if (bytes_overlap(d_out, bytes, d_num, bytes) || bytes_overlap(d_out, bytes, d_den, bytes))
        return fail(MPYC_B200_EINVAL, "ff_div: out overlaps an operand");
    cudaStream_t st = (cudaStream_t)stream;
    u64 e[4];
    wide_copy(e, f->fp.p, 4);
    wide_sub_small(e, 4, 2);   // p - 2
    ExpParams ex;
    memset(&ex, 0, sizeof ex);
    for (int i = 0; i < 4; i++) ex.e[i] = e[i];
    ex.ebits = bit_length(ex.e, 8);
    ZeroFlag zf;
    if (int zrc = zf.acquire(st)) return zrc;
    int rc = with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::inv_batch(f->fp, ex, (const u64*)d_den, (u64*)d_out, zf.d, n, st, (const u64*)d_num),
                             "ff_div launch");
    });
    if (rc != MPYC_B200_OK) return rc;
    int flag = 0;
    CU(cudaMemcpyAsync(&flag, zf.d, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return flag ? fail(MPYC_B200_EZERODIV, "inverse of zero") : MPYC_B200_OK;
}

MPYC_API int mpyc_b200_ff_select(const mpyc_b200_field* f, const uint8_t* d_mask, int invert, const void* d_x,
                                 const uint64_t* h_x_st, const void* d_y, const uint64_t* h_y_st, void* d_out, size_t n,
                                 void* stream) {
    if (int rc = prime_only(f, "ff_select: field is null")) return rc;
    if (!h_x_st || !h_y_st) return fail(MPYC_B200_EINVAL, "ff_select: null affine map");
    const size_t L = f->fp.L, E = L * sizeof(u64);
    for (const uint64_t* m : {h_x_st, h_y_st})
        if (!canonical(f, m) || !canonical(f, m + L)) return fail(MPYC_B200_EINVAL, "ff_select: scalars must be canonical residues");
    size_t bytes = 0;
    if (__builtin_mul_overflow(n, E, &bytes) || bytes > (size_t)INT64_MAX) return fail(MPYC_B200_EINVAL, "ff_select: size overflow");
    if (n == 0) return MPYC_B200_OK;
    if (!d_mask || !d_out) return fail(MPYC_B200_EINVAL, "ff_select: null buffer");
    if (bytes_overlap(d_out, bytes, d_mask, n) || (d_x && bytes_overlap(d_out, bytes, d_x, bytes)) ||
        (d_y && bytes_overlap(d_out, bytes, d_y, bytes)))
        return fail(MPYC_B200_EINVAL, "ff_select: out overlaps an operand");
    const u64* xst = (const u64*)h_x_st;
    const u64* yst = (const u64*)h_y_st;
    return launch_status(launch_select(f->fp, d_mask, invert != 0, (const u64*)d_x, xst, xst + L, (const u64*)d_y, yst, yst + L,
                                       (u64*)d_out, n, (cudaStream_t)stream),
                         "ff_select launch");
}

// ---------------------------------------------------------------------------------------
// K12: per-element exponents (powexp.cuh; prime fields)
// ---------------------------------------------------------------------------------------

// The comb window of the fixed-base form: the widest w <= 8 whose tables (one, or two with signs) fit MPYC_PE_SMEM_MAX.
// An element costs ceil(B / w) - 1 products, the host ceil(B / w) 2^w to build a table.
static int powexp_window(int bits, int L, int ntab, int* nwin, u32* bytes) {
    for (int w = 8; w >= 1; w--) {
        const int nw = (bits + w - 1) / w;
        const size_t b = (size_t)ntab * ((size_t)nw << w) * L * sizeof(u64);
        if (b <= MPYC_PE_SMEM_MAX) {
            *nwin = nw;
            *bytes = (u32)b;
            return w;
        }
    }
    return 0;   // unreachable: w = 1 needs 2 * 256 * 2 * 32 bytes at most
}

// g(s, j, d) = b_s^(d 2^(w j)) in the domain, b_0 = base, b_1 = base^-1 (ntab == 2); false when base == 0 and ntab == 2
static bool powexp_tables(const FieldParams& fp, const u64* base, int w, int nwin, int ntab, std::vector<u64>& host) {
    return with_field(fp, [&](auto Lc, auto Kc) {
        constexpr int L = decltype(Lc)::value;
        constexpr int K = decltype(Kc)::value;
        typedef Fp<L, K> F;
        constexpr int N = 2 * L;
        const size_t D = (size_t)1 << w;
        host.assign((size_t)ntab * nwin * D * L, 0);
        for (int s = 0; s < ntab; s++) {
            u32 b[N], g[N];
            for (int i = 0; i < L; i++) set64(b, i, base[i]);
            if (s == 1 && !h_inv<L, K>(b, b, fp)) return 0;
            F::to_dom(g, b, fp);                                  // g = b^(2^(w j)) for the current j
            for (int j = 0; j < nwin; j++) {
                u64* row = &host[((size_t)s * nwin + j) * D * L];
                u32 x[N];
                F::dom_one(x, fp);
                for (size_t d = 0; d < D; d++) {
                    for (int i = 0; i < L; i++) row[d * L + i] = get64(x, i);
                    F::dmul(x, x, g, fp);
                }
                copy_n<N>(g, x);                                  // g^(2^w)
            }
        }
        return 1;
    }) == 1;
}

MPYC_API int mpyc_b200_ff_pow_exp(const mpyc_b200_field* f, const void* d_base, const uint64_t* h_base, const uint64_t* d_exps,
                                  int exp_limbs, int exp_bits, const uint8_t* d_signs, size_t n, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_pow_exp: field is null")) return rc;
    if ((d_base == nullptr) == (h_base == nullptr)) return fail(MPYC_B200_EINVAL, "ff_pow_exp: give exactly one of the two bases");
    if (exp_limbs < 1 || exp_limbs > 4) return fail(MPYC_B200_EINVAL, "ff_pow_exp: exp_limbs must be 1..4");
    if (exp_bits < 0 || exp_bits > 64 * exp_limbs) return fail(MPYC_B200_EINVAL, "ff_pow_exp: exp_bits exceeds 64 * exp_limbs");
    if (d_signs && d_base) return fail(MPYC_B200_EINVAL, "ff_pow_exp: signs need the fixed base");
    if (h_base && !canonical(f, h_base)) return fail(MPYC_B200_EINVAL, "ff_pow_exp: the base must be a canonical residue");
    const size_t L = f->fp.L;
    size_t bytes = 0, ebytes = 0;
    if (__builtin_mul_overflow(n, L * sizeof(u64), &bytes) || bytes > (size_t)INT64_MAX ||
        __builtin_mul_overflow(n, (size_t)exp_limbs * sizeof(u64), &ebytes) || ebytes > (size_t)INT64_MAX)
        return fail(MPYC_B200_EINVAL, "ff_pow_exp: size overflow");
    if (n == 0) return MPYC_B200_OK;
    if (!d_exps || !d_out) return fail(MPYC_B200_EINVAL, "ff_pow_exp: null buffer");
    if (bytes_overlap(d_out, bytes, d_exps, ebytes) || (d_signs && bytes_overlap(d_out, bytes, d_signs, n)) ||
        (d_base && bytes_overlap(d_out, bytes, d_base, bytes)))
        return fail(MPYC_B200_EINVAL, "ff_pow_exp: out overlaps an operand");
    cudaStream_t st = (cudaStream_t)stream;
    if (d_base)
        return launch_status(launch_powexp(f->fp, (const u64*)d_base, nullptr, 0, 0, 0, (const u64*)d_exps, exp_limbs, exp_bits,
                                           nullptr, (u64*)d_out, n, st),
                             "ff_pow_exp launch");
    const int ntab = d_signs ? 2 : 1;
    int nwin = 0;
    u32 tab_bytes = 0;
    const int w = powexp_window(std::max(exp_bits, 1), (int)L, ntab, &nwin, &tab_bytes);
    std::vector<u64> host;
    if (!powexp_tables(f->fp, (const u64*)h_base, w, nwin, ntab, host)) return fail(MPYC_B200_EZERODIV, "inverse of zero");
    u64* tab = nullptr;
    CU(cudaMallocAsync(&tab, tab_bytes, st));
    cudaError_t e = cudaMemcpyAsync(tab, host.data(), tab_bytes, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // host vector goes out of scope
    if (e == cudaSuccess)
        e = launch_powexp(f->fp, nullptr, tab, tab_bytes, w, nwin, (const u64*)d_exps, exp_limbs, exp_bits, d_signs, (u64*)d_out, n, st);
    cudaFreeAsync(tab, st);
    return launch_status(e, "ff_pow_exp launch");
}

// ---------------------------------------------------------------------------------------
// K13: products, running products and all / any along an axis (prod.cuh; prime fields)
// ---------------------------------------------------------------------------------------

// byte counts of an (outer, len, inner) input and an (outer, out_len, inner) output; false when one overflows
static bool axis_bytes(const mpyc_b200_field* f, size_t outer, size_t len, size_t out_len, size_t inner, size_t* in_b, size_t* out_b) {
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    return !__builtin_mul_overflow(outer, len, in_b) && !__builtin_mul_overflow(*in_b, inner, in_b) &&
           !__builtin_mul_overflow(*in_b, E, in_b) && *in_b <= (size_t)INT64_MAX && !__builtin_mul_overflow(outer, out_len, out_b) &&
           !__builtin_mul_overflow(*out_b, inner, out_b) && !__builtin_mul_overflow(*out_b, E, out_b) && *out_b <= (size_t)INT64_MAX;
}

MPYC_API int mpyc_b200_ff_prod_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                                    const uint64_t* initial, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_prod_axis: field is null")) return rc;
    size_t ib = 0, ob = 0;
    if (!axis_bytes(f, outer, len, 1, inner, &ib, &ob)) return fail(MPYC_B200_EINVAL, "ff_prod_axis: size overflow");
    if (initial && !canonical(f, initial)) return fail(MPYC_B200_EINVAL, "ff_prod_axis: initial must be a canonical residue");
    if (outer == 0 || inner == 0) return MPYC_B200_OK;
    if (!d_out || (len && !d_in)) return fail(MPYC_B200_EINVAL, "ff_prod_axis: null buffer");
    if (bytes_overlap(d_in, ib, d_out, ob)) return fail(MPYC_B200_EINVAL, "ff_prod_axis: out overlaps the input");
    return launch_status(launch_prod_axis(f->fp, (const u64*)d_in, (u64*)d_out, outer, len, inner, (const u64*)initial,
                                          (cudaStream_t)stream),
                         "ff_prod_axis launch");
}

MPYC_API int mpyc_b200_ff_cumprod_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner,
                                       int include_initial, void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_cumprod_axis: field is null")) return rc;
    const size_t inc = include_initial ? 1 : 0;
    size_t ib = 0, ob = 0;
    if (len > SIZE_MAX - inc || !axis_bytes(f, outer, len, len + inc, inner, &ib, &ob))
        return fail(MPYC_B200_EINVAL, "ff_cumprod_axis: size overflow");
    if (outer == 0 || inner == 0 || len + inc == 0) return MPYC_B200_OK;
    if (!d_out || (len && !d_in)) return fail(MPYC_B200_EINVAL, "ff_cumprod_axis: null buffer");
    if (bytes_overlap(d_in, ib, d_out, ob)) return fail(MPYC_B200_EINVAL, "ff_cumprod_axis: out overlaps the input");
    return launch_status(launch_cumprod_axis(f->fp, (const u64*)d_in, (u64*)d_out, outer, len, inner, inc != 0, (cudaStream_t)stream),
                         "ff_cumprod_axis launch");
}

MPYC_API int mpyc_b200_ff_all_any_axis(const mpyc_b200_field* f, const void* d_in, size_t outer, size_t len, size_t inner, int any,
                                       void* d_out, void* stream) {
    if (int rc = prime_only(f, "ff_all_any_axis: field is null")) return rc;
    size_t ib = 0, ob = 0;
    if (!axis_bytes(f, outer, len, 1, inner, &ib, &ob)) return fail(MPYC_B200_EINVAL, "ff_all_any_axis: size overflow");
    if (outer == 0 || inner == 0) return MPYC_B200_OK;
    if (!d_out || (len && !d_in)) return fail(MPYC_B200_EINVAL, "ff_all_any_axis: null buffer");
    if (bytes_overlap(d_in, ib, d_out, ob)) return fail(MPYC_B200_EINVAL, "ff_all_any_axis: out overlaps the input");
    return launch_status(launch_all_any_axis(f->fp, (const u64*)d_in, (u64*)d_out, outer, len, inner, any != 0, (cudaStream_t)stream),
                         "ff_all_any_axis launch");
}

// ---------------------------------------------------------------------------------------
// K14: field matrix times public 64-bit integer matrix (matmul_int.cuh; prime fields)
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_ff_matmul_int(const mpyc_b200_field* f, const void* d_x, const void* d_w, int w_unsigned, int w_left,
                                     void* d_c, size_t r, size_t k, size_t c, void* stream) {
    if (int rc = prime_only(f, "ff_matmul_int: field is null")) return rc;
    const size_t E = (size_t)f->fp.L * sizeof(u64);
    size_t xe = 0, we = 0, xb = 0, wb = 0, cb = 0;
    size_t rk = 0, kc = 0;
    if (__builtin_mul_overflow(r, k, &rk) || __builtin_mul_overflow(k, c, &kc) || __builtin_mul_overflow(r, c, &cb))
        return fail(MPYC_B200_EINVAL, "ff_matmul_int: size overflow");
    xe = w_left ? kc : rk;
    we = w_left ? rk : kc;
    if (__builtin_mul_overflow(xe, E, &xb) || __builtin_mul_overflow(we, sizeof(u64), &wb) || __builtin_mul_overflow(cb, E, &cb) ||
        xb > (size_t)INT64_MAX || wb > (size_t)INT64_MAX || cb > (size_t)INT64_MAX)
        return fail(MPYC_B200_EINVAL, "ff_matmul_int: size overflow");
    if (r == 0 || c == 0) return MPYC_B200_OK;
    if (!d_c || (k && (!d_x || !d_w))) return fail(MPYC_B200_EINVAL, "ff_matmul_int: null buffer");
    const uintptr_t any = reinterpret_cast<uintptr_t>(d_c) | (k ? reinterpret_cast<uintptr_t>(d_x) | reinterpret_cast<uintptr_t>(d_w) : 0);
    if (any & 7u) return fail(MPYC_B200_EINVAL, "ff_matmul_int: buffers must be 8-byte aligned");
    if (bytes_overlap(d_c, cb, d_x, xb) || bytes_overlap(d_c, cb, d_w, wb))
        return fail(MPYC_B200_EINVAL, "ff_matmul_int: c overlaps an operand");
    return launch_status(launch_matmul_int(f->fp, (const u64*)d_x, (const u64*)d_w, w_unsigned != 0, w_left != 0, (u64*)d_c, r, k, c,
                                           (cudaStream_t)stream),
                         "ff_matmul_int launch");
}

// ---------------------------------------------------------------------------------------
// K15: GF(2^8) bit composition, broadcast arithmetic and stacked products (gf_local.cuh)
// ---------------------------------------------------------------------------------------

static int gf_only(const mpyc_b200_field* f, const char* what) {
    if (!f) return fail(MPYC_B200_EINVAL, what);
    if (f->kind != MPYC_B200_KIND_GF256) return fail(MPYC_B200_EUNSUPPORTED, "K15 kernels cover GF(2^8) only");
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_gf_bits_compose(const mpyc_b200_field* f, const void* d_bits, size_t n, size_t l, void* d_out, void* stream) {
    if (int rc = gf_only(f, "gf_bits_compose: field is null")) return rc;
    if (l == 0) return fail(MPYC_B200_EINVAL, "gf_bits_compose: l must be at least 1");
    size_t ib = 0;
    if (__builtin_mul_overflow(n, l, &ib) || ib > (size_t)INT64_MAX) return fail(MPYC_B200_EINVAL, "gf_bits_compose: size overflow");
    if (n == 0) return MPYC_B200_OK;
    if (!d_bits || !d_out) return fail(MPYC_B200_EINVAL, "gf_bits_compose: null buffer");
    if (bytes_overlap(d_bits, ib, d_out, n)) return fail(MPYC_B200_EINVAL, "gf_bits_compose: out overlaps the input");
    return launch_status(launch_gf_bits_compose(f->gf_poly, (const unsigned char*)d_bits, n, l, (unsigned char*)d_out,
                                                (cudaStream_t)stream),
                         "gf_bits_compose launch");
}

MPYC_API int mpyc_b200_gf_binop_view(const mpyc_b200_field* f, int op, const void* d_a, size_t a_len, const mpyc_b200_view* a,
                                     const void* d_b, size_t b_len, const mpyc_b200_view* b, void* d_out, void* stream) {
    if (int rc = gf_only(f, "gf_binop_view: field is null")) return rc;
    if (op < 0 || op > 2) return fail(MPYC_B200_EINVAL, "gf_binop_view: op must be ADD, SUB or MUL");
    const long long na = view_check(a, a_len, false), nb = view_check(b, b_len, false);
    if (na < 0 || nb < 0) return fail(MPYC_B200_EINVAL, "gf_binop_view: bad view (rank > 6, negative extent, index table or outside its buffer)");
    if (!same_extents(a, b)) return fail(MPYC_B200_EINVAL, "gf_binop_view: views of different extents");
    if (na == 0) return MPYC_B200_OK;
    if (!d_a || !d_b || !d_out) return fail(MPYC_B200_EINVAL, "gf_binop_view: null buffer");
    if (bytes_overlap(d_out, (size_t)na, d_a, a_len) || bytes_overlap(d_out, (size_t)na, d_b, b_len))
        return fail(MPYC_B200_EINVAL, "gf_binop_view: out overlaps an operand");
    BinopPlan p = {};
    p.rank = a->rank;
    p.aoff = a->offset, p.boff = b->offset;
    for (int k = 0; k < p.rank; k++) p.ext[k] = a->extent[k], p.astr[k] = a->stride[k], p.bstr[k] = b->stride[k];
    if (p.rank == 0) p.rank = 1, p.ext[0] = 1;
    return launch_status(launch_gf_binop_view(f->gf_poly, op, p, (const unsigned char*)d_a, (const unsigned char*)d_b,
                                              (unsigned char*)d_out, (cudaStream_t)stream),
                         "gf_binop_view launch");
}

MPYC_API int mpyc_b200_gf_matmul_batched(const mpyc_b200_field* f, const void* d_a, size_t a_batch_stride, const void* d_b,
                                         size_t b_batch_stride, void* d_c, size_t batch, size_t r, size_t k, size_t c, void* stream) {
    if (int rc = gf_only(f, "gf_matmul_batched: field is null")) return rc;
    size_t rk = 0, kc = 0, rc_ = 0, ab = 0, bb = 0, cb = 0;
    if (__builtin_mul_overflow(r, k, &rk) || __builtin_mul_overflow(k, c, &kc) || __builtin_mul_overflow(r, c, &rc_) ||
        __builtin_mul_overflow(rc_, batch, &cb) || cb > (size_t)INT64_MAX)
        return fail(MPYC_B200_EINVAL, "gf_matmul_batched: size overflow");
    if ((a_batch_stride != 0 && a_batch_stride != rk) || (b_batch_stride != 0 && b_batch_stride != kc))
        return fail(MPYC_B200_EINVAL, "gf_matmul_batched: a batch stride must be 0 or the matrix size");
    if (__builtin_mul_overflow(a_batch_stride ? batch : 1, rk, &ab) || __builtin_mul_overflow(b_batch_stride ? batch : 1, kc, &bb) ||
        ab > (size_t)INT64_MAX || bb > (size_t)INT64_MAX)
        return fail(MPYC_B200_EINVAL, "gf_matmul_batched: size overflow");
    if (cb == 0) return MPYC_B200_OK;
    if (!d_c || (k && (!d_a || !d_b))) return fail(MPYC_B200_EINVAL, "gf_matmul_batched: null buffer");
    if (bytes_overlap(d_c, cb, d_a, ab) || bytes_overlap(d_c, cb, d_b, bb))
        return fail(MPYC_B200_EINVAL, "gf_matmul_batched: c overlaps an operand");
    return launch_status(launch_gf_matmul_batched(f->gf_poly, (const unsigned char*)d_a, a_batch_stride, (const unsigned char*)d_b,
                                                  b_batch_stride, (unsigned char*)d_c, batch, r, k, c, (cudaStream_t)stream),
                         "gf_matmul_batched launch");
}

MPYC_API int mpyc_b200_ff_binop_rows(const mpyc_b200_field* f, int op, int reflected, const void* d_a, const void* d_b, void* d_out,
                                     size_t rows, size_t cols, void* stream) {
    if (int rc = prime_only(f, "ff_binop_rows: field is null")) return rc;
    if (op < 0 || op > 2) return fail(MPYC_B200_EINVAL, "ff_binop_rows: op must be ADD, SUB or MUL");
    if (rows && cols && (!d_a || !d_b || !d_out)) return fail(MPYC_B200_EINVAL, "ff_binop_rows: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::binop_rows(f->fp, op, reflected != 0, (const u64*)d_a, (const u64*)d_b, (u64*)d_out, rows, cols, st),
                             "ff_binop_rows launch");
    });
}

MPYC_API int mpyc_b200_ff_conv2d(const mpyc_b200_field* f, const void* d_x, const void* d_w, const void* d_b, void* d_y,
                                 int k, int r, int m, int n, int v, int s, void* stream) {
    if (int rc = prime_only(f, "ff_conv2d: field is null")) return rc;
    if (k < 0 || r < 1 || m < 1 || n < 1 || v < 1 || s < 1) return fail(MPYC_B200_EINVAL, "ff_conv2d: bad shape");
    if (s % 2 == 0) return fail(MPYC_B200_EUNSUPPORTED, "ff_conv2d: even filter sizes are not covered");
    // rows shorter than the filter: np.correlate(.., 'same') returns max(n, s) values and the demo's row assignment fails --
    // the engine does not compute where the reference raises
    if (n < s) return fail(MPYC_B200_EUNSUPPORTED, "ff_conv2d: image rows shorter than the filter");
    if ((size_t)r * s * s > FF_MAX_LAZY_TERMS) return fail(MPYC_B200_EUNSUPPORTED, "ff_conv2d: too many taps for one lazy sum");
    if ((size_t)r * s * s * f->fp.L * 8 > 200u * 1024u) return fail(MPYC_B200_EUNSUPPORTED, "ff_conv2d: filter does not fit shared memory");
    if (k == 0) return MPYC_B200_OK;
    if (!d_x || !d_w || !d_b || !d_y) return fail(MPYC_B200_EINVAL, "ff_conv2d: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int L = decltype(Lc)::value;
        return launch_status(Launch<L>::conv2d(f->fp, (const u64*)d_x, (const u64*)d_w, (const u64*)d_b, (u64*)d_y, k, r, m, n, v, s, st),
                             "ff_conv2d launch");
    });
}

// ---------------------------------------------------------------------------------------
// Shamir split
// ---------------------------------------------------------------------------------------

static int split_table(const mpyc_b200_field* cf, int t, int m, DevTable* tab) {
    mpyc_b200_field* f = const_cast<mpyc_b200_field*>(cf);
    int64_t key[2] = {t, m};
    return get_table(f, key_of("split", current_device(), key, 2, nullptr, 0), tab,
                     [&](std::vector<u64>& host, bool& full) { return build_split_table(f->fp, t, m, host, full); });
}

MPYC_API int mpyc_b200_shamir_split(const mpyc_b200_field* f, const void* d_secrets, const void* d_coeffs,
                                      size_t coeff_stride, void* d_shares, size_t share_stride, size_t n, int t, int m,
                                      void* stream) {
    if (!f) return fail(MPYC_B200_EINVAL, "shamir_split: field is null");
    if (m < 1 || t < 0 || t >= m) return fail(MPYC_B200_EINVAL, "shamir_split: need 0 <= t < m");
    if (n == 0) return MPYC_B200_OK;
    if (!d_secrets || !d_shares || (t > 0 && !d_coeffs)) return fail(MPYC_B200_EINVAL, "shamir_split: null buffer");
    if (share_stride < n || (t > 1 && coeff_stride < n)) return fail(MPYC_B200_EINVAL, "shamir_split: stride < n");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256) {
        if (m > 255) return fail(MPYC_B200_EUNSUPPORTED, "GF(2^8) has only 255 nonzero points");
        return launch_status(gf256_split(f->gf_poly, (const unsigned char*)d_secrets, (const unsigned char*)d_coeffs,
                                         coeff_stride, (unsigned char*)d_shares, share_stride, n, t, m, st),
                             "gf256 split");
    }
    DevTable tab;
    int rc = split_table(f, t, m, &tab);
    if (rc) return rc;
    if (tab.bytes > MAX_SMEM_TABLE) return fail(MPYC_B200_EUNSUPPORTED, "shamir_split: (m, t) table exceeds shared memory");
    const size_t L = f->fp.L;
    return with_limbs((int)L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        return launch_status(Launch<LL>::split(f->fp, tab.full, (const u64*)d_secrets, (const u64*)d_coeffs,
                                               coeff_stride * LL, (u64*)d_shares, share_stride * LL, n, t, m, tab.d,
                                               tab.bytes, st),
                             "shamir_split launch");
    });
}

static int split_generate_impl(const mpyc_b200_field* f, const void* d_secrets, void* d_shares, size_t share_stride,
                               void* const* d_share_rows, size_t n, int t, int m, const uint8_t key32[32], uint64_t nonce,
                               void* stream) {
    if (!f || !key32) return fail(MPYC_B200_EINVAL, "shamir_split_generate: null argument");
    if (m < 1 || t < 0 || t >= m) return fail(MPYC_B200_EINVAL, "shamir_split: need 0 <= t < m");
    REQUIRE_PRIME(f, "shamir_split_generate");
    if (t > 4) return fail(MPYC_B200_EUNSUPPORTED, "shamir_split_generate: t <= 4 (use explicit coefficients beyond)");
    if (d_share_rows && m > MPYC_MAX_SHARE_ROWS) return fail(MPYC_B200_EUNSUPPORTED, "shamir_split_generate_rows: at most 32 rows");
    if (n == 0) return MPYC_B200_OK;
    if (!d_secrets || (!d_share_rows && (!d_shares || share_stride < n))) return fail(MPYC_B200_EINVAL, "shamir_split_generate: bad buffers");
    DevTable tab;
    int rc = split_table(f, t, m, &tab);
    if (rc) return rc;
    if (tab.bytes > MAX_SMEM_TABLE) return fail(MPYC_B200_EUNSUPPORTED, "shamir_split: (m, t) table exceeds shared memory");
    ChaChaKey key;
    memcpy(key.k, key32, 32);
    key.nonce[0] = (u32)nonce;
    key.nonce[1] = (u32)(nonce >> 32) & 0x7FFFFFFFu;   // top bit separates the tail keystream
    cudaStream_t st = (cudaStream_t)stream;
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        ShareDst dst;
        if (d_share_rows) {
            dst.use_rows = 1;
            for (int i = 0; i < m; i++) {
                if (!d_share_rows[i]) return fail(MPYC_B200_EINVAL, "shamir_split_generate_rows: null row");
                dst.rows[i] = (u64*)d_share_rows[i];
            }
        } else {
            dst.base = (u64*)d_shares;
            dst.stride = share_stride * LL;
        }
        return launch_status(Launch<LL>::split_gen(f->fp, tab.full, key, (const u64*)d_secrets, dst, n, t, m, tab.d, tab.bytes, st),
                             "shamir_split_generate launch");
    });
}

MPYC_API int mpyc_b200_shamir_split_generate(const mpyc_b200_field* f, const void* d_secrets, void* d_shares,
                                             size_t share_stride, size_t n, int t, int m, const uint8_t key32[32],
                                             uint64_t nonce, void* stream) {
    return split_generate_impl(f, d_secrets, d_shares, share_stride, nullptr, n, t, m, key32, nonce, stream);
}

MPYC_API int mpyc_b200_shamir_split_generate_rows(const mpyc_b200_field* f, const void* d_secrets, void* const* d_share_rows,
                                                  size_t n, int t, int m, const uint8_t key32[32], uint64_t nonce,
                                                  void* stream) {
    if (!d_share_rows) return fail(MPYC_B200_EINVAL, "shamir_split_generate_rows: null row table");
    return split_generate_impl(f, d_secrets, nullptr, 0, d_share_rows, n, t, m, key32, nonce, stream);
}

// ---------------------------------------------------------------------------------------
// recombination
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_recombination_vector(const mpyc_b200_field* f, const int64_t* xs, int k, const int64_t* x_rs,
                                              int width, uint64_t* h_lambda) {
    if (!f || !xs || !x_rs || !h_lambda || k < 1 || width < 1) return fail(MPYC_B200_EINVAL, "recombination_vector: bad arguments");
    if (f->kind == MPYC_B200_KIND_GF256) {
        std::vector<unsigned char> lam((size_t)width * k);
        int rc = gf256_lambda(f->gf_poly, xs, k, x_rs, width, lam.data());
        if (rc) return fail(rc, "recombination: repeated x-coordinate");
        for (size_t i = 0; i < lam.size(); i++) h_lambda[i] = lam[i];
        return MPYC_B200_OK;
    }
    std::vector<u64> lam;
    int rc = compute_lambda(f->fp, xs, k, x_rs, width, lam);
    if (rc) return rc;
    memcpy(h_lambda, lam.data(), lam.size() * sizeof(u64));
    return MPYC_B200_OK;
}

static int recombine_table(const mpyc_b200_field* cf, const int64_t* xs, int k, const int64_t* x_rs, int width, DevTable* tab) {
    mpyc_b200_field* f = const_cast<mpyc_b200_field*>(cf);
    return get_table(f, key_of("rec", current_device(), xs, k, x_rs, width), tab, [&](std::vector<u64>& host, bool& full) {
        full = true;
        int rc = compute_lambda(f->fp, xs, k, x_rs, width, host);
        if (rc) return rc;
        // signed-magnitude form: |lambda| < 2^58 for every entry (e.g. x-coordinates 1..k at 0:
        // lambda_i = (-1)^(i-1) C(k,i)) -> 64-bit-constant kernel.  Fields of >= 2 limbs: always (k <= 32); 1-limb fields:
        // only when additionally every row's sum of |lambda| is <= 2^31, so that the per-element sum is < 2^(k+31) and the
        // cheap reductions apply (Fp::reduce_small_q32: one-limb-quotient Barrett / single-multiply fold) -- otherwise the
        // full product is as cheap there.
        if (k <= 32 && getenv("MPYC_B200_NO_SMALL_LAMBDA") == nullptr) {
            const int L = (int)f->fp.L;
            std::vector<u64> sm((size_t)width * k * 2);
            bool ok = true;
            bool q32 = getenv("MPYC_B200_NO_Q32") == nullptr;
            for (int r = 0; r < width && ok; r++) {
                unsigned __int128 row_sum = 0;
                for (int i = 0; i < k && ok; i++) {
                    const size_t e = (size_t)r * k + i;
                    const u64* lam = &host[e * L];
                    bool small_pos = lam[0] < (1ull << 58);
                    for (int l = 1; l < L; l++) small_pos = small_pos && lam[l] == 0;
                    if (small_pos) {
                        sm[2 * e] = lam[0];
                        sm[2 * e + 1] = 0;
                        row_sum += lam[0];
                        continue;
                    }
                    u64 neg[4];   // p - lambda
                    unsigned __int128 bw = 0;
                    for (int l = 0; l < L; l++) {
                        unsigned __int128 d = (unsigned __int128)f->fp.p[l] - lam[l] - (u64)bw;
                        neg[l] = (u64)d;
                        bw = (d >> 64) & 1;
                    }
                    bool small_neg = neg[0] < (1ull << 58);
                    for (int l = 1; l < L; l++) small_neg = small_neg && neg[l] == 0;
                    if (!small_neg) ok = false;
                    sm[2 * e] = neg[0];
                    sm[2 * e + 1] = 1;
                    row_sum += neg[0];
                }
                if (row_sum > ((unsigned __int128)1 << 31)) q32 = false;
            }
            if (ok && (L >= 2 || q32)) {
                host.swap(sm);
                full = false;
                tl_table_aux = q32 ? 1u : 0u;
                return MPYC_B200_OK;
            }
        }
        to_table_form(f->fp, host);
        return MPYC_B200_OK;
    });
}

MPYC_API int mpyc_b200_shamir_recombine(const mpyc_b200_field* f, const void* const* d_share_rows, const int64_t* xs,
                                          int k, const int64_t* x_rs, int width, void* d_out, size_t out_stride, size_t n,
                                          void* stream) {
    if (!f || !d_share_rows || !xs || !x_rs) return fail(MPYC_B200_EINVAL, "shamir_recombine: null argument");
    if (k < 1 || width < 1) return fail(MPYC_B200_EINVAL, "shamir_recombine: need k >= 1 and width >= 1");
    if (k > MPYC_B200_MAX_POINTS) return fail(MPYC_B200_EUNSUPPORTED, "shamir_recombine: more than MPYC_B200_MAX_POINTS shares");
    if (n == 0) return MPYC_B200_OK;
    if (!d_out || (width > 1 && out_stride < n)) return fail(MPYC_B200_EINVAL, "shamir_recombine: bad output");
    for (int i = 0; i < k; i++)
        if (!d_share_rows[i]) return fail(MPYC_B200_EINVAL, "shamir_recombine: null share row");
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256) {
        std::vector<unsigned char> lam((size_t)width * k);
        int rc = gf256_lambda(f->gf_poly, xs, k, x_rs, width, lam.data());
        if (rc) return fail(rc, "recombination: repeated x-coordinate");
        return launch_status(gf256_recombine(f->gf_poly, (const unsigned char* const*)d_share_rows, k, width, lam.data(),
                                             (unsigned char*)d_out, out_stride, n, st), "gf256 recombine");
    }
    DevTable tab;
    int rc = recombine_table(f, xs, k, x_rs, width, &tab);
    if (rc) return rc;
    if (tab.bytes > MAX_SMEM_TABLE) return fail(MPYC_B200_EUNSUPPORTED, "shamir_recombine: table exceeds shared memory");
    RowPtrs rows;
    memset(&rows, 0, sizeof rows);
    for (int i = 0; i < k; i++) rows.p[i] = (const u64*)d_share_rows[i];
    FieldParams fq = f->fp;
    fq.q32 = (!tab.full && tab.aux) ? 1u : 0u;       // small-lambda sums below 2^(k+31): cheap per-element reduction
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        return launch_status(Launch<LL>::recombine(fq, !tab.full, rows, k, width, tab.d, tab.bytes, (u64*)d_out, out_stride * LL, n, st),
                             "shamir_recombine launch");
    });
}

// ---------------------------------------------------------------------------------------
// PRSS linear step
// ---------------------------------------------------------------------------------------

namespace {

// per-call PRSS constants on the device: [coef_S (nsub) | weight_j (d)] in table form (prime fields)
struct PrssTable {
    u64* d_tab = nullptr;
    u32 bytes = 0;
    std::vector<unsigned char> gf;     // GF(2^8): passed to the kernel by value
    bool small = false;                // [(|num_S|, sign_S) x nsub | w_j x d | D^-1 (L limbs)]: see prss_small_table
    bool simple = false;               // small, d == 1 and weight 1: the plain pseudorandom share
    bool owned = false;                // false: d_tab lives in the field handle's table cache
    cudaStream_t st = nullptr;
    ~PrssTable() {
        if (d_tab && owned) cudaFreeAsync(d_tab, st);
    }
};

// Small-integer form of the subset coefficients.  f_S(i) = prod_{j not in S} (i - j) / (-(j + 1)) (thresha.py:135-141) is a
// ratio of small integers, so for D = m! the products f_S(i) D are small signed integers: if some D = k!, k <= 20, makes
// every coef_S D mod p representable as +-v with v < 2^57 (and the weights are plain integers < 2^58, as (i+1)^j is),
// the kernel multiplies by 64-bit constants into one (L+1)-limb sum -- the K3s trick -- and multiplies the reduced
// sum by D^-1 once per element instead of doing nsub full products.  Same residues, bit for bit.
bool prss_small_table(const FieldParams& fp, int nsub, int d, const uint64_t* h_coef, const uint64_t* h_weights,
                      std::vector<u64>& host) {
    if (nsub > 64 || d > 32 || getenv("MPYC_B200_PRSS_FULL") != nullptr) return false;
    const int L = (int)fp.L;
    for (int j = 0; j < d; j++) {
        if (h_weights[(size_t)j * L] >= (1ull << 58)) return false;
        for (int l = 1; l < L; l++)
            if (h_weights[(size_t)j * L + l]) return false;
    }
    bool found = false;
    with_field(fp, [&](auto Lc, auto Kc) {
        constexpr int LL = decltype(Lc)::value;
        constexpr int K = decltype(Kc)::value;
        typedef Fp<LL, K> F;
        constexpr int N = 2 * LL;
        u64 D = 1;
        for (int k = 1; k <= 20 && !found; k++) {
            D *= (u64)k;
            u32 Dm[N];
            h_from_int<LL, K>(Dm, (int64_t)D, fp);
            if (is_zero_n<N>(Dm)) continue;                     // p divides k! (tiny fields)
            std::vector<u64> tab((size_t)2 * nsub + d + LL);
            bool ok = true;
            for (int S = 0; S < nsub && ok; S++) {
                u32 c[N], r[N], neg[N];
                for (int l = 0; l < LL; l++) set64(c, l, h_coef[(size_t)S * LL + l]);
                F::mul(r, c, Dm, fp);
                F::neg(neg, r, fp);
                auto small = [&](const u32* v) {
                    for (int l = 1; l < LL; l++)
                        if (get64(v, l)) return false;
                    return get64(v, 0) < (1ull << 57);
                };
                if (small(r)) {
                    tab[2 * S] = get64(r, 0);
                    tab[2 * S + 1] = 0;
                } else if (small(neg)) {
                    tab[2 * S] = get64(neg, 0);
                    tab[2 * S + 1] = 1;
                } else {
                    ok = false;
                }
            }
            if (!ok) continue;
            u32 inv[N];
            if (!h_inv<LL, K>(inv, Dm, fp)) continue;
            for (int j = 0; j < d; j++) tab[(size_t)2 * nsub + j] = h_weights[(size_t)j * LL];
            for (int l = 0; l < LL; l++) tab[(size_t)2 * nsub + d + l] = get64(inv, l);
            host.swap(tab);
            found = true;
        }
        return MPYC_B200_OK;
    });
    return found;
}

int prss_prepare(const mpyc_b200_field* f, int nsub, int d, int chunk_bytes, int bound_bits, const uint64_t* h_coef,
                 const uint64_t* h_weights, cudaStream_t st, PrssTable& tab) {
    if (f->kind == MPYC_B200_KIND_GF256) {
        if (chunk_bytes != 1 || bound_bits < 0 || bound_bits > 8) return fail(MPYC_B200_EINVAL, "prss: GF(2^8) PRF chunks are one byte, bound 2^b <= 256");
        tab.gf.resize((size_t)nsub + d);
        for (int i = 0; i < nsub; i++) tab.gf[i] = (unsigned char)h_coef[i];
        for (int j = 0; j < d; j++) tab.gf[nsub + j] = (unsigned char)h_weights[j];
        return MPYC_B200_OK;
    }
    if (chunk_bytes > 8 * (int)f->fp.L + 32) return fail(MPYC_B200_EINVAL, "prss: chunk too wide for this field");
    if (bound_bits < 0 || bound_bits >= (int)f->fp.k) return fail(MPYC_B200_EINVAL, "prss: need 2^bound_bits <= p");
    if (bound_bits > 0 && chunk_bytes != (bound_bits + 7) / 8) return fail(MPYC_B200_EINVAL, "prss: chunk_bytes != ceil(bound_bits/8)");
    if ((unsigned)nsub > FF_MAX_LAZY_TERMS || (unsigned)d > FF_MAX_LAZY_TERMS) return fail(MPYC_B200_EUNSUPPORTED, "prss: too many terms");
    const size_t L = f->fp.L;
    auto build = [&](std::vector<u64>& host, bool& full) {
        const bool small = prss_small_table(f->fp, nsub, d, h_coef, h_weights, host);
        if (!small) {
            host.resize(((size_t)nsub + d) * L);
            memcpy(host.data(), h_coef, (size_t)nsub * L * sizeof(u64));
            memcpy(host.data() + (size_t)nsub * L, h_weights, (size_t)d * L * sizeof(u64));
            to_table_form(f->fp, host);
        }
        if (host.size() * sizeof(u64) > MAX_SMEM_TABLE) return fail(MPYC_B200_EUNSUPPORTED, "prss: coefficient table exceeds shared memory");
        full = !small;
        return MPYC_B200_OK;
    };
    // The constants depend only on (m, t, party): a handful of distinct tables per computation.  They are kept in the
    // field handle's cache, keyed by their bytes, so that a call costs no allocation, upload or synchronisation;
    // beyond 512 cached tables (a caller inventing coefficients per call) the table is uploaded per call instead.
    mpyc_b200_field* fm = const_cast<mpyc_b200_field*>(f);
    bool cache_ok;
    {
        std::lock_guard<std::mutex> g(fm->mu);
        cache_ok = fm->tables.size() < 512;
    }
    bool full = false;
    if (cache_ok) {
        std::string key = "prss:" + std::to_string(current_device()) + ":" + std::to_string(nsub) + ":" + std::to_string(d) + ":" +
                          (getenv("MPYC_B200_PRSS_FULL") ? "F" : "S") + ":";
        key.append((const char*)h_coef, (size_t)nsub * L * sizeof(u64));
        key.append((const char*)h_weights, (size_t)d * L * sizeof(u64));
        DevTable t;
        int rc = get_table(fm, key, &t, build);
        if (rc) return rc;
        tab.d_tab = t.d;
        tab.bytes = t.bytes;
        full = t.full;
    } else {
        std::vector<u64> host;
        int rc = build(host, full);
        if (rc) return rc;
        if (host.size() % 2) host.push_back(0);
        tab.bytes = (u32)(host.size() * sizeof(u64));
        tab.st = st;
        tab.owned = true;
        CU(cudaMallocAsync(&tab.d_tab, tab.bytes, st));
        cudaError_t e = cudaMemcpyAsync(tab.d_tab, host.data(), tab.bytes, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // host vector goes out of scope
        if (e != cudaSuccess) return cuda_fail(e, "prss table upload");
    }
    tab.small = !full;
    // d == 1 with weight 1 (the plain pseudorandom share) has its own compile-time kernel variant
    // (MPYC_B200_PRSS_NO_SIMPLE=1 selects the general small form: parity tests compare both)
    tab.simple = tab.small && d == 1 && h_weights[0] == 1 && getenv("MPYC_B200_PRSS_NO_SIMPLE") == nullptr;
    return MPYC_B200_OK;
}

int prss_launch(const mpyc_b200_field* f, const PrssTable& tab, const uint8_t* d_prf_bytes, size_t subset_stride_bytes, int nsub,
                int d, int chunk_bytes, int bound_bits, void* d_out, size_t n, cudaStream_t st) {
    if (f->kind == MPYC_B200_KIND_GF256)
        return launch_status(gf256_prss(f->gf_poly, d_prf_bytes, subset_stride_bytes, nsub, d, tab.gf.data(),
                                        bound_bits > 0 && bound_bits < 8 ? (1u << bound_bits) - 1u : 0xFFu, (unsigned char*)d_out, n, st), "gf256 prss");
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        return launch_status(Launch<LL>::prss(f->fp, tab.small, tab.simple, d_prf_bytes, subset_stride_bytes, nsub, d, chunk_bytes, bound_bits,
                                              tab.d_tab, tab.bytes, (u64*)d_out, n, st), "prss_combine launch");
    });
}

}   // namespace

// Host-only view of prss_small_table (no GPU involved): which scale k! makes the subset coefficients small integers.
MPYC_API int mpyc_b200_prss_small_form(const mpyc_b200_field* f, int nsub, int d, const uint64_t* h_coef,
                                         const uint64_t* h_weights, int64_t* h_num, uint64_t* h_scale_inv) {
    if (!f || !h_coef || !h_weights || !h_num || nsub < 1 || d < 1) return fail(MPYC_B200_EINVAL, "prss_small_form: bad arguments");
    REQUIRE_PRIME(f, "prss_small_form");
    std::vector<u64> tab;
    if (!prss_small_table(f->fp, nsub, d, h_coef, h_weights, tab)) return fail(MPYC_B200_EUNSUPPORTED, "prss_small_form: no small-integer form");
    for (int S = 0; S < nsub; S++) h_num[S] = tab[2 * S + 1] ? -(int64_t)tab[2 * S] : (int64_t)tab[2 * S];
    if (h_scale_inv)
        for (size_t l = 0; l < f->fp.L; l++) h_scale_inv[l] = tab[(size_t)2 * nsub + d + l];
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_prss_combine(const mpyc_b200_field* f, const uint8_t* d_prf_bytes, size_t subset_stride_bytes, int nsub,
                                      int d, int chunk_bytes, int bound_bits, const uint64_t* h_coef,
                                      const uint64_t* h_weights, void* d_out, size_t n, void* stream) {
    if (!f || !h_coef || !h_weights || nsub < 1 || d < 1 || chunk_bytes < 1) return fail(MPYC_B200_EINVAL, "prss_combine: bad arguments");
    if (n == 0) return MPYC_B200_OK;
    if (!d_prf_bytes || !d_out) return fail(MPYC_B200_EINVAL, "prss_combine: null buffer");
    cudaStream_t st = (cudaStream_t)stream;
    PrssTable tab;
    int rc = prss_prepare(f, nsub, d, chunk_bytes, bound_bits, h_coef, h_weights, st, tab);
    if (rc) return rc;
    return prss_launch(f, tab, d_prf_bytes, subset_stride_bytes, nsub, d, chunk_bytes, bound_bits, d_out, n, st);
}

namespace {

// description of a general PRF bound for prf_reduce.cuh
struct BoundSpec {
    FieldParams fb;        // Barrett constants (not used for powers of two)
    int pow2_bits = 0;     // > 0: bound = 2^pow2_bits
    int LB = 1;            // 64-bit limbs of a reduced value
};

// h_bound: nlimbs little-endian limbs of the bound (leading zero limbs allowed), 3 <= bound <= 2^256 (2 = 2^1 too)
int bound_spec(const uint64_t* h_bound, int nlimbs, BoundSpec& b) {
    if (!h_bound || nlimbs < 1 || nlimbs > 5) return fail(MPYC_B200_EINVAL, "prf bound: 1..5 limbs");
    int nz = nlimbs;
    while (nz > 0 && h_bound[nz - 1] == 0) nz--;
    if (nz == 0) return fail(MPYC_B200_EINVAL, "prf bound: zero");
    int pop = 0;
    for (int i = 0; i < nz; i++) pop += __builtin_popcountll(h_bound[i]);
    const int bits = 64 * (nz - 1) + 64 - __builtin_clzll(h_bound[nz - 1]);
    if (pop == 1) {
        b.pow2_bits = bits - 1;
        if (b.pow2_bits < 1) return fail(MPYC_B200_EINVAL, "prf bound: must be >= 2");
        if (b.pow2_bits > 256) return fail(MPYC_B200_EUNSUPPORTED, "prf bound wider than 256 bits");
        b.LB = std::max(1, (b.pow2_bits + 63) / 64);
        memset(&b.fb, 0, sizeof b.fb);
        return MPYC_B200_OK;
    }
    if (nz > 4) return fail(MPYC_B200_EUNSUPPORTED, "prf bound wider than 256 bits");
    if (nz == 1 && h_bound[0] < 3) return fail(MPYC_B200_EINVAL, "prf bound: must be >= 2");
    b.pow2_bits = 0;
    b.LB = nz;
    bound_params_init(h_bound, nz, &b.fb);
    return MPYC_B200_OK;
}

int prf_reduce_launch(const BoundSpec& b, unsigned gf_poly, const uint8_t* d_bytes, size_t subset_stride, int nsub, size_t count,
                      int chunk_bytes, void* d_values, size_t value_stride, cudaStream_t st) {
    if (chunk_bytes < 1 || chunk_bytes > 8 * (b.LB + 2)) return fail(MPYC_B200_EINVAL, "prf_reduce: chunk too wide for this bound");
    if (!gf_poly && (((uintptr_t)d_values | value_stride) & 7u)) return fail(MPYC_B200_EINVAL, "prf_reduce: values must be 8-byte aligned");
    const size_t total = (size_t)nsub * count;
    return with_limbs(b.LB, [&](auto Lc) {
        constexpr int LB = decltype(Lc)::value;
        if (total == 0) return (int)MPYC_B200_OK;
        const int grid = mpyc_grid_size((const void*)k_prf_reduce<LB>, total, 0);
        if (grid <= 0) return fail(MPYC_B200_ECUDA, "prf_reduce: no device");
        k_prf_reduce<LB><<<grid, MPYC_THREADS, 0, st>>>(b.fb, b.pow2_bits, (const unsigned char*)d_bytes, subset_stride, nsub, count, chunk_bytes,
                                                        (unsigned char*)d_values, value_stride, gf_poly);
        g_mpyc_launches.fetch_add(1);
        return launch_status(cudaGetLastError(), "prf_reduce launch");
    });
}

}   // namespace

MPYC_API int mpyc_b200_prf_reduce(const mpyc_b200_field* f, const uint8_t* d_prf_bytes, size_t subset_stride_bytes, int nsub,
                                    size_t count, int chunk_bytes, const uint64_t* h_bound, int bound_nlimbs, void* d_values,
                                    size_t value_stride_bytes, int* value_bytes, void* stream) {
    if (nsub < 1 || chunk_bytes < 1) return fail(MPYC_B200_EINVAL, "prf_reduce: bad arguments");
    BoundSpec b;
    int rc = bound_spec(h_bound, bound_nlimbs, b);
    if (rc) return rc;
    const bool gf = f && f->kind == MPYC_B200_KIND_GF256;
    if (value_bytes) *value_bytes = gf ? 1 : 8 * b.LB;
    if (count == 0) return MPYC_B200_OK;
    if (!d_prf_bytes || !d_values) return fail(MPYC_B200_EINVAL, "prf_reduce: null buffer");
    return prf_reduce_launch(b, gf ? f->gf_poly : 0u, d_prf_bytes, subset_stride_bytes, nsub, count, chunk_bytes, d_values,
                             value_stride_bytes, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------
// utilities
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_fill_random(const mpyc_b200_field* f, void* d_out, size_t n, uint64_t seed, uint64_t stream_id,
                                     void* stream) {
    if (!f || (n && !d_out)) return fail(MPYC_B200_EINVAL, "fill_random: bad arguments");
    const u64 base = seed + (stream_id << 56);
    cudaStream_t st = (cudaStream_t)stream;
    if (f->kind == MPYC_B200_KIND_GF256)
        return launch_status(gf256_fill(base, (unsigned char*)d_out, n, st), "gf256 fill");
    return with_limbs((int)f->fp.L, [&](auto Lc) {
        constexpr int LL = decltype(Lc)::value;
        return launch_status(Launch<LL>::fill_random(f->fp, (u64*)d_out, n, base, st), "fill_random launch");
    });
}

MPYC_API int mpyc_b200_count_mismatch(const mpyc_b200_field* f, const void* d_a, const void* d_b, size_t n,
                                        uint64_t* d_count, void* stream) {
    if (!f || !d_count || (n && (!d_a || !d_b))) return fail(MPYC_B200_EINVAL, "count_mismatch: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    CU(cudaMemsetAsync(d_count, 0, sizeof(uint64_t), st));
    if (n == 0) return MPYC_B200_OK;
    if (f->kind == MPYC_B200_KIND_GF256)
        return launch_status(gf256_mismatch((const unsigned char*)d_a, (const unsigned char*)d_b, n, (unsigned long long*)d_count, st), "gf256 mismatch");
    int grid = mpyc_grid_size((const void*)k_count_mismatch, n, 0);
    if (grid <= 0) return fail(MPYC_B200_ECUDA, "count_mismatch: no device");
    k_count_mismatch<<<grid, MPYC_THREADS, 0, st>>>((const u64*)d_a, (const u64*)d_b, n, (int)f->fp.L, (unsigned long long*)d_count);
    g_mpyc_launches.fetch_add(1);
    return launch_status(cudaGetLastError(), "count_mismatch launch");
}

// ---------------------------------------------------------------------------------------
// host-buffer pipelines: H2D copy, kernel and D2H copy of successive chunks overlap on
// three streams; device staging buffers are kept per device and grown on demand.
// ---------------------------------------------------------------------------------------

namespace {

constexpr int kSlots = 3;

struct Workspace {
    int device = -1;
    cudaStream_t streams[kSlots] = {nullptr, nullptr, nullptr};
    void* d_in[kSlots] = {nullptr, nullptr, nullptr};
    void* d_out[kSlots] = {nullptr, nullptr, nullptr};
    void* d_tmp[kSlots] = {nullptr, nullptr, nullptr};   // intermediate values (PRSS with a general PRF bound)
    size_t in_cap = 0, out_cap = 0, tmp_cap = 0;
    std::mutex mu;
};

// Two independent workspaces (streams + staging buffers + lock) per device: set 0 serves the split / elementwise / PRSS
// entry points, set 1 mpyc_b200_shamir_recombine_host.  A caller that pipelines batches -- split of batch j+1 from one
// thread while batch j is recombined from another -- keeps both PCIe directions busy at once: the split is
// D2H-heavy (m rows out for 1 + t in), the recombination H2D-heavy (k rows in for one out).
Workspace g_ws[16][2];
std::mutex g_ws_mu;

// Restores the calling thread's current CUDA device when it goes out of scope: the host-buffer entry points select
// `device` for their copies and launches and must not leave a multi-GPU caller (one torch process driving several
// GPUs, or rank r on cuda:r calling with the default device 0) on another device than it was on.
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() {
        if (cudaGetDevice(&prev) != cudaSuccess) {
            cudaGetLastError();
            prev = -1;
        }
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// creates the per-device workspace (streams) on first use; the caller then locks w->mu and calls reserve().
// Callers hold a DeviceGuard: the current device is switched here and restored when the entry point returns.
int acquire_workspace(int device, Workspace** out, int set = 0) {
    if (device < 0 || device >= 16) return fail(MPYC_B200_EINVAL, "device ordinal out of range");
    CU(cudaSetDevice(device));
    Workspace& w = g_ws[device][set];
    {
        std::lock_guard<std::mutex> g(g_ws_mu);
        if (w.device < 0) {
            for (int s = 0; s < kSlots; s++) CU(cudaStreamCreateWithFlags(&w.streams[s], cudaStreamNonBlocking));
            w.device = device;
        }
    }
    *out = &w;
    return MPYC_B200_OK;
}

// grow the staging buffers (call with w.mu held)
int reserve(Workspace& w, size_t in_bytes, size_t out_bytes) {
    if (in_bytes > w.in_cap) {
        for (int s = 0; s < kSlots; s++) {
            if (w.d_in[s]) cudaFree(w.d_in[s]);
            w.d_in[s] = nullptr;
        }
        w.in_cap = 0;
        for (int s = 0; s < kSlots; s++) CU(cudaMalloc(&w.d_in[s], in_bytes));
        w.in_cap = in_bytes;
    }
    if (out_bytes > w.out_cap) {
        for (int s = 0; s < kSlots; s++) {
            if (w.d_out[s]) cudaFree(w.d_out[s]);
            w.d_out[s] = nullptr;
        }
        w.out_cap = 0;
        for (int s = 0; s < kSlots; s++) CU(cudaMalloc(&w.d_out[s], out_bytes));
        w.out_cap = out_bytes;
    }
    return MPYC_B200_OK;
}

int reserve_tmp(Workspace& w, size_t bytes) {
    if (bytes <= w.tmp_cap) return MPYC_B200_OK;
    for (int s = 0; s < kSlots; s++) {
        if (w.d_tmp[s]) cudaFree(w.d_tmp[s]);
        w.d_tmp[s] = nullptr;
    }
    w.tmp_cap = 0;
    for (int s = 0; s < kSlots; s++) CU(cudaMalloc(&w.d_tmp[s], bytes));
    w.tmp_cap = bytes;
    return MPYC_B200_OK;
}

size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// elements per pipeline chunk, a multiple of 16: about a sixteenth of the call's traffic, at least 32 MiB and at most
// 256 MiB per chunk: many small 2-D copies in both directions leave PCIe below what two large concurrent copies
// reach.  MPYC_B200_CHUNK_MB overrides (tuning).
size_t chunk_elems(size_t n, size_t bytes_per_elem_total) {
    static const size_t forced = [] {
        const char* e = getenv("MPYC_B200_CHUNK_MB");
        const long mb = e ? atol(e) : 0;
        return (size_t)(mb >= 1 && mb <= 1024 ? mb : 0) << 20;
    }();
    const size_t per = std::max<size_t>(bytes_per_elem_total, 1);
    size_t chunk_bytes = forced;
    if (!chunk_bytes) chunk_bytes = std::min<size_t>(std::max<size_t>(n * per / 16, (size_t)32 << 20), (size_t)256 << 20);
    size_t c = chunk_bytes / per;
    c = std::max<size_t>(c / 16 * 16, 16);
    return std::min(c, round_up(n, 16));
}

}   // namespace

// one pipeline chunk of a split with explicit coefficients: H2D of the t+1 input rows, K2, D2H of the m share rows,
// all on slot `s` of workspace `w` (ch = chunk capacity in elements, eb = bytes per element)
static int split_chunk(const mpyc_b200_field* f, Workspace* w, int s, size_t ch, size_t eb, const void* h_secrets,
                       const void* h_coeffs, size_t coeff_stride, void* h_shares, size_t share_stride, size_t off, size_t cn,
                       int t, int m) {
    cudaStream_t st = w->streams[s];
    char* din = (char*)w->d_in[s];
    char* dout = (char*)w->d_out[s];
    CU(cudaMemcpyAsync(din, (const char*)h_secrets + off * eb, cn * eb, cudaMemcpyHostToDevice, st));
    if (t > 0)
        CU(cudaMemcpy2DAsync(din + ch * eb, ch * eb, (const char*)h_coeffs + off * eb, coeff_stride * eb, cn * eb, t,
                             cudaMemcpyHostToDevice, st));
    int rc = mpyc_b200_shamir_split(f, din, din + ch * eb, ch, dout, ch, cn, t, m, st);
    if (rc) return rc;
    CU(cudaMemcpy2DAsync((char*)h_shares + off * eb, share_stride * eb, dout, ch * eb, cn * eb, m, cudaMemcpyDeviceToHost, st));
    return MPYC_B200_OK;
}

// one pipeline chunk of a recombination: H2D of the k share rows, K3, D2H of the `width` result rows
static int recombine_chunk(const mpyc_b200_field* f, Workspace* w, int s, size_t ch, size_t eb, const void* const* h_share_rows,
                           const int64_t* xs, int k, const int64_t* x_rs, int width, void* h_out, size_t out_stride, size_t off,
                           size_t cn) {
    cudaStream_t st = w->streams[s];
    char* din = (char*)w->d_in[s];
    char* dout = (char*)w->d_out[s];
    const void* rows[MPYC_B200_MAX_POINTS];
    for (int i = 0; i < k; i++) {
        CU(cudaMemcpyAsync(din + (size_t)i * ch * eb, (const char*)h_share_rows[i] + off * eb, cn * eb, cudaMemcpyHostToDevice, st));
        rows[i] = din + (size_t)i * ch * eb;
    }
    int rc = mpyc_b200_shamir_recombine(f, rows, xs, k, x_rs, width, dout, ch, cn, st);
    if (rc) return rc;
    CU(cudaMemcpy2DAsync((char*)h_out + off * eb, out_stride * eb, dout, ch * eb, cn * eb, width, cudaMemcpyDeviceToHost, st));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_shamir_split_host(const mpyc_b200_field* f, const void* h_secrets, const void* h_coeffs,
                                           size_t coeff_stride, void* h_shares, size_t share_stride, size_t n, int t, int m,
                                           int device) {
    if (!f) return fail(MPYC_B200_EINVAL, "field is null");
    if (m < 1 || t < 0 || t >= m) return fail(MPYC_B200_EINVAL, "shamir_split: need 0 <= t < m");
    if (n == 0) return MPYC_B200_OK;
    if (!h_secrets || !h_shares || (t > 0 && !h_coeffs)) return fail(MPYC_B200_EINVAL, "shamir_split_host: null buffer");
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    const size_t ch = chunk_elems(n, eb * (size_t)(t + 1 + m));
    DeviceGuard guard;
    Workspace* w;
    int rc = acquire_workspace(device, &w);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(w->mu);
    rc = reserve(*w, ch * eb * (size_t)(t + 1), ch * eb * (size_t)m);
    if (rc) return rc;
    size_t c = 0;
    for (size_t off = 0; off < n; off += ch, c++) {
        rc = split_chunk(f, w, (int)(c % kSlots), ch, eb, h_secrets, h_coeffs, coeff_stride, h_shares, share_stride, off,
                         std::min(ch, n - off), t, m);
        if (rc) return rc;
    }
    for (int s = 0; s < kSlots && (size_t)s < c; s++) CU(cudaStreamSynchronize(w->streams[s]));   // only the slots this call used
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_shamir_split_generate_host(const mpyc_b200_field* f, const void* h_secrets, void* h_shares,
                                                    size_t share_stride, size_t n, int t, int m, const uint8_t key32[32],
                                                    uint64_t nonce, int device) {
    if (!f || !key32) return fail(MPYC_B200_EINVAL, "shamir_split_generate_host: null argument");
    if (m < 1 || t < 0 || t >= m) return fail(MPYC_B200_EINVAL, "shamir_split: need 0 <= t < m");
    if (n == 0) return MPYC_B200_OK;
    if (!h_secrets || !h_shares || share_stride < n) return fail(MPYC_B200_EINVAL, "shamir_split_generate_host: bad buffers");
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    const size_t ch = chunk_elems(n, eb * (size_t)(1 + m));
    DeviceGuard guard;
    Workspace* w;
    int rc = acquire_workspace(device, &w);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(w->mu);
    rc = reserve(*w, ch * eb, ch * eb * (size_t)m);
    if (rc) return rc;
    size_t c = 0;
    for (size_t off = 0; off < n; off += ch, c++) {
        const int s = (int)(c % kSlots);
        const size_t cn = std::min(ch, n - off);
        cudaStream_t st = w->streams[s];
        char* din = (char*)w->d_in[s];
        char* dout = (char*)w->d_out[s];
        CU(cudaMemcpyAsync(din, (const char*)h_secrets + off * eb, cn * eb, cudaMemcpyHostToDevice, st));
        // every chunk draws from its own keystream: the kernel's block counters restart at 0 per launch
        rc = mpyc_b200_shamir_split_generate(f, din, dout, ch, cn, t, m, key32, nonce + c, st);
        if (rc) return rc;
        CU(cudaMemcpy2DAsync((char*)h_shares + off * eb, share_stride * eb, dout, ch * eb, cn * eb, m,
                             cudaMemcpyDeviceToHost, st));
    }
    for (int s = 0; s < kSlots && (size_t)s < c; s++) CU(cudaStreamSynchronize(w->streams[s]));   // only the slots this call used
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_shamir_recombine_host(const mpyc_b200_field* f, const void* const* h_share_rows, const int64_t* xs,
                                               int k, const int64_t* x_rs, int width, void* h_out, size_t out_stride,
                                               size_t n, int device) {
    if (!f || !h_share_rows || !xs || !x_rs) return fail(MPYC_B200_EINVAL, "shamir_recombine_host: null argument");
    if (k < 1 || width < 1) return fail(MPYC_B200_EINVAL, "shamir_recombine_host: bad k/width");
    if (k > MPYC_B200_MAX_POINTS) return fail(MPYC_B200_EUNSUPPORTED, "shamir_recombine_host: more than MPYC_B200_MAX_POINTS shares");
    if (n == 0) return MPYC_B200_OK;
    if (!h_out) return fail(MPYC_B200_EINVAL, "shamir_recombine_host: null output");
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    const size_t ch = chunk_elems(n, eb * (size_t)(k + width));
    DeviceGuard guard;
    Workspace* w;
    int rc = acquire_workspace(device, &w, 1);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(w->mu);
    rc = reserve(*w, ch * eb * (size_t)k, ch * eb * (size_t)width);
    if (rc) return rc;
    size_t c = 0;
    for (size_t off = 0; off < n; off += ch, c++) {
        rc = recombine_chunk(f, w, (int)(c % kSlots), ch, eb, h_share_rows, xs, k, x_rs, width, h_out, out_stride, off,
                             std::min(ch, n - off));
        if (rc) return rc;
    }
    for (int s = 0; s < kSlots && (size_t)s < c; s++) CU(cudaStreamSynchronize(w->streams[s]));   // only the slots this call used
    return MPYC_B200_OK;
}

// A party's steady state in a stream of resharing rounds (runtime.py:660-680): while it recombines the 2t+1 rows it
// received for batch j (H2D-heavy: k rows in, one out) it already deals its shares of batch j+1 (D2H-heavy: t+1 rows in,
// m out).  This entry point runs both jobs from ONE host thread with their pipeline chunks issued alternately on the
// two workspaces' streams, so that both PCIe directions carry traffic all the time.  Either job may be empty
// (n_split == 0 / n_rec == 0); the two jobs are independent (different buffers).
MPYC_API int mpyc_b200_shamir_reshare_step_host(const mpyc_b200_field* f, const void* h_secrets, const void* h_coeffs,
                                                  size_t coeff_stride, void* h_shares, size_t share_stride, size_t n_split, int t,
                                                  int m, const void* const* h_share_rows, const int64_t* xs, int k,
                                                  const int64_t* x_rs, int width, void* h_out, size_t out_stride, size_t n_rec,
                                                  int device) {
    if (!f) return fail(MPYC_B200_EINVAL, "field is null");
    if (n_split) {
        if (m < 1 || t < 0 || t >= m) return fail(MPYC_B200_EINVAL, "shamir_split: need 0 <= t < m");
        if (!h_secrets || !h_shares || (t > 0 && !h_coeffs)) return fail(MPYC_B200_EINVAL, "reshare_step_host: null split buffer");
    }
    if (n_rec) {
        if (!h_share_rows || !xs || !x_rs || !h_out) return fail(MPYC_B200_EINVAL, "reshare_step_host: null recombine argument");
        if (k < 1 || width < 1) return fail(MPYC_B200_EINVAL, "reshare_step_host: bad k/width");
        if (k > MPYC_B200_MAX_POINTS) return fail(MPYC_B200_EUNSUPPORTED, "reshare_step_host: more than MPYC_B200_MAX_POINTS shares");
    }
    if (n_split == 0 && n_rec == 0) return MPYC_B200_OK;
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    // half-size chunks: twice as many interleaving points between the two jobs for the same staging memory
    const size_t chs = n_split ? std::max<size_t>(chunk_elems(n_split, 2 * eb * (size_t)(t + 1 + m)), 16) : 16;
    const size_t chr = n_rec ? std::max<size_t>(chunk_elems(n_rec, 2 * eb * (size_t)(k + width)), 16) : 16;
    DeviceGuard guard;
    Workspace *ws, *wr;
    int rc = acquire_workspace(device, &ws, 0);
    if (rc == MPYC_B200_OK) rc = acquire_workspace(device, &wr, 1);
    if (rc) return rc;
    std::lock_guard<std::mutex> g0(ws->mu);          // always set 0 before set 1
    std::lock_guard<std::mutex> g1(wr->mu);
    if (n_split) rc = reserve(*ws, chs * eb * (size_t)(t + 1), chs * eb * (size_t)m);
    if (rc == MPYC_B200_OK && n_rec) rc = reserve(*wr, chr * eb * (size_t)k, chr * eb * (size_t)width);
    if (rc) return rc;
    const size_t cs = n_split ? (n_split + chs - 1) / chs : 0, cr = n_rec ? (n_rec + chr - 1) / chr : 0;
    for (size_t c = 0; c < std::max(cs, cr); c++) {
        if (c < cs) {
            rc = split_chunk(f, ws, (int)(c % kSlots), chs, eb, h_secrets, h_coeffs, coeff_stride, h_shares, share_stride, c * chs,
                             std::min(chs, n_split - c * chs), t, m);
            if (rc) return rc;
        }
        if (c < cr) {
            rc = recombine_chunk(f, wr, (int)(c % kSlots), chr, eb, h_share_rows, xs, k, x_rs, width, h_out, out_stride, c * chr,
                                 std::min(chr, n_rec - c * chr));
            if (rc) return rc;
        }
    }
    for (int s = 0; s < kSlots && (size_t)s < cs; s++) CU(cudaStreamSynchronize(ws->streams[s]));
    for (int s = 0; s < kSlots && (size_t)s < cr; s++) CU(cudaStreamSynchronize(wr->streams[s]));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_ff_binop_host(const mpyc_b200_field* f, int op, const void* h_a, const void* h_b, void* h_out,
                                       size_t n, int device) {
    if (!f || (n && (!h_a || !h_b || !h_out))) return fail(MPYC_B200_EINVAL, "ff_binop_host: null argument");
    if (n == 0) return MPYC_B200_OK;
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    const size_t ch = chunk_elems(n, eb * 3);
    DeviceGuard guard;
    Workspace* w;
    int rc = acquire_workspace(device, &w);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(w->mu);
    rc = reserve(*w, ch * eb * 2, ch * eb);
    if (rc) return rc;
    size_t c = 0;
    for (size_t off = 0; off < n; off += ch, c++) {
        const int s = (int)(c % kSlots);
        const size_t cn = std::min(ch, n - off);
        cudaStream_t st = w->streams[s];
        char* din = (char*)w->d_in[s];
        char* dout = (char*)w->d_out[s];
        CU(cudaMemcpyAsync(din, (const char*)h_a + off * eb, cn * eb, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(din + ch * eb, (const char*)h_b + off * eb, cn * eb, cudaMemcpyHostToDevice, st));
        rc = mpyc_b200_ff_binop(f, op, din, din + ch * eb, dout, cn, st);
        if (rc) return rc;
        CU(cudaMemcpyAsync((char*)h_out + off * eb, dout, cn * eb, cudaMemcpyDeviceToHost, st));
    }
    for (int s = 0; s < kSlots && (size_t)s < c; s++) CU(cudaStreamSynchronize(w->streams[s]));   // only the slots this call used
    return MPYC_B200_OK;
}

// ---------------------------------------------------------------------------------------
// PRF / PRSS with the XOF inside the library
// ---------------------------------------------------------------------------------------

MPYC_API int mpyc_b200_enable_peer_access(int device, int peer_device) {
    if (device == peer_device) return MPYC_B200_OK;
    int can = 0;
    CU(cudaDeviceCanAccessPeer(&can, device, peer_device));
    if (!can) return fail(MPYC_B200_EUNSUPPORTED, "enable_peer_access: the devices cannot access each other's memory");
    int prev = 0;
    CU(cudaGetDevice(&prev));
    CU(cudaSetDevice(device));
    cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();   // clear the sticky-less error state
        e = cudaSuccess;
    }
    cudaSetDevice(prev);
    return e == cudaSuccess ? MPYC_B200_OK : cuda_fail(e, "cudaDeviceEnablePeerAccess");
}

// Receive buffers another process's kernels can store into: plain cudaMalloc allocations exported / imported with
// CUDA IPC.  The importer opens the handle in ITS OWN device's context (cudaIpcMemLazyEnablePeerAccess turns peer
// access to the exporting GPU on), so kernels it launches can address the memory directly over NVLink.
MPYC_API int mpyc_b200_peer_alloc(size_t bytes, void** d_ptr, uint8_t handle[64]) {
    if (!d_ptr || !handle || bytes == 0) return fail(MPYC_B200_EINVAL, "peer_alloc: bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    void* p = nullptr;
    CU(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();   // the memset is asynchronous with respect to the host
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return cuda_fail(e, "peer_alloc");
    }
    memcpy(handle, &h, 64);
    *d_ptr = p;
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_peer_open(const uint8_t handle[64], void** d_ptr) {
    if (!d_ptr || !handle) return fail(MPYC_B200_EINVAL, "peer_open: bad arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CU(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_peer_close(void* d_ptr) {
    if (d_ptr) CU(cudaIpcCloseMemHandle(d_ptr));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_peer_free(void* d_ptr) {
    if (d_ptr) CU(cudaFree(d_ptr));
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_shake128(const uint8_t* in, size_t inlen, uint8_t* out, size_t outlen) {
    if ((inlen && !in) || (outlen && !out)) return fail(MPYC_B200_EINVAL, "shake128: null buffer");
    mpyc_shake::Shake128 x;
    x.absorb(in, inlen);
    x.squeeze(out, outlen);
    return MPYC_B200_OK;
}

// count sponges SHAKE128(key_i || suffix), i < count, squeezed to outlen bytes each at out + i * out_stride: the XOF
// streams of one PRSS call (thresha.py:257 with key_i per subset and suffix = uci).  Sponges are processed eight at a
// time in the AVX-512 lock-step form when the host has it (*used_wide = 1), else one by one.  Host only.
MPYC_API int mpyc_b200_shake128_multi(const uint8_t* keys, int key_bytes, const uint8_t* suffix, size_t suffix_len, int count,
                                        uint8_t* out, size_t out_stride, size_t outlen, int* used_wide) {
    if (count < 0 || key_bytes < 0 || (count && key_bytes && !keys) || (suffix_len && !suffix) || (count && outlen && !out))
        return fail(MPYC_B200_EINVAL, "shake128_multi: bad arguments");
    const bool wide = mpyc_shake::x8_available();
    if (used_wide) *used_wide = wide ? 1 : 0;
    for (int b = 0; b < count;) {
        const int take = (wide && count - b >= 2) ? std::min(count - b, 8) : 1;
        if (take >= 2) {
            mpyc_shake::Shake128x8 g;
            g.reset(take);
            const uint8_t* kp[8] = {};
            const uint8_t* sp[8] = {};
            uint8_t* op[8] = {};
            for (int q = 0; q < take; q++) {
                kp[q] = keys + (size_t)(b + q) * key_bytes;
                sp[q] = suffix;
                op[q] = out + (size_t)(b + q) * out_stride;
            }
            g.absorb(kp, (size_t)key_bytes);
            g.absorb(sp, suffix_len);
            g.squeeze(op, outlen);
        } else {
            mpyc_shake::Shake128 x;
            x.absorb(keys + (size_t)b * key_bytes, (size_t)key_bytes);
            x.absorb(suffix, suffix_len);
            x.squeeze(out + (size_t)b * out_stride, outlen);
        }
        b += take;
    }
    return MPYC_B200_OK;
}

namespace {

struct PinnedStage {   // pinned host staging for the PRF byte streams, one buffer per pipeline slot, per device
    void* h[kSlots] = {nullptr, nullptr, nullptr};
    size_t cap = 0;
};
PinnedStage g_pin[16];

int reserve_pinned(PinnedStage& p, size_t bytes) {
    if (bytes <= p.cap) return MPYC_B200_OK;
    for (int s = 0; s < kSlots; s++) {
        if (p.h[s]) cudaFreeHost(p.h[s]);
        p.h[s] = nullptr;
    }
    p.cap = 0;
    for (int s = 0; s < kSlots; s++) CU(cudaHostAlloc(&p.h[s], bytes, cudaHostAllocDefault));
    p.cap = bytes;
    return MPYC_B200_OK;
}

}   // namespace

// CPUs this process may actually use: hardware threads, capped by the scheduler affinity mask and by a cgroup CPU quota
// (a container that sees 128 hardware threads but is limited to 8 CPUs' worth of time -- the round-1 GPU box)
static int usable_cpus() {
    int n = (int)std::thread::hardware_concurrency();
    if (n < 1) n = 1;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) {
        const int a = CPU_COUNT(&set);
        if (a >= 1 && a < n) n = a;
    }
    if (FILE* fh = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char quota[32] = "";
        long period = 0;
        if (fscanf(fh, "%31s %ld", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0) {
            const long q = (atol(quota) + period - 1) / period;
            if (q >= 1 && q < n) n = (int)q;
        }
        fclose(fh);
    }
    return n;
}

// general: PRF bound given by `general` (two kernels per chunk: k_prf_reduce, then K4 on the reduced values);
// otherwise bound_bits as in mpyc_b200_prss_combine
static int prss_host_impl(const mpyc_b200_field* f, const uint8_t* h_keys, int key_bytes, const uint8_t* h_uci,
                          size_t uci_bytes, int nsub, int d, int chunk_bytes, int bound_bits, const BoundSpec* general,
                          const uint64_t* h_coef, const uint64_t* h_weights, void* h_out, size_t n, int device, int max_threads) {
    if (!f || !h_keys || key_bytes < 0 || (uci_bytes && !h_uci) || !h_coef || !h_weights || nsub < 1 || d < 1 || chunk_bytes < 1 ||
        (n && !h_out))
        return fail(MPYC_B200_EINVAL, "prss_host: bad arguments");
    if (n == 0) return MPYC_B200_OK;
    const bool gf = f->kind == MPYC_B200_KIND_GF256;
    const int vbytes = general ? (gf ? 1 : 8 * general->LB) : 0;      // width of a reduced value (general bounds)
    if (general && (chunk_bytes > 8 * (general->LB + 2))) return fail(MPYC_B200_EINVAL, "prss_host: chunk too wide for this bound");
    size_t eb;
    mpyc_b200_field_info(f, nullptr, nullptr, nullptr, &eb);
    const size_t per_elem = (size_t)d * chunk_bytes;
    // elements per pipeline chunk: a multiple of the kernel's 256-element tiles; at least ~384 KiB of XOF output per
    // sponge (about a millisecond of squeezing) and, for long calls, about a sixth of the call (at most 4 MiB per
    // sponge): every chunk boundary is a rendezvous of all sponge threads with the copy/launch thread, and with
    // ~1 ms chunks the scheduling jitter of 20 threads cost a third of the throughput (round 2: 26 chunks per
    // np_cnnmnist-sized call, 164 MB/s per sponge thread against 367 MB/s for a free-running sponge)
    size_t ce = std::max<size_t>((384u << 10) / per_elem / 256 * 256, 256);
    const size_t sixth = round_up((n + 5) / 6, 256);
    const size_t cap = std::max<size_t>((4u << 20) / per_elem / 256 * 256, 256);
    ce = std::max(ce, std::min(sixth, cap));
    if (getenv("MPYC_B200_PRSS_CHUNK")) ce = std::max<size_t>(round_up((size_t)atol(getenv("MPYC_B200_PRSS_CHUNK")), 256), 256);
    ce = std::min(ce, round_up(n, 256));
    const size_t cstride = round_up(ce * per_elem, 16);               // bytes per subset per chunk
    const size_t nchunks = (n + ce - 1) / ce;
    DeviceGuard guard;
    Workspace* w;
    int rc = acquire_workspace(device, &w);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(w->mu);
    rc = reserve(*w, cstride * nsub, ce * eb);
    if (rc) return rc;
    rc = reserve_pinned(g_pin[device], cstride * nsub);
    if (rc) return rc;
    const size_t vstride = general ? round_up(ce * (size_t)d * vbytes, 16) : 0;   // reduced values per subset per chunk
    if (general) {
        rc = reserve_tmp(*w, vstride * nsub);
        if (rc) return rc;
    }
    PinnedStage& pin = g_pin[device];
    PrssTable tab;
    rc = general ? prss_prepare(f, nsub, d, vbytes, 0, h_coef, h_weights, w->streams[0], tab)
                 : prss_prepare(f, nsub, d, chunk_bytes, bound_bits, h_coef, h_weights, w->streams[0], tab);
    if (rc) return rc;

    // One sponge per key subset (thresha.py:257: shake_128(key + s)), dealt round-robin to the worker threads.  A worker
    // that owns several sponges squeezes them in lock step, eight at a time, with the AVX-512 form (shake128_x8.h)
    // when the host has it; a worker with a single sponge, or a host without AVX-512, uses the scalar sponge.
    const int hw = usable_cpus();
    int nthreads = std::min(nsub, max_threads > 0 ? max_threads : hw);
    if ((size_t)nsub * n * per_elem < (64u << 10)) nthreads = 1;       // tiny calls: thread start-up costs more than it saves
    struct Unit {
        std::vector<int> subs;             // key subsets of this unit (1 for scalar, 2..8 for the wide form)
        mpyc_shake::Shake128 scalar;
        mpyc_shake::Shake128x8 wide;
        bool is_wide = false;
    };
    const bool use_x8 = mpyc_shake::x8_available();
    std::vector<std::vector<Unit>> units(nthreads);
    for (int wk = 0; wk < nthreads; wk++) {
        std::vector<int> mine;
        for (int S = wk; S < nsub; S += nthreads) mine.push_back(S);
        for (size_t b = 0; b < mine.size();) {
            const size_t left = mine.size() - b;
            const size_t take = (use_x8 && left >= 2) ? std::min<size_t>(left, 8) : 1;
            units[wk].emplace_back();
            Unit& u = units[wk].back();
            u.subs.assign(mine.begin() + b, mine.begin() + b + take);
            if (take >= 2) {
                u.is_wide = true;
                u.wide.reset((int)take);
                const uint8_t* kp[8] = {};
                const uint8_t* up[8] = {};
                for (size_t q = 0; q < take; q++) {
                    kp[q] = h_keys + (size_t)u.subs[q] * key_bytes;
                    up[q] = h_uci;
                }
                u.wide.absorb(kp, (size_t)key_bytes);
                u.wide.absorb(up, uci_bytes);
            } else {
                u.scalar.absorb(h_keys + (size_t)u.subs[0] * key_bytes, (size_t)key_bytes);
                u.scalar.absorb(h_uci, uci_bytes);
            }
            b += take;
        }
    }
    auto squeeze_worker = [&](int wk, uint8_t* base, size_t len) {
        for (Unit& u : units[wk]) {
            if (u.is_wide) {
                uint8_t* outs[8] = {};
                for (size_t q = 0; q < u.subs.size(); q++) outs[q] = base + (size_t)u.subs[q] * cstride;
                u.wide.squeeze(outs, len);
            } else {
                u.scalar.squeeze(base + (size_t)u.subs[0] * cstride, len);
            }
        }
    };
    std::vector<std::atomic<int>> produced(nchunks);
    for (auto& p : produced) p.store(0, std::memory_order_relaxed);
    std::atomic<size_t> consumed{0};                                  // chunks whose pinned slot may be overwritten
    std::atomic<bool> abort_flag{false};
    auto produce = [&](int worker) {
        for (size_t c = 0; c < nchunks; c++) {
            while (c >= consumed.load(std::memory_order_acquire) + kSlots) {   // slot c % kSlots still in flight
                if (abort_flag.load(std::memory_order_relaxed)) return;
                std::this_thread::sleep_for(std::chrono::microseconds(50));   // do not burn a core the sponges could use
            }
            const size_t cn = std::min(ce, n - c * ce);
            squeeze_worker(worker, (uint8_t*)pin.h[c % kSlots], cn * per_elem);
            produced[c].fetch_add(1, std::memory_order_release);
        }
    };
    std::vector<std::thread> workers;
    if (nthreads > 1)
        for (int t = 0; t < nthreads; t++) workers.emplace_back(produce, t);
    auto finish_workers = [&]() {
        abort_flag.store(true);
        for (auto& t : workers) t.join();
    };
    cudaEvent_t copied[kSlots];
    for (int s = 0; s < kSlots; s++) cudaEventCreateWithFlags(&copied[s], cudaEventDisableTiming);
    auto cleanup = [&](int code) {   // error path: stop the producers, drain the streams (the table is freed after this)
        finish_workers();
        for (int s = 0; s < kSlots; s++) cudaStreamSynchronize(w->streams[s]);
        for (int s = 0; s < kSlots; s++) cudaEventDestroy(copied[s]);
        return code;
    };
    for (size_t c = 0; c < nchunks; c++) {
        const int s = (int)(c % kSlots);
        const size_t cn = std::min(ce, n - c * ce);
        cudaStream_t st = w->streams[s];
        if (nthreads == 1) {
            if (c >= kSlots) {                                        // slot reuse: its H2D copy must have left the host buffer
                if (cudaEventSynchronize(copied[s]) != cudaSuccess) return cleanup(cuda_fail(cudaGetLastError(), "prss_host event"));
            }
            squeeze_worker(0, (uint8_t*)pin.h[s], cn * per_elem);
        } else {
            while (produced[c].load(std::memory_order_acquire) < nthreads) std::this_thread::sleep_for(std::chrono::microseconds(50));
        }
        cudaError_t e = cudaMemcpyAsync(w->d_in[s], pin.h[s], cstride * nsub, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaEventRecord(copied[s], st);
        if (e != cudaSuccess) return cleanup(cuda_fail(e, "prss_host H2D"));
        if (general) {
            rc = prf_reduce_launch(*general, gf ? f->gf_poly : 0u, (const uint8_t*)w->d_in[s], cstride, nsub, cn * (size_t)d, chunk_bytes,
                                   w->d_tmp[s], vstride, st);
            if (rc == MPYC_B200_OK) rc = prss_launch(f, tab, (const uint8_t*)w->d_tmp[s], vstride, nsub, d, vbytes, 0, w->d_out[s], cn, st);
        } else {
            rc = prss_launch(f, tab, (const uint8_t*)w->d_in[s], cstride, nsub, d, chunk_bytes, bound_bits, w->d_out[s], cn, st);
        }
        if (rc) return cleanup(rc);
        e = cudaMemcpyAsync((char*)h_out + c * ce * eb, w->d_out[s], cn * eb, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return cleanup(cuda_fail(e, "prss_host D2H"));
        if (nthreads > 1 && c + 1 >= (size_t)kSlots) {
            // chunk c+1-kSlots's slot is needed next by the producers: wait until its copy has left the host buffer
            const size_t old = c + 1 - kSlots;
            if (cudaEventSynchronize(copied[old % kSlots]) != cudaSuccess) return cleanup(cuda_fail(cudaGetLastError(), "prss_host event"));
            consumed.store(old + 1, std::memory_order_release);
        }
    }
    for (int s = 0; s < kSlots; s++)
        if (cudaStreamSynchronize(w->streams[s]) != cudaSuccess) return cleanup(cuda_fail(cudaGetLastError(), "prss_host sync"));
    for (auto& t : workers) t.join();
    workers.clear();
    for (int s = 0; s < kSlots; s++) cudaEventDestroy(copied[s]);
    return MPYC_B200_OK;
}

MPYC_API int mpyc_b200_prss_host(const mpyc_b200_field* f, const uint8_t* h_keys, int key_bytes, const uint8_t* h_uci,
                                   size_t uci_bytes, int nsub, int d, int chunk_bytes, int bound_bits, const uint64_t* h_coef,
                                   const uint64_t* h_weights, void* h_out, size_t n, int device, int max_threads) {
    return prss_host_impl(f, h_keys, key_bytes, h_uci, uci_bytes, nsub, d, chunk_bytes, bound_bits, nullptr, h_coef, h_weights, h_out, n,
                          device, max_threads);
}

MPYC_API int mpyc_b200_prss_host_bound(const mpyc_b200_field* f, const uint8_t* h_keys, int key_bytes, const uint8_t* h_uci,
                                         size_t uci_bytes, int nsub, int d, int chunk_bytes, const uint64_t* h_bound, int bound_nlimbs,
                                         const uint64_t* h_coef, const uint64_t* h_weights, void* h_out, size_t n, int device,
                                         int max_threads) {
    BoundSpec b;
    int rc = bound_spec(h_bound, bound_nlimbs, b);
    if (rc) return rc;
    return prss_host_impl(f, h_keys, key_bytes, h_uci, uci_bytes, nsub, d, chunk_bytes, 0, &b, h_coef, h_weights, h_out, n, device,
                          max_threads);
}
