// Stream probe: the memory traffic of K2 (share generation) and K3 (Lagrange recombination) with no arithmetic, so
// that each kernel can be set against what its access pattern and its read/write mix allow on this card.
// A mix is `nin` rows read and `nout` rows written, every row the same number of bytes; output row o of an element is
// the XOR of its inputs with o.  Access forms:
//   item32     a thread moves one 32-byte item per row as two 16-byte accesses, lanes 32 bytes apart (the layout K2
//              and K3 had before they were tiled)
//   coalesced  a CTA owns 8 KB of every row per trip; a thread moves 16-byte chunks tid and tid + 256, so that a warp
//              access covers 512 contiguous bytes (k_split_tiled, k_recombine_tiled for L <= 2)
//   bulk       coalesced loads; the outputs go to an nout x 8 KB stage in shared memory and leave as one TMA bulk
//              store per row (cp.async.bulk; k_split_tiled, k_recombine_tiled for L = 4)
// plus a device-to-device copy of 2 GiB.  Prints one JSON object per measurement.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/stream_probe.cu (tools/stream_probe.py does this).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

#define THREADS 256
#define TILE 512   // 16-byte chunks per row and tile (8 KB)
#define MAXR 8

#define CK(x)                                                                              \
    do {                                                                                   \
        cudaError_t e_ = (x);                                                              \
        if (e_ != cudaSuccess) {                                                           \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                       \
        }                                                                                  \
    } while (0)

struct Rows {
    const uint4* in[MAXR];
    uint4* out[MAXR];
};

__device__ __forceinline__ uint4 ld(const uint4* p) {
    uint4 v;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st(uint4* p, uint4 v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 x4(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }
__device__ __forceinline__ uint4 xo(uint4 a, unsigned o) { return make_uint4(a.x ^ o, a.y, a.z, a.w); }

enum { ITEM32 = 0, COALESCED = 1, BULK = 2 };

template <int NIN, int NOUT, int FORM>
__global__ void __launch_bounds__(THREADS, 1) k_probe(Rows r, size_t chunks) {
    const size_t nth = (size_t)gridDim.x * blockDim.x;
    if constexpr (FORM == ITEM32) {
        for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < chunks / 2; it += nth) {
            uint4 a = ld(r.in[0] + 2 * it), b = ld(r.in[0] + 2 * it + 1);
#pragma unroll
            for (int j = 1; j < NIN; j++) {
                a = x4(a, ld(r.in[j] + 2 * it));
                b = x4(b, ld(r.in[j] + 2 * it + 1));
            }
#pragma unroll
            for (int o = 0; o < NOUT; o++) {
                st(r.out[o] + 2 * it, xo(a, o));
                st(r.out[o] + 2 * it + 1, xo(b, o));
            }
        }
    } else {
        extern __shared__ __align__(128) uint4 stage[];
        for (size_t tile = blockIdx.x; tile < chunks / TILE; tile += gridDim.x) {
            const size_t c = tile * TILE + threadIdx.x;
            uint4 a = ld(r.in[0] + c), b = ld(r.in[0] + c + THREADS);
#pragma unroll
            for (int j = 1; j < NIN; j++) {
                a = x4(a, ld(r.in[j] + c));
                b = x4(b, ld(r.in[j] + c + THREADS));
            }
            if constexpr (FORM == COALESCED) {
#pragma unroll
                for (int o = 0; o < NOUT; o++) {
                    st(r.out[o] + c, xo(a, o));
                    st(r.out[o] + c + THREADS, xo(b, o));
                }
            } else {
                if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                __syncthreads();
#pragma unroll
                for (int o = 0; o < NOUT; o++) {
                    stage[o * TILE + threadIdx.x] = xo(a, o);
                    stage[o * TILE + threadIdx.x + THREADS] = xo(b, o);
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncthreads();
                if (threadIdx.x == 0) {
                    for (int o = 0; o < NOUT; o++)
                        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(r.out[o] + tile * TILE),
                                     "r"((unsigned)__cvta_generic_to_shared(stage + o * TILE)), "n"(TILE * 16)
                                     : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if constexpr (FORM == BULK) {
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        }
    }
}

static const char* FORMS[] = {"item32", "coalesced", "bulk"};
static int g_sms;

template <int NIN, int NOUT, int FORM>
static void run(const char* mix, size_t row_bytes, uint4* pool, int reps) {
    auto kernel = k_probe<NIN, NOUT, FORM>;
    const size_t smem = FORM == BULK ? (size_t)NOUT * TILE * 16 : 0;
    if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, THREADS, smem));
    const size_t chunks = row_bytes / 16;
    const size_t work = FORM == ITEM32 ? chunks / 2 / THREADS : chunks / TILE;   // CTAs' worth of items
    const int grid = (int)(work < (size_t)g_sms * occ ? work : (size_t)g_sms * occ);
    Rows r;
    for (int j = 0; j < NIN; j++) r.in[j] = pool + (size_t)j * chunks;
    for (int o = 0; o < NOUT; o++) r.out[o] = pool + (size_t)(NIN + o) * chunks;
    for (int i = 0; i < 3; i++) kernel<<<grid, THREADS, smem>>>(r, chunks);
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int i = 0; i < reps; i++) kernel<<<grid, THREADS, smem>>>(r, chunks);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= reps;
    const double bytes = (double)(NIN + NOUT) * row_bytes;
    printf("{\"mix\": \"%s\", \"in\": %d, \"out\": %d, \"row_bytes\": %zu, \"form\": \"%s\", \"ctas_per_sm\": %d, "
           "\"ms\": %.4f, \"GBps\": %.1f}\n",
           mix, NIN, NOUT, row_bytes, FORMS[FORM], occ, ms, bytes / (ms * 1e-3) / 1e9);
    fflush(stdout);
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
}

template <int NIN, int NOUT>
static void mix(const char* name, size_t row_bytes, uint4* pool, int reps) {
    row_bytes = row_bytes / (TILE * 16) * (TILE * 16);
    run<NIN, NOUT, ITEM32>(name, row_bytes, pool, reps);
    run<NIN, NOUT, COALESCED>(name, row_bytes, pool, reps);
    run<NIN, NOUT, BULK>(name, row_bytes, pool, reps);
}

int main(int argc, char** argv) {
    const int reps = argc > 1 ? atoi(argv[1]) : 20;
    CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
    // rows as long as the bench's: 1e8 16-byte (C3), 2e8 8-byte (ns64) and 2e7 32-byte (C5) elements
    const size_t c3 = 1600000000ull, ns64 = 1600000000ull, c5 = 640000000ull;
    const size_t pool_bytes = 8 * c3;   // the largest mix: 3 + 5 rows of C3's length
    uint4* pool;
    CK(cudaMalloc(&pool, pool_bytes));
    CK(cudaMemset(pool, 0x5a, pool_bytes));
    mix<3, 1>("K3 c3", c3, pool, reps);
    mix<2, 1>("K3 ns64", ns64, pool, reps);
    mix<7, 1>("K3 c5", c5, pool, reps);
    mix<3, 5>("K2 c3", c3, pool, reps);
    mix<2, 3>("K2 ns64", ns64, pool, reps);
    mix<4, 7>("K2 c5", c5, pool, reps);
    // device-to-device copy of 2 GiB (read + write counted)
    const size_t cb = 2ull << 30;
    for (int i = 0; i < 3; i++) CK(cudaMemcpyAsync(pool + cb / 16, pool, cb, cudaMemcpyDeviceToDevice));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int i = 0; i < reps; i++) CK(cudaMemcpyAsync(pool + cb / 16, pool, cb, cudaMemcpyDeviceToDevice));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= reps;
    printf("{\"mix\": \"copy 2 GiB\", \"in\": 1, \"out\": 1, \"row_bytes\": %zu, \"form\": \"cudaMemcpy\", \"ms\": %.4f, "
           "\"GBps\": %.1f}\n",
           cb, ms, 2.0 * cb / (ms * 1e-3) / 1e9);
    CK(cudaFree(pool));
    return 0;
}
