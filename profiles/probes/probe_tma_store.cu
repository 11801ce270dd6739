// probe_tma_store.cu -- what is the ceiling of the render kernel's output pattern?
// Persistent CTAs each own one shared-memory buffer and bulk-store it (cp.async.bulk.global.shared::cta) to
// consecutive `chunk`-byte slots of a large output, round-robin over CTAs, waiting for the previous store's
// smem read-out before re-issuing (exactly the render kernel's store discipline, nothing else).
// usage: probe_tma_store  -> prints GB/s for a sweep of chunk sizes / alignments / CTAs per SM / mode
//   mode 0: TMA bulk store; mode 1: st.global.v4 by all threads (coalesced) from smem; mode 2: mode 0 + wait_group 0;
//   mode 3 (slots sweep only): no store at all
// usage: probe_tma_store slots -> the render's tile loop with one or two tile buffers per CTA: tile i of a CTA goes
//   to buffer i % slots, and before a buffer is refilled the CTA waits (wait_group.read slots - 1) only for the store
//   that read it last.  Between the wait and the store the CTA stands in for the composition: it rewrites the first
//   `fill` bytes of the buffer with 16-byte stores, then every thread spins for a fixed number of clock cycles;
//   "compose only" runs the same loop with the stores left out (mode 3).  The whole sweep runs three times.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void store_kernel(unsigned char *out, size_t n_chunks, unsigned chunk, int mode, int slots, long long spin,
                             unsigned fill) {
    extern __shared__ __align__(128) unsigned char buf[];
    for (unsigned q = threadIdx.x; q < slots * chunk / 4; q += blockDim.x) ((unsigned *)buf)[q] = q * 2654435761u + blockIdx.x;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    unsigned i = 0;
    for (size_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++i) {
        unsigned char *dst = out + c * (size_t)chunk;
        unsigned char *src = buf + (slots == 2 ? (i & 1u) * chunk : 0u);
        if (mode == 1) {
            for (unsigned q = threadIdx.x; q < chunk / 16; q += blockDim.x) ((uint4 *)dst)[q] = ((uint4 *)buf)[q];
        } else {
            if (threadIdx.x == 0) {
                if (mode == 2) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
                else if (slots == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            }
            __syncthreads();
            // (the render kernel composes the tile here)
            for (unsigned q = threadIdx.x; q < fill / 16; q += blockDim.x) ((uint4 *)src)[q] = make_uint4(q, i, q, i);
            if (spin > 0) {
                const long long t0 = clock64();
                while (clock64() - t0 < spin) {}
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (threadIdx.x == 0 && mode != 3) {
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst), "r"(smem_u32(src)), "r"(chunk) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// one launch shape, timed over `reps` launches after one warm-up; returns the mean ms
static float run(unsigned char *out, unsigned char *flush, size_t flush_bytes, size_t n_chunks, unsigned chunk,
                 int mode, int slots, long long spin, unsigned fill, int grid, int threads, float *best_ms) {
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e9f, sum = 0;
    const int reps = 5;
    for (int r = 0; r < reps + 1; ++r) {
        CK(cudaMemsetAsync(flush, r, flush_bytes));
        CK(cudaEventRecord(e0));
        store_kernel<<<grid, threads, (size_t)slots * chunk>>>(out, n_chunks, chunk, mode, slots, spin, fill);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r == 0) continue;
        if (ms < best) best = ms;
        sum += ms;
    }
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
    *best_ms = best;
    return sum / reps;
}

int main(int argc, char **argv) {
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    printf("PROBE device %s, %d SMs, %zu B shared memory per SM\n", prop.name, sms, prop.sharedMemPerMultiprocessor);
    const size_t total = (size_t)2574336000ull;            // bytes of one render launch in bench.py
    unsigned char *out; CK(cudaMalloc(&out, total + (1 << 20)));
    unsigned char *flush; const size_t flush_bytes = 512u << 20; CK(cudaMalloc(&flush, flush_bytes));
    CK(cudaFuncSetAttribute(store_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CK(cudaFuncSetAttribute(store_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    if (argc > 1 && !strcmp(argv[1], "slots")) {
        // battle512: one launch renders 64000 tiles of 8 records of 4732 bytes with 256 threads per CTA
        const unsigned chunk = 37856;
        const size_t n_chunks = 64000;
        const int threads = 256;
        // spins: none, and 4000 / 4800 / 6000 cycles (4800 makes one slot at 4 CTAs/SM compose for about the 0.349 ms
        // the render's composition takes without its store); fill: none, or a quarter tile (the render rebuilds a
        // record about once every four tiles)
        const long long spins[] = {0, 4000, 4800, 6000};
        const unsigned fills[] = {0, chunk / 4 & ~15u};
        const int shapes[][2] = {{1, 4}, {2, 3}, {2, 2}, {1, 3}};   // {slots, CTAs per SM}
        for (int round = 0; round < 3; ++round)
            for (unsigned fill : fills)
                for (long long spin : spins)
                    for (const auto &s : shapes) {
                        const int slots = s[0], c = s[1];
                        int occ = 0;
                        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, store_kernel, threads, (size_t)slots * chunk));
                        if (occ < c) { printf("PROBE slots %d ctas/sm %d: only %d fit\n", slots, c, occ); continue; }
                        float best, best0;
                        const float ms = run(out, flush, flush_bytes, n_chunks, chunk, 0, slots, spin, fill, c * sms, threads, &best);
                        const float ms0 = run(out, flush, flush_bytes, n_chunks, chunk, 3, slots, spin, fill, c * sms, threads, &best0);
                        printf("PROBE round %d slots %d ctas/sm %d fill %5u B spin %4lld cycles  store mean %.3f ms (%.0f GB/s) "
                               "best %.3f ms   compose only mean %.3f ms\n", round, slots, c, fill, spin, ms,
                               n_chunks * (double)chunk / ms / 1e6, best, ms0);
                        fflush(stdout);
                    }
        return 0;
    }
    const unsigned chunks[] = {18928, 18944, 9472, 37856, 16384, 32768, 65536};
    const int ctas[] = {4, 8, 11, 16};
    for (int mode = 0; mode < 3; ++mode)
        for (unsigned chunk : chunks)
            for (int c : ctas) {
                if ((size_t)c * (chunk + 1024) > 227 * 1024) continue;
                const size_t n_chunks = total / chunk;
                float best;
                const float mean = run(out, flush, flush_bytes, n_chunks, chunk, mode, 1, 0, 0, c * sms, 128, &best);
                printf("PROBE mode %d chunk %6u ctas/sm %2d  mean %.3f ms  %.0f GB/s   best %.0f GB/s\n", mode, chunk, c,
                       mean, n_chunks * (double)chunk / mean / 1e6, n_chunks * (double)chunk / best / 1e6);
                fflush(stdout);
            }
    // reference point: cudaMemset of the same range
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int r = 0; r < 3; ++r) {
        CK(cudaEventRecord(e0)); CK(cudaMemsetAsync(out, 1, total)); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        printf("PROBE memset %.3f ms %.0f GB/s\n", ms, total / ms / 1e6);
    }
    return 0;
}
