// backend_cuda.cu -- the sm_90a backend: CUDA runtime plumbing + every kernel of the engine.
//
// Kernels (DESIGN.md §5):
//   step_kernel_cta   one CTA per arena runs the whole step pipeline (run_step) with __syncthreads
//                     between phases; arenas are looped grid-stride.          [many small arenas]
//   step_kernel_grid  cooperative launch; the whole grid is one team per arena with grid.sync()
//                     between phases.                                          [one huge arena]
//   cull_kernel_*     clear_dead: stable compaction into the ping-pong SoA buffers.
//   offsets_kernel    prefix of per-arena counts -> ABI concatenation offsets.
//   minimap_*         per (arena, group) histogram of coarse cells + normalisation.
//   obs_render_kernel the observation gather: the HBM-write-bound kernel the roofline is quoted on.
//   info_kernel       id/pos/alive/reward gathers and the action scatter.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "backend.h"
#if defined(MG_PHASE_TIMING)
namespace mg { __device__ long long mg_phase_clock[8 * 32]; }
#endif
#include "obs_phases.h"
#include "mask_phases.h"
#include "nbr_phases.h"
#include "rule_phases.h"
#include "slot_phases.h"
#include "replay_phases.h"

namespace cg = cooperative_groups;

namespace mg {
[[noreturn]] void fatal(const char *fmt, ...);
namespace be {

#define CUDA_CHECK(expr)                                                                          \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) mg::fatal("CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e),   \
                                         __FILE__, __LINE__, #expr);                              \
    } while (0)

static std::atomic<long long> g_launches{0};       // instrumentation only (magent_b200_launch_count)

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to (function, device), not to an engine: it is only ever raised,
// under a lock, so that a second engine with a smaller need cannot pull it from under the first.  The same slots cache
// each kernel's static shared memory.
enum { ATTR_STEP = 0, ATTR_OBS0 = 1, ATTR_MEAN = 1 + 12, ATTR_MEAN_SLOTS, ATTR_MASK, ATTR_MASK_SLOTS, ATTR_WIRE,
       ATTR_MINIMAP_SMALL, ATTR_N, ATTR_MAX_DEVICES = 64 };
static std::mutex g_attr_mu;
static size_t g_attr_smem[ATTR_MAX_DEVICES][ATTR_N];
static size_t g_attr_static[ATTR_MAX_DEVICES][ATTR_N];      // static shared memory + 1 (0: not queried yet)
template <class K>
static void ensure_dynamic_smem(int device, int slot, K kernel, size_t smem) {
    std::lock_guard<std::mutex> lk(g_attr_mu);
    size_t &have = g_attr_smem[device % ATTR_MAX_DEVICES][slot];
    if (smem <= have) return;
    CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    have = smem;
}
// The kernel's own __shared__ variables as the compiler laid them out (cudaFuncAttributes::sharedSizeBytes: 6400 bytes
// for the kernels that hold an EngineDev copy, 128 for the render and the wire kernel with CUDA 12.9), which a launch
// adds to its dynamic shared memory.  Queried once per (kernel, device).
template <class K>
static size_t static_smem(int device, int slot, K kernel) {
    std::lock_guard<std::mutex> lk(g_attr_mu);
    size_t &have = g_attr_static[device % ATTR_MAX_DEVICES][slot];
    if (!have) {
        cudaFuncAttributes fa;
        CUDA_CHECK(cudaFuncGetAttributes(&fa, kernel));
        have = fa.sharedSizeBytes + 1;
    }
    return have - 1;
}

// Per-engine device context.  Everything the backend needs to remember between calls lives here, nothing in
// process-global state: two engines on two devices (or on one) never see each other's scratch.
struct Ctx {
    int device = 0, sms = 0;
    // shared memory one block may use, static and dynamic together: by default, and with the opt-in of
    // cudaFuncAttributeMaxDynamicSharedMemorySize (49152 and 232448 bytes on an H100)
    size_t smem_block = 0, smem_optin = 0;
    cudaStream_t stream = nullptr;       // every kernel of this engine; created blocking, so work queued on the legacy
                                         // default stream (torch's default stream) stays ordered with it both ways
    cudaStream_t copy = nullptr;         // wire / dense DMA traffic (non-blocking; ordered by events)
    cudaEvent_t ev_wire = nullptr, ev_done = nullptr;
    bool profile = false;
    std::vector<cudaEvent_t> events;     // pairs recorded around obs-render launches
    size_t events_used = 0;
    // products of the last launch_obs_prepare
    float *mm_pad = nullptr; size_t mm_pad_n = 0; int mm_stride = 0;
    // per-observer headers of the render kernel
    int4 *obs_hdr = nullptr; size_t obs_hdr_n = 0;
    // slot-ordered observations (launch_obs_slots): the [A][S] slot -> row scratch (launch_action_mask_slots,
    // launch_mean_action_slots and launch_neighbours_slots use it too), and the render's count bound ([A + 1] words of
    // INT_MAX)
    int *obs_slot_row = nullptr; size_t obs_slot_row_n = 0;
    int *obs_slot_bound = nullptr; size_t obs_slot_bound_n = 0;
    // cudaFuncSetAttribute caches (per device: a context never changes device)
    struct ObsCfg { size_t smem = (size_t)-1; int ctas_per_sm = 1; } obs_cfg[12];
    int obs_last[8] = {0, 0, 0, 0, 0, 0, 0, 0};            // the last render launch (obs_launch_report)
    int step_last[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};     // the last step and cull launches (step_launch_report)
    unsigned *obs_deal = nullptr;        // [sms + 1] render chunk counters; zero between launches (the kernel resets them)
    ObsCfg state_cfg[2];                 // global_state_kernel<float>, <__half>: CTAs per SM (smem 0 once queried)
    int restore_ctas_per_sm = 0;         // restore_kernel (0: not queried yet)
    int *pin_done = nullptr; size_t pin_done_n = 0;         // pinned read-back of EngineDev::done
    int *pin_counts = nullptr; size_t pin_counts_n = 0;     // pinned read-back of EngineDev::off (clear_dead)
    cudaEvent_t ev_counts = nullptr;
    // wire path (host-buffer observations)
    WireMark *wire_slots = nullptr; size_t wire_slots_n = 0;         // [n_total][n_in] worst-case slots
    WireMark *wire_stream = nullptr; size_t wire_stream_n = 0;       // compacted marks
    WireHdr *wire_hdr = nullptr; size_t wire_hdr_n = 0;
    long long *wire_base = nullptr; size_t wire_base_n = 0;          // [n_chunks + 1] (device)
    int *wire_chunk_total = nullptr;
    // page-locked staging of the above
    WireHdr *h_wire_hdr = nullptr; size_t h_wire_hdr_n = 0;
    WireMark *h_wire_marks = nullptr; size_t h_wire_marks_n = 0;
    long long *h_wire_base = nullptr; size_t h_wire_base_n = 0;
    float *h_mm = nullptr; size_t h_mm_n = 0;
    std::vector<cudaEvent_t> wave_events;
    int waves_queued = 0;
    std::vector<cudaEvent_t> dma_events; size_t dma_head = 0, dma_tail = 0;
    // CUDA graphs (capture_begin / capture_end / graph_launch)
    bool capturing = false;
    std::vector<cudaGraphExec_t> graphs;
};

// Where `dyn` bytes of dynamic shared memory put a launch of `kernel` (attribute slot `slot`), its static shared memory
// added: 0 within the device's default per-block limit, 1 within the opt-in limit only, -1 beyond both.  *need: the total.
template <class K>
static int smem_band(const Ctx *c, int slot, K kernel, size_t dyn, size_t *need = nullptr) {
    const size_t total = static_smem(c->device, slot, kernel) + dyn;
    if (need) *need = total;
    return total <= c->smem_block ? 0 : total <= c->smem_optin ? 1 : -1;
}
// Ready `kernel` for a launch with `dyn` bytes of dynamic shared memory: the opt-in when it needs it.  Beyond the opt-in
// limit the process stops; the engine refuses such calls before they get here (smem_fits).
template <class K>
static void smem_prepare(const Ctx *c, int slot, K kernel, size_t dyn, const char *what) {
    size_t need;
    const int band = smem_band(c, slot, kernel, dyn, &need);
    if (band < 0) mg::fatal("%s: %zu bytes of shared memory, more than the %zu one block may use", what, need, c->smem_optin);
    if (band > 0) ensure_dynamic_smem(c->device, slot, kernel, dyn);
}

static void no_capture(const Ctx *c, const char *what) {
    if (c->capturing) mg::fatal("%s is not possible while a CUDA graph is being captured (run one un-captured step first so that "
                                "every buffer has its size)", what);
}

struct DeviceGuard {                     // every entry point runs on its context's device, whatever the caller selected
    explicit DeviceGuard(const Ctx *c) { int cur = -1; cudaGetDevice(&cur); if (cur != c->device) CUDA_CHECK(cudaSetDevice(c->device)); }
};

const char *name() { return "cuda-sm_90a"; }

#if defined(MG_PHASE_TIMING)
extern "C" __attribute__((visibility("default"))) void magent_b200_debug_phase_clocks(long long *out) {
    CUDA_CHECK(cudaMemcpyFromSymbol(out, mg::mg_phase_clock, sizeof(long long) * 8 * 32));
}
#endif

int device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

Ctx *create(int device, std::string *err) {
    int n = device_count();
    if (n <= 0) { if (err) *err = "cudaGetDeviceCount found no device"; return nullptr; }
    if (device < 0) {
        if (cudaGetDevice(&device) != cudaSuccess) device = 0;
    }
    if (device >= n) { if (err) *err = "device_id out of range"; return nullptr; }
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) { if (err) *err = cudaGetErrorString(e); return nullptr; }
    cudaDeviceProp prop;
    CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    Ctx *c = new Ctx();
    c->device = device;
    c->sms = prop.multiProcessorCount;
    c->smem_block = prop.sharedMemPerBlock;
    c->smem_optin = prop.sharedMemPerBlockOptin;
    CUDA_CHECK(cudaStreamCreate(&c->stream));
    CUDA_CHECK(cudaStreamCreateWithFlags(&c->copy, cudaStreamNonBlocking));
    CUDA_CHECK(cudaEventCreateWithFlags(&c->ev_wire, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&c->ev_counts, cudaEventDisableTiming));
    CUDA_CHECK(cudaMalloc(&c->obs_deal, (c->sms + 1) * sizeof(unsigned)));
    CUDA_CHECK(cudaMemset(c->obs_deal, 0, (c->sms + 1) * sizeof(unsigned)));
    return c;
}
void destroy(Ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    for (cudaGraphExec_t e : c->graphs) if (e) cudaGraphExecDestroy(e);
    cudaStreamSynchronize(c->stream); cudaStreamSynchronize(c->copy);
    for (cudaEvent_t e : c->events) cudaEventDestroy(e);
    for (cudaEvent_t e : c->wave_events) cudaEventDestroy(e);
    for (cudaEvent_t e : c->dma_events) cudaEventDestroy(e);
    cudaEventDestroy(c->ev_wire); cudaEventDestroy(c->ev_done);
    cudaFree(c->mm_pad); cudaFree(c->obs_hdr); cudaFree(c->obs_deal); cudaFree(c->obs_slot_row); cudaFree(c->obs_slot_bound);
    cudaFree(c->wire_slots); cudaFree(c->wire_stream); cudaFree(c->wire_hdr); cudaFree(c->wire_base); cudaFree(c->wire_chunk_total);
    cudaEventDestroy(c->ev_counts); cudaFreeHost(c->pin_counts);
    cudaFreeHost(c->pin_done); cudaFreeHost(c->h_wire_hdr); cudaFreeHost(c->h_wire_marks); cudaFreeHost(c->h_wire_base); cudaFreeHost(c->h_mm);
    cudaStreamDestroy(c->stream); cudaStreamDestroy(c->copy);
    delete c;
}
int device_of(const Ctx *c) { return c->device; }
int sm_count(const Ctx *c) { return c->sms; }
void *stream_handle(const Ctx *c) { return (void *)c->stream; }

void *dmalloc(Ctx *c, size_t bytes) { no_capture(c, "a device allocation"); DeviceGuard g(c); void *p = nullptr; CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 16)); return p; }
void dfree(Ctx *c, void *p) { if (p) { DeviceGuard g(c); cudaFree(p); } }
void dmemset(Ctx *c, void *p, int byte, size_t bytes) { DeviceGuard g(c); CUDA_CHECK(cudaMemsetAsync(p, byte, bytes, c->stream)); }
void h2d(Ctx *c, void *dst, const void *src, size_t bytes) {
    if (!bytes) return;
    no_capture(c, "a blocking host-to-device copy");
    DeviceGuard g(c);
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}
void d2h(Ctx *c, void *dst, const void *src, size_t bytes) {
    if (!bytes) return;
    no_capture(c, "a blocking device-to-host copy");
    DeviceGuard g(c);
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}
void d2d(Ctx *c, void *dst, const void *src, size_t bytes) {
    if (!bytes) return;
    DeviceGuard g(c);
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c->stream));
}
void *host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void host_free(void *p) { if (p) cudaFreeHost(p); }
bool host_register(void *p, size_t bytes) {
    if (cudaHostRegister(p, bytes, cudaHostRegisterPortable) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}
void host_unregister(void *p) { if (cudaHostUnregister(p) != cudaSuccess) cudaGetLastError(); }
bool is_device_ptr(const void *p) {
    if (!p) return false;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}
bool is_pinned_host_ptr(const void *p) {
    if (!p) return false;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}
void sync(Ctx *c) { no_capture(c, "a synchronisation"); DeviceGuard g(c); CUDA_CHECK(cudaStreamSynchronize(c->stream)); CUDA_CHECK(cudaStreamSynchronize(c->copy)); }
long long launch_count() { return g_launches.load(); }
void profile_enable(Ctx *c, bool on) { c->profile = on; c->events_used = 0; }
static void profile_pair(Ctx *c, cudaEvent_t *e0, cudaEvent_t *e1) {
    if (c->events_used + 2 > c->events.size()) {
        for (int i = 0; i < 64; ++i) { cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); c->events.push_back(e); }
    }
    *e0 = c->events[c->events_used]; *e1 = c->events[c->events_used + 1];
    c->events_used += 2;
}
// total device time of the obs-render launches recorded since profile_enable(true); no sync was added
// to the timed region: the events are read here, after the fact
void profile_read(Ctx *c, double *ms, long long *n) {
    DeviceGuard g(c);
    double total = 0.0;
    for (size_t i = 0; i + 1 < c->events_used; i += 2) {
        CUDA_CHECK(cudaEventSynchronize(c->events[i + 1]));
        float t = 0;
        CUDA_CHECK(cudaEventElapsedTime(&t, c->events[i], c->events[i + 1]));
        total += t;
    }
    *ms = total; *n = (long long)(c->events_used / 2);
}

bool capture_begin(Ctx *c) {
    DeviceGuard guard(c);
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    CUDA_CHECK(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
    c->capturing = true;
    return true;
}
int capture_end(Ctx *c) {
    DeviceGuard guard(c);
    cudaGraph_t g = nullptr;
    c->capturing = false;
    CUDA_CHECK(cudaStreamEndCapture(c->stream, &g));
    cudaGraphExec_t exec = nullptr;
    CUDA_CHECK(cudaGraphInstantiate(&exec, g, 0));
    CUDA_CHECK(cudaGraphDestroy(g));
    c->graphs.push_back(exec);
    return (int)c->graphs.size() - 1;
}
bool capturing(const Ctx *c) { return c->capturing; }
void graph_launch(Ctx *c, int id) {
    DeviceGuard guard(c);
    if (id < 0 || id >= (int)c->graphs.size() || !c->graphs[id]) mg::fatal("invalid graph id %d", id);
    CUDA_CHECK(cudaGraphLaunch(c->graphs[id], c->stream));
}
void graph_destroy_all(Ctx *c) {
    DeviceGuard guard(c);
    for (cudaGraphExec_t e : c->graphs) if (e) cudaGraphExecDestroy(e);
    c->graphs.clear();
}

static void post_launch(const char *what) {
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) mg::fatal("kernel launch failed (%s): %s", what, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------
// team contexts
__device__ __forceinline__ int block_excl_scan(int v, int &total) {
    __shared__ int warp_sums[32];
    __shared__ int block_total;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int w = lane < nw ? warp_sums[lane] : 0;
        int wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += t;
        }
        if (lane < nw) warp_sums[lane] = wi - w;          // exclusive prefix of warp totals
        if (lane == 31) block_total = wi;
    }
    __syncthreads();
    int excl = incl - v + warp_sums[wid];
    total = block_total;
    __syncthreads();
    return excl;
}

struct CtaCtx {
    GroupEnum *enum_smem;
    MG_HD GroupEnum *enums() { return enum_smem; }
    MG_HD bool is_cta_leader() const {
#if defined(__CUDA_ARCH__)
        return threadIdx.x == 0;
#else
        return true;
#endif
    }
    MG_HD void sync_cta() {
#if defined(__CUDA_ARCH__)
        __syncthreads();
#endif
    }
    int *flag_smem;
    MG_HD int *flags(ArenaHdr *) { return flag_smem; }
    int cnt[MG_N_COUNTERS];
    MG_HD void add_count(const EngineDev &, int kind, long long v) { cnt[kind] += (int)v; }
    // warp-reduced, then one shared-memory add per warp and ONE global atomic per counter per arena-step (the 8 counters
    // are 8 addresses for the whole GPU: a global atomic per warp made them a hot spot)
    int *cnt_smem;                      // [MG_N_COUNTERS], zero between arena-steps
    MG_HD void flush_counts(const EngineDev &E) {
#if defined(__CUDA_ARCH__)
#pragma unroll
        for (int k = 0; k < MG_N_COUNTERS; ++k) {
            int v = cnt[k];
            cnt[k] = 0;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (v && (threadIdx.x & 31) == 0) atomicAdd(&cnt_smem[k], v);
        }
        __syncthreads();
        if (threadIdx.x < MG_N_COUNTERS) {
            const int v = cnt_smem[threadIdx.x];
            cnt_smem[threadIdx.x] = 0;
            if (v) atomicAdd((unsigned long long *)&E.counters[threadIdx.x], (unsigned long long)v);
        }
#endif
    }
    MG_HD int tid() const {
#if defined(__CUDA_ARCH__)
        return threadIdx.x;
#else
        return 0;
#endif
    }
    MG_HD int nth() const {
#if defined(__CUDA_ARCH__)
        return blockDim.x;
#else
        return 1;
#endif
    }
    MG_HD void sync() {
#if defined(__CUDA_ARCH__)
        __syncthreads();
#endif
    }
    template <class P, class Em>
    MG_HD int scan(int n, P pred, Em emit) {
#if defined(__CUDA_ARCH__)
        int running = 0;
        for (int tile = 0; tile < n; tile += blockDim.x) {
            int i = tile + threadIdx.x;
            int p = i < n ? pred(i) : 0;
            int tot;
            int ex = block_excl_scan(p, tot);
            if (p) emit(i, running + ex);
            running += tot;
        }
        return running;
#else
        return 0;
#endif
    }
};

struct GridCtx {
    GroupEnum *enum_smem;
    MG_HD GroupEnum *enums() { return enum_smem; }
    MG_HD bool is_cta_leader() const {
#if defined(__CUDA_ARCH__)
        return threadIdx.x == 0;
#else
        return true;
#endif
    }
    MG_HD void sync_cta() {
#if defined(__CUDA_ARCH__)
        __syncthreads();
#endif
    }
    int *scratch;       // [2][4096]
    int parity;
    MG_HD int *flags(ArenaHdr *hdr) { return hdr->changed; }
    int cnt[MG_N_COUNTERS];
    MG_HD void add_count(const EngineDev &, int kind, long long v) { cnt[kind] += (int)v; }
    // one warp-reduced atomic per counter per warp, once per arena-step
    MG_HD void flush_counts(const EngineDev &E) {
#if defined(__CUDA_ARCH__)
#pragma unroll
        for (int k = 0; k < MG_N_COUNTERS; ++k) {
            int v = cnt[k];
            cnt[k] = 0;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (v && (threadIdx.x & 31) == 0) atomicAdd((unsigned long long *)&E.counters[k], (unsigned long long)v);
        }
#endif
    }
    MG_HD int tid() const {
#if defined(__CUDA_ARCH__)
        return blockIdx.x * blockDim.x + threadIdx.x;
#else
        return 0;
#endif
    }
    MG_HD int nth() const {
#if defined(__CUDA_ARCH__)
        return gridDim.x * blockDim.x;
#else
        return 1;
#endif
    }
    MG_HD void sync() {
#if defined(__CUDA_ARCH__)
        cg::this_grid().sync();
#endif
    }
    template <class P, class Em>
    MG_HD int scan(int n, P pred, Em emit) {
#if defined(__CUDA_ARCH__)
        // contiguous chunk per CTA keeps the emitted order == index order
        const int nb = gridDim.x, bid = blockIdx.x;
        const int L = (n + nb - 1) / nb;
        const int lo = min(n, bid * L), hi = min(n, lo + L);
        int cnt = 0;
        for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) cnt += pred(i);
        int cta_total;
        block_excl_scan(cnt, cta_total);
        int *sc = scratch + (parity & 1) * 4096;
        parity ^= 1;
        if (threadIdx.x == 0) sc[bid] = cta_total;
        cg::this_grid().sync();
        int below = 0, all = 0;
        for (int b = threadIdx.x; b < nb; b += blockDim.x) { int v = sc[b]; all += v; if (b < bid) below += v; }
        int base, total;
        block_excl_scan(below, base);
        block_excl_scan(all, total);
        int running = base;
        for (int tile = lo; tile < hi; tile += blockDim.x) {
            int i = tile + threadIdx.x;
            int p = i < hi ? pred(i) : 0;
            int tot;
            int ex = block_excl_scan(p, tot);
            if (p) emit(i, running + ex);
            running += tot;
        }
        return total;
#else
        return 0;
#endif
    }
};

__device__ __forceinline__ void load_engine(EngineDev *sE, const EngineDev *gE) {
    const int *src = (const int *)gE;
    int *dst = (int *)sE;
    for (int i = threadIdx.x; i < (int)(sizeof(EngineDev) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

constexpr int STEP_THREADS = 1024;      // launch bound; the launch picks 256..1024 (step_block_size)
constexpr int GRID_THREADS = 512;       // block size of the cooperative whole-grid team

// bytes of per-arena step scratch (the arrays step_scratch_to_smem() re-homes)
static size_t step_scratch_bytes(int cap_total, int max_body) {
    return (size_t)cap_total * (9 * 4 + 4 * (size_t)max_body) + (((size_t)cap_total + 15) & ~(size_t)15);
}

// Point the scratch arrays of the CTA's private EngineDev copy at dynamic shared memory.  One CTA works on one
// arena at a time, so the scratch needs no per-arena stride (scratch_stride = 0): every dependent load of the
// relaxation / list walks becomes an LDS instead of an L2/HBM round trip.  The shuffle scratch (dead after
// phase_rank_target) shares storage with the mover scratch (first written in phase_attack_apply_starve):
// 41 B/agent => two 2x1000-agent arenas per SM.
__device__ __forceinline__ void step_scratch_to_smem(EngineDev *sE, unsigned char *base) {
    const size_t n = (size_t)sE->cap_total;
    int *p = (int *)base;
    sE->att_rank = p; p += n;  sE->tgt = p; p += n;       sE->in_head = p; p += n;  sE->in_next = p; p += n;
    sE->death = p; p += n;
    sE->mv_nx = p; sE->jv = p; p += n;
    sE->mv_ny = p; sE->sh_head = p; p += n;
    sE->mv_key = (unsigned *)p; sE->sh_next = p; p += n;
    sE->hp_fin = (float *)p; sE->att_agent = p; p += n;
    sE->cl_next = p; sE->sh_first = p; p += n * sE->max_body;
    sE->mv_state = (unsigned char *)p;
    sE->scratch_stride = 0;
}

__global__ void __launch_bounds__(STEP_THREADS) step_kernel_cta(const EngineDev *gE, StepArgs S, int scratch_in_smem) {
    extern __shared__ __align__(16) unsigned char step_smem[];
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    if (scratch_in_smem) {
        if (threadIdx.x == 0) step_scratch_to_smem(&sE, step_smem);
        __syncthreads();
    }
    __shared__ int relax_flags[3];
    __shared__ int counter_sums[MG_N_COUNTERS];
    __shared__ GroupEnum enum_store[2];
    if (threadIdx.x < MG_N_COUNTERS) counter_sums[threadIdx.x] = 0;
    CtaCtx c;
    c.flag_smem = relax_flags;
    c.cnt_smem = counter_sums;
    c.enum_smem = enum_store;
    for (int k = 0; k < MG_N_COUNTERS; ++k) c.cnt[k] = 0;
    for (int a = blockIdx.x; a < sE.A; a += gridDim.x) run_step(c, sE, S, a);
}

__global__ void __launch_bounds__(STEP_THREADS) step_kernel_grid(const EngineDev *gE, StepArgs S) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    __shared__ GroupEnum enum_store[2];
    GridCtx c;
    c.scratch = sE.team_scratch;
    c.parity = 0;
    c.enum_smem = enum_store;
    for (int k = 0; k < MG_N_COUNTERS; ++k) c.cnt[k] = 0;
    for (int a = 0; a < sE.A; ++a) run_step(c, sE, S, a);
}

__global__ void __launch_bounds__(STEP_THREADS) cull_kernel_cta(const EngineDev *gE, unsigned curmask) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    CtaCtx c;
    c.flag_smem = nullptr;
    c.cnt_smem = nullptr;
    c.enum_smem = nullptr;
    for (int a = blockIdx.x; a < sE.A; a += gridDim.x) run_cull(c, sE, curmask, a);
}

__global__ void __launch_bounds__(STEP_THREADS) cull_kernel_grid(const EngineDev *gE, unsigned curmask) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    GridCtx c;
    c.scratch = sE.team_scratch;
    c.parity = 0;
    c.enum_smem = nullptr;
    for (int a = 0; a < sE.A; ++a) run_cull(c, sE, curmask, a);
}

static const int GRID_MODE_THRESHOLD = 32768;    // agents per arena above which the whole grid teams up

// {mode (0 CTA per arena, 1 whole-grid team), grid, threads, dynamic smem bytes, scratch in smem} (step_launch_report)
static void record_launch(int *out, int mode, int grid, int threads, int smem, int scratch_in_smem) {
    const int report[5] = {mode, grid, threads, smem, scratch_in_smem};
    memcpy(out, report, sizeof report);
}

// CTA-per-arena block size: the phases are latency-bound loops over the arena's agents, so with many
// arenas we want many (small) CTAs resident per SM; with few arenas the single CTA should be wide.
static int step_block_size(int sms, int arenas, int max_agents) {
    if (arenas >= 2 * sms) return 256;
    if (max_agents >= 768) return 1024;
    return max_agents >= 384 ? 512 : 256;
}

static int coop_grid(const Ctx *c, const void *kernel) {
    int per_sm = 0;
    CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, GRID_THREADS, 0));
    if (per_sm < 1) mg::fatal("cooperative kernel does not fit on an SM");
    int g = per_sm * c->sms;
    return g > 4096 ? 4096 : g;
}

void launch_step(Ctx *c, const EngineDev *dE, const EngineDev &hE, const StepArgs &S, int max_agents) {
    DeviceGuard guard(c);
    const int g_sms = c->sms;
    if (max_agents > GRID_MODE_THRESHOLD) {
        int grid = coop_grid(c, (const void *)step_kernel_grid);
        StepArgs s = S;
        void *args[] = {(void *)&dE, (void *)&s};
        CUDA_CHECK(cudaLaunchCooperativeKernel((const void *)step_kernel_grid, dim3(grid), dim3(GRID_THREADS), args, 0, c->stream));
        post_launch("step_kernel_grid");
        record_launch(c->step_last, 1, grid, GRID_THREADS, 0, 0);
    } else {
        // scratch in shared memory whenever one arena's scratch fits: fewer, wider CTAs (latency per phase drops
        // from HBM/L2 round trips to LDS), and the concurrently active arenas stay L2-resident
        const size_t sbytes = step_scratch_bytes(hE.cap_total, hE.max_body);
        static const int smem_pref = getenv("MAGENT_B200_STEP_SMEM") ? atoi(getenv("MAGENT_B200_STEP_SMEM")) : -1;
        const bool in_smem = sbytes <= 200 * 1024 && smem_pref != 0;
        int threads = step_block_size(g_sms, hE.A, max_agents);
        size_t smem = 0;
        if (in_smem) {
            smem = sbytes;
            // few arenas: one wide CTA each; many arenas: narrower CTAs so that two fit on an SM and overlap
            threads = max_agents >= 768 ? (hE.A > g_sms ? 512 : 1024) : (max_agents >= 384 ? 512 : 256);
            ensure_dynamic_smem(c->device, ATTR_STEP, step_kernel_cta, smem);
        }
        // measurement knob: MAGENT_B200_STEP_THREADS=256..1024 overrides the block size choice above
        static const int threads_pref = getenv("MAGENT_B200_STEP_THREADS") ? atoi(getenv("MAGENT_B200_STEP_THREADS")) : 0;
        if (threads_pref >= 32 && threads_pref <= STEP_THREADS) threads = threads_pref & ~31;
        int per_sm = 1;
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, step_kernel_cta, threads, smem));
        if (per_sm < 1) per_sm = 1;
        int grid = hE.A < per_sm * g_sms ? hE.A : per_sm * g_sms;
        step_kernel_cta<<<grid, threads, smem, c->stream>>>(dE, S, in_smem ? 1 : 0);
        post_launch("step_kernel_cta");
        record_launch(c->step_last, 0, grid, threads, (int)smem, in_smem ? 1 : 0);
    }
}

void launch_cull(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int max_agents) {
    DeviceGuard guard(c);
    const int g_sms = c->sms;
    if (max_agents > GRID_MODE_THRESHOLD) {
        int grid = coop_grid(c, (const void *)cull_kernel_grid);
        void *args[] = {(void *)&dE, (void *)&curmask};
        CUDA_CHECK(cudaLaunchCooperativeKernel((const void *)cull_kernel_grid, dim3(grid), dim3(GRID_THREADS), args, 0, c->stream));
        post_launch("cull_kernel_grid");
        record_launch(c->step_last + 5, 1, grid, GRID_THREADS, 0, 0);
    } else {
        int grid = hE.A < 8 * g_sms ? hE.A : 8 * g_sms;
        // measurement knob: MAGENT_B200_CULL_THREADS overrides the block size
        static const int cull_pref = getenv("MAGENT_B200_CULL_THREADS") ? atoi(getenv("MAGENT_B200_CULL_THREADS")) : 0;
        // the compaction is a chain of block scans (three barriers per tile of blockDim agents): 512 threads for arenas of
        // ~1000 agents per group
        int threads = max_agents >= 768 ? 512 : step_block_size(g_sms, hE.A, max_agents);
        if (cull_pref >= 32 && cull_pref <= STEP_THREADS) threads = cull_pref & ~31;
        cull_kernel_cta<<<grid, threads, 0, c->stream>>>(dE, curmask);
        post_launch("cull_kernel_cta");
        record_launch(c->step_last + 5, 0, grid, threads, 0, 0);
    }
}

// off[g][0..A] = exclusive prefix of n[g][0..A-1], by one whole CTA
__device__ __forceinline__ void offsets_group(const EngineDev *gE, int g) {
    const int A = gE->A;
    const int *n = gE->n + (size_t)g * A;
    int *off = gE->off + (size_t)g * (A + 1);
    int running = 0;
    for (int tile = 0; tile < A; tile += blockDim.x) {
        int a = tile + threadIdx.x;
        int v = a < A ? n[a] : 0;
        int tot;
        int ex = block_excl_scan(v, tot);
        if (a < A) off[a] = running + ex;
        running += tot;
    }
    if (threadIdx.x == 0) off[A] = running;
}

// one CTA per group
__global__ void __launch_bounds__(1024) offsets_kernel(const EngineDev *gE) { offsets_group(gE, blockIdx.x); }

void launch_offsets(Ctx *c, const EngineDev *dE, const EngineDev &hE) {
    DeviceGuard guard(c);
    offsets_kernel<<<hE.G, 1024, 0, c->stream>>>(dE);
    post_launch("offsets_kernel");
}

// arena of the idx-th agent in the concatenation of group g
__device__ __forceinline__ int locate_arena(const int *off, int A, int idx) {
    int lo = 0, hi = A;                 // invariant: off[lo] <= idx < off[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (off[mid] <= idx) lo = mid; else hi = mid;
    }
    return lo;
}

// One thread per agent, CTAs dealt per arena (blockIdx says which arena: no search).  `n_total` is the host's count, which
// may still be the one from before the last cull (an upper bound): the device-side offsets decide.
__global__ void __launch_bounds__(256) info_kernel(const EngineDev *gE, unsigned curmask, int kind, int g,
                                                   void *buf, int n_total, int chunks_per_arena) {
    const EngineDev &E = *gE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = E.grp[g].soa[(curmask >> g) & 1u];
    const int a = blockIdx.x / chunks_per_arena;
    const int i = (blockIdx.x - a * chunks_per_arena) * blockDim.x + threadIdx.x;
    const int o0 = off[a];
    const int o = o0 + i;
    if (i < off[a + 1] - o0 && o < n_total) {
        const long gi = (long)a * E.grp[g].cap + i;
        switch (kind) {
            case INFO_ID: ((int *)buf)[o] = s.id[gi]; break;
            case INFO_POS: ((int2 *)buf)[o] = make_int2(s.x[gi], s.y[gi]); break;
            case INFO_ALIVE: ((unsigned char *)buf)[o] = (s.flags[gi] & FLAG_DEAD) ? 0 : 1; break;
            case INFO_REWARD: ((float *)buf)[o] = s.next_reward[gi] + E.hdr[a].grp_reward[g]; break;
            case INFO_HP: ((float *)buf)[o] = s.hp[gi]; break;
            case INFO_ACTION_SCATTER: s.act[gi] = ((const int *)buf)[o]; break;
        }
    }
}

void launch_info(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int kind, int group, void *buf, int n_total) {
    DeviceGuard guard(c);
    const int cap = hE.grp[group].cap;
    const int threads = cap >= 256 ? 256 : ((cap + 31) & ~31);
    const int cpa = (cap + threads - 1) / threads;
    info_kernel<<<(unsigned)((size_t)hE.A * cpa), threads, 0, c->stream>>>(dE, curmask, kind, group, buf, n_total, cpa);
    post_launch("info_kernel");
}

__global__ void __launch_bounds__(256) random_actions_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                             unsigned long long seed, int n_total, int chunks_per_arena) {
    const EngineDev &E = *gE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = E.grp[g].soa[(curmask >> g) & 1u];
    const unsigned na = (unsigned)E.grp[g].n_action;
    // the device-side step counter rides in the seed: a replayed CUDA graph (same kernel arguments) still draws fresh actions
    seed += (unsigned long long)E.counters[CNT_STEPS] * 0xA24BAED4963EE407ull;
    const int a = blockIdx.x / chunks_per_arena;
    const int i = (blockIdx.x - a * chunks_per_arena) * blockDim.x + threadIdx.x;
    const int o0 = off[a];
    const int o = o0 + i;
    if (i < off[a + 1] - o0 && o < n_total)
        s.act[(long)a * E.grp[g].cap + i] = (int)((splitmix64(seed ^ ((unsigned long long)o * 0xD1342543DE82EF95ull)) >> 33) % na);
}

void launch_random_actions(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group,
                           unsigned long long seed, int n_total) {
    DeviceGuard guard(c);
    const int cap = hE.grp[group].cap;
    const int threads = cap >= 256 ? 256 : ((cap + 31) & ~31);
    const int cpa = (cap + threads - 1) / threads;
    random_actions_kernel<<<(unsigned)((size_t)hE.A * cpa), threads, 0, c->stream>>>(dE, curmask, group, seed, n_total, cpa);
    post_launch("random_actions_kernel");
}

// ------------------------------------------------------------------------------------------------
// legal-action mask (magent_b200_get_action_mask) and legal draws (magent_b200_random_legal_actions): mask_phases.h
// action_legal for every (agent, action) of a group.  CTAs are dealt per arena like info_kernel (blockIdx says which
// arena, the device-side offsets decide how many agents it has, the host's count is only an upper bound).  A CTA owns
// MASK_THREADS consecutive agents.  In the mask kernel a warp takes 32 of them: lane j loads agent j's own fields
// (coalesced), then the warp visits its agents one after the other with the lanes spread over the actions, every lane
// deciding one action per 32 from one to a handful of cells of the arena's `occ` plane (an L2 hit: a plane is
// 40-200 KB).
constexpr int MASK_THREADS = 256;

struct MaskWarp {                    // the agents of one warp: lane j holds agent i0 + j
    int a, g, o0, c0, i0, cnt;       // arena, group, the arena's first ABI row, first agent of the CTA / of the warp
    MaskAgent mine;
    __device__ __forceinline__ MaskAgent agent(int j) const {
        MaskAgent m;
        m.x = __shfl_sync(0xffffffffu, mine.x, j); m.y = __shfl_sync(0xffffffffu, mine.y, j);
        m.dir = __shfl_sync(0xffffffffu, mine.dir, j); m.code = code_make(g, i0 + j);
        m.flags = (unsigned char)__shfl_sync(0xffffffffu, (int)mine.flags, j);
        return m;
    }
};
// returns the number of agents of the CTA (the same in every thread of it)
__device__ __forceinline__ int mask_warp_setup(const EngineDev &E, unsigned curmask, int g, int n_total, int chunks_per_arena,
                                               MaskWarp &w) {
    const int *off = E.off + (size_t)g * (E.A + 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    w.g = g;
    w.a = blockIdx.x / chunks_per_arena;
    const int c0 = w.c0 = (blockIdx.x - w.a * chunks_per_arena) * MASK_THREADS;
    w.o0 = off[w.a];
    int cta_cnt = min(MASK_THREADS, off[w.a + 1] - w.o0 - c0);
    cta_cnt = min(cta_cnt, n_total - (w.o0 + c0));               // never beyond the caller's buffer
    w.i0 = c0 + 32 * warp;
    w.cnt = min(32, cta_cnt - 32 * warp);
    w.mine.x = w.mine.y = 0; w.mine.dir = DIR_NORTH; w.mine.code = 0; w.mine.flags = FLAG_DEAD;
    if (lane < w.cnt) w.mine = mask_agent(E, curmask, w.a, g, w.i0 + lane);
    return cta_cnt;
}

// The `total` bytes a CTA composed at `rows` (mask_smem + the 16-byte phase of `dst`) into `dst`: a byte head up to the
// first 16-byte boundary, 16 bytes per thread in the body, a byte tail.  Every thread of the CTA calls it after a barrier.
__device__ __forceinline__ void mask_rows_store(unsigned char *dst, const unsigned char *rows, int total) {
    const int shift = (int)((size_t)dst & 15);
    const int head = min(total, (16 - shift) & 15);
    const int body = (total - head) >> 4;
    for (int q = threadIdx.x; q < head; q += MASK_THREADS) dst[q] = rows[q];
    for (int q = threadIdx.x; q < body; q += MASK_THREADS) ((uint4 *)(dst + head))[q] = ((const uint4 *)(rows + head))[q];
    for (int q = head + (body << 4) + threadIdx.x; q < total; q += MASK_THREADS) dst[q] = rows[q];
}

__global__ void __launch_bounds__(MASK_THREADS) action_mask_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                                  unsigned char *out, int n_total, int chunks_per_arena) {
    __shared__ EngineDev sE;
    extern __shared__ __align__(16) unsigned char mask_smem[];
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    MaskWarp w;
    const int cta_cnt = mask_warp_setup(E, curmask, g, n_total, chunks_per_arena, w);
    if (cta_cnt <= 0) return;
    const int na = E.grp[g].n_action, lane = threadIdx.x & 31;
    // the CTA's rows are one contiguous byte range of the output: composed in shared memory at the same offset from a
    // 16-byte boundary as their destination, so that the body of the copy below is 16 bytes per thread on both sides
    unsigned char *dst = out + (size_t)(w.o0 + w.c0) * na;
    const int shift = (int)((size_t)dst & 15);
    unsigned char *rows = mask_smem + shift;
    const int *occ = E.occ + (long)w.a * E.W * E.H;
    for (int j = 0; j < w.cnt; ++j) {
        const MaskAgent m = w.agent(j);
        unsigned char *row = rows + (size_t)(w.i0 - w.c0 + j) * na;
        for (int k = lane; k < na; k += 32) row[k] = action_legal(E, curmask, w.a, occ, g, m, k) ? 1 : 0;
    }
    __syncthreads();
    mask_rows_store(dst, rows, cta_cnt * na);
}

// The byte mask is never materialised: one thread per agent counts its legal actions, draws r = legal_draw(...) below
// that count and walks to the r-th legal action in ascending action order.  The walk decides the same cells again; they
// are L1 hits by then.  No legal action (dead, or an absorbed absorber with nothing to attack): action 0, which the step
// ignores for such an agent.
__global__ void __launch_bounds__(MASK_THREADS) random_legal_actions_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                                           unsigned long long seed, int n_total,
                                                                           int chunks_per_arena) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const int a = blockIdx.x / chunks_per_arena;
    const int i = (blockIdx.x - a * chunks_per_arena) * MASK_THREADS + threadIdx.x;
    const int o0 = off[a];
    const int o = o0 + i;
    if (i >= off[a + 1] - o0 || o >= n_total) return;
    const int na = E.grp[g].n_action;
    const int *occ = E.occ + (long)a * E.W * E.H;
    const MaskAgent m = mask_agent(E, curmask, a, g, i);
    int n_legal = 0;
    for (int k = 0; k < na; ++k) n_legal += action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
    int act = 0;
    if (n_legal > 0) {
        int r = legal_draw(seed, E.counters[CNT_STEPS], o, n_legal);
        for (; r >= 0; ++act) r -= action_legal(E, curmask, a, occ, g, m, act) ? 1 : 0;
        --act;
    }
    cur_soa(E, curmask, g).act[gidx(E, a, g, i)] = act;
}

static int mask_chunks_per_arena(const EngineDev &hE, int group) { return (hE.grp[group].cap + MASK_THREADS - 1) / MASK_THREADS; }
// dynamic shared memory of both mask kernels: MASK_THREADS rows and the 16 bytes of the store's alignment shift
static size_t mask_dyn_smem(const EngineDev &hE, int group) { return (size_t)MASK_THREADS * hE.grp[group].n_action + 16; }

void launch_action_mask(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group, unsigned char *out,
                        int n_total) {
    DeviceGuard guard(c);
    const size_t smem = mask_dyn_smem(hE, group);
    smem_prepare(c, ATTR_MASK, action_mask_kernel, smem, "action_mask_kernel");
    const int cpa = mask_chunks_per_arena(hE, group);
    action_mask_kernel<<<(unsigned)((size_t)hE.A * cpa), MASK_THREADS, smem, c->stream>>>(dE, curmask, group, out, n_total, cpa);
    post_launch("action_mask_kernel");
}

void launch_random_legal_actions(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group,
                                 unsigned long long seed, int n_total) {
    DeviceGuard guard(c);
    const int cpa = mask_chunks_per_arena(hE, group);
    random_legal_actions_kernel<<<(unsigned)((size_t)hE.A * cpa), MASK_THREADS, 0, c->stream>>>(dE, curmask, group, seed, n_total, cpa);
    post_launch("random_legal_actions_kernel");
}

// ------------------------------------------------------------------------------------------------
// mean neighbour action (magent_b200_get_mean_action): nbr_phases.h for every observer of a group.  CTAs are dealt per
// arena like action_mask_kernel (blockIdx says which arena, the device-side offsets decide how many observers it has,
// the host's count is only an upper bound).  A CTA owns MEAN_OBS consecutive observers; warp w takes observers w, w + 8,
// ... of them, one at a time, after its lanes have loaded all of their own fields at once.  The lanes stride over the
// observer's in-range view cells through the CTA's view LUT (four in turn_mode, one per heading), and every lane issues
// the `kind`-byte loads of MEAN_UNROLL cells before it looks at any of them, so the cell loads of an observer do not
// wait on one another.  Only a cell whose byte shows group `of` (about 5 % of battle's cells) goes on to `occ`, the
// footprint test of longer bodies and the neighbour's action; the counts land in the warp's shared-memory histogram of
// n_action(of) ints.  The pad of the planes covers every view window in every heading: no bounds check on the bytes.
constexpr int MEAN_THREADS = 256, MEAN_OBS = 128, MEAN_UNROLL = 4;
constexpr int MEAN_WARPS = MEAN_THREADS / 32;
static_assert(MEAN_OBS / MEAN_WARPS <= 32, "a warp's observers are loaded one per lane");
// The kernel is latency-bound (a kind -> occ -> act chain per observer), so resident warps matter: five CTAs per SM
// leave it 44 registers without spills (58 unbounded, four CTAs; six CTAs spill).  DESIGN.md §5 has the numbers.

// Who observer v of a CTA of the mean-action and neighbours kernels is, by a compile-time policy.  Rows (SLOTS false:
// mean_action_kernel, neighbours_kernel): row v of arena a in the group's order.  Slots (SLOTS true: the *_slots kernels):
// slot v of arena a, whose row slot_row (arena a's [S] block of slots_kernel's map) names; a vacant slot loads as the
// dead placeholder, which takes the dead observer's path (zero row, no neighbours).  o0 is the arena's first row.  A
// slot's lane keeps its row in arena i (< 2^24, code_index), its heading and its dead bit in one word, mine.code =
// i << 8 | dir << 1 | dead: the slot's cell code has to be held through the walk, where a row's is recomputed from v,
// and a lane word less keeps neighbours_slots_kernel free of spills at five CTAs per SM.
template <bool SLOTS>
__device__ __forceinline__ void nbr_cta_load(const EngineDev &E, unsigned curmask, int a, int g, int o0,
                                             const int *slot_row, int v, NbrObserver &mine) {
    if (!SLOTS) { mine = nbr_observer(E, curmask, a, g, v); return; }
    const int r = slot_row[v];
    if (r < 0) { mine.code = FLAG_DEAD; return; }
    mine = nbr_observer(E, curmask, a, g, r - o0);
    mine.code = (r - o0) << 8 | mine.dir << 1 | (mine.flags & FLAG_DEAD);
}
// the heading, cell code (which nbr_at and nbr_nearest_at exclude) and flags of observer v, loaded by lane u of the warp
template <bool SLOTS>
__device__ __forceinline__ void nbr_cta_take(int g, int v, const NbrObserver &mine, int u, NbrObserver &o) {
    if (SLOTS) {
        const int w = __shfl_sync(0xffffffffu, mine.code, u);
        o.dir = (w >> 1) & 3; o.code = code_make(g, (int)((unsigned)w >> 8)); o.flags = (unsigned char)(w & FLAG_DEAD);
        return;
    }
    o.dir = __shfl_sync(0xffffffffu, mine.dir, u); o.code = code_make(g, v);
    o.flags = (unsigned char)__shfl_sync(0xffffffffu, (int)mine.flags, u);
}

// One CTA of the mean-action kernels: observers c0 .. c0 + cta_cnt - 1 of arena a (nbr_cta_load), the row of observer v
// written at out0 + v.  The view LUT and the warps' histograms live in `smem`.
template <bool SLOTS>
__device__ __forceinline__ void mean_action_cta(const EngineDev &E, unsigned curmask, int g, int of, float *mean,
                                                int *count, int a, int c0, int cta_cnt, int o0, const int *slot_row,
                                                int out0, unsigned char *smem, int &n_in_s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const GroupDev &G = E.grp[g];
    const int na = E.grp[of].n_action;
    const int lut_stride = G.view_count;
    // lut[k] = {offset of the map cell in the padded planes from the observer's own cell, dx | dy << 16}
    int2 *lut = (int2 *)smem;
    int *hist = (int *)(lut + (E.turn_mode ? 4 : 1) * lut_stride) + warp * na;
    if (warp == 0) {                                          // compact the view mask, order-preserving
        const int cells = G.view_w * G.view_h;
        int k = 0;
        for (int base = 0; base < cells; base += 32) {
            const int cell = base + lane;
            const bool in = cell < cells && G.view_mask[cell];
            const unsigned bal = __ballot_sync(0xffffffffu, in);
            if (in) {
                const int vy = cell / G.view_w, vx = cell - vy * G.view_w;
                const int q = k + __popc(bal & ((1u << lane) - 1u));
                for (int d = 0; d < (E.turn_mode ? 4 : 1); ++d) {
                    int dx, dy;
                    nbr_view_delta(E, G, d, vx, vy, dx, dy);
                    lut[d * lut_stride + q] = make_int2(dy * E.kw + dx, (dx & 0xffff) | (int)((unsigned)dy << 16));
                }
            }
            k += __popc(bal);
        }
        if (lane == 0) n_in_s = k;
    }
    __syncthreads();
    const int n_in = n_in_s;
    const int n_mine = cta_cnt > warp ? (cta_cnt - warp + MEAN_WARPS - 1) / MEAN_WARPS : 0;
    NbrObserver mine;                                         // lane u: observer c0 + warp + MEAN_WARPS * u
    mine.x = mine.y = 0; mine.dir = DIR_NORTH; mine.code = 0; mine.flags = FLAG_DEAD;
    if (lane < n_mine) nbr_cta_load<SLOTS>(E, curmask, a, g, o0, slot_row, c0 + warp + MEAN_WARPS * lane, mine);
    const unsigned char *kplane = E.kind + (long)a * E.kplane;
    for (int u = 0; u < n_mine; ++u) {
        const int i = c0 + warp + MEAN_WARPS * u;
        NbrObserver o;
        o.x = __shfl_sync(0xffffffffu, mine.x, u); o.y = __shfl_sync(0xffffffffu, mine.y, u);
        nbr_cta_take<SLOTS>(g, i, mine, u, o);
        for (int k = lane; k < na; k += 32) hist[k] = 0;
        __syncwarp();
        int cnt = 0;
        if (!(o.flags & FLAG_DEAD)) {
            const unsigned char *kp = kplane + (long)(o.y + E.kpad) * E.kw + o.x + E.kpad;
            const int2 *l = lut + (E.turn_mode ? o.dir * lut_stride : 0);
            for (int q0 = lane; q0 < n_in; q0 += 32 * MEAN_UNROLL) {
                int t[MEAN_UNROLL];
#pragma unroll
                for (int r = 0; r < MEAN_UNROLL; ++r) t[r] = q0 + 32 * r < n_in ? __ldg(kp + l[q0 + 32 * r].x) : 0;
#pragma unroll
                for (int r = 0; r < MEAN_UNROLL; ++r) {
                    if (!nbr_kind_of(t[r], of)) continue;
                    const int d = l[q0 + 32 * r].y;
                    const int j = nbr_at(E, curmask, a, g, of, o, o.x + (short)(d & 0xffff), o.y + (d >> 16));
                    if (j < 0) continue;
                    ++cnt;
                    const int k = nbr_bin(E, curmask, a, of, j);
                    if (k >= 0) atomicAdd(hist + k, 1);
                }
            }
            cnt = __reduce_add_sync(0xffffffffu, cnt);
        }
        __syncwarp();
        float *row = mean + (size_t)(out0 + i) * na;
        for (int k = lane; k < na; k += 32) row[k] = nbr_mean(hist[k], cnt);
        if (count && lane == 0) count[out0 + i] = cnt;
        __syncwarp();                                         // the histogram is read before the next observer clears it
    }
}

__global__ void __launch_bounds__(MEAN_THREADS, 5) mean_action_kernel(const EngineDev *gE, unsigned curmask, int g, int of,
                                                                  float *mean, int *count, int n_total,
                                                                  int chunks_per_arena) {
    __shared__ EngineDev sE;
    __shared__ int n_in_s;
    extern __shared__ __align__(16) unsigned char mean_smem[];
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * MEAN_OBS;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const int o0 = off[a];
    int cta_cnt = min(MEAN_OBS, off[a + 1] - o0 - c0);
    cta_cnt = min(cta_cnt, n_total - (o0 + c0));                 // never beyond the caller's buffers
    if (cta_cnt <= 0) return;
    mean_action_cta<false>(E, curmask, g, of, mean, count, a, c0, cta_cnt, o0, nullptr, o0, mean_smem, n_in_s);
}

// dynamic shared memory of both mean-action kernels: the view LUT (one per heading in turn_mode) and the warps' histograms
static size_t mean_dyn_smem(const EngineDev &hE, int group, int of) {
    return (size_t)(hE.turn_mode ? 4 : 1) * hE.grp[group].view_count * sizeof(int2) +
           (size_t)MEAN_WARPS * hE.grp[of].n_action * sizeof(int);
}

void launch_mean_action(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group, int of,
                        float *mean, int *count, int n_total) {
    DeviceGuard guard(c);
    const size_t smem = mean_dyn_smem(hE, group, of);
    smem_prepare(c, ATTR_MEAN, mean_action_kernel, smem, "mean_action_kernel");
    const int cpa = (hE.grp[group].cap + MEAN_OBS - 1) / MEAN_OBS;
    mean_action_kernel<<<(unsigned)((size_t)hE.A * cpa), MEAN_THREADS, smem, c->stream>>>(dE, curmask, group, of, mean,
                                                                                          count, n_total, cpa);
    post_launch("mean_action_kernel");
}

// ------------------------------------------------------------------------------------------------
// nearest visible neighbours (magent_b200_get_neighbours): the first k members of N(i) in key order (nbr_phases.h
// nbr_cell_key) for every observer of a group.  The mapping is mean_action_kernel's: CTAs are dealt per arena, a CTA
// owns NBR_OBS consecutive observers, warp w takes observers w, w + 8, ... of them one at a time after its lanes have
// loaded all of their fields.  The lanes walk the group's view LUT, sorted by key on the host (Engine::to_device), in
// rounds of 32 cells: lane order is key order, so a ballot over the cells that list a neighbour hands out consecutive
// slots (found so far + popc of the lower lanes) and the row comes out sorted without a sort.  Every lane issues the
// `kind`-byte loads of NBR_ROUNDS rounds before it looks at any of them; only a byte that shows group `of` goes on to
// `occ` and, for a longer body, the smallest-key test (nbr_nearest_at).  Without `count` the warp stops after the round
// that fills slot k.  The LUT stays in global memory (L1-resident: 16 bytes per cell, the same for every observer), so the
// CTA holds nothing but the EngineDev copy.
constexpr int NBR_THREADS = 256, NBR_OBS = 128, NBR_ROUNDS = 4;
constexpr int NBR_WARPS = NBR_THREADS / 32;
static_assert(NBR_OBS / NBR_WARPS <= 32, "a warp's observers are loaded one per lane");

// The idx entry of neighbour j (index j of group `of` in arena a): its row, base + j, or (SLOTS) its flat slot
// a * S_of + slot, looked up through its id as slots_kernel looks up a row's (slot_phases.h slot_flat).  Only stored
// entries are translated: two dependent loads per stored neighbour.
template <bool SLOTS>
__device__ __forceinline__ int nbr_cta_index(const EngineDev &E, unsigned curmask, int a, int of, int base, int j,
                                             const SlotDev *T, int S_of) {
    if (!SLOTS) return base + j;
    return slot_flat(T->tab, T->id_cap, a, cur_soa(E, curmask, of).id[gidx(E, a, of, j)], S_of);
}

// One CTA of the neighbours kernels: observers c0 .. c0 + cta_cnt - 1 of arena a (nbr_cta_load), the row of observer v
// written at out0 + v.
template <bool SLOTS>
__device__ __forceinline__ void neighbours_cta(const EngineDev &E, const NbrCell *lut, unsigned curmask, int g, int of,
                                               int k, int *idx, int *rel, int *count, int a, int c0, int cta_cnt, int o0,
                                               const int *slot_row, int out0, const SlotDev *T, int S_of) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int base = E.off[(size_t)of * (E.A + 1) + a];          // row of j = base + j in `of`'s concatenation
    const int n_in = E.grp[g].view_count;
    const int n_mine = cta_cnt > warp ? (cta_cnt - warp + NBR_WARPS - 1) / NBR_WARPS : 0;
    NbrObserver mine;                                             // lane u: observer c0 + warp + NBR_WARPS * u
    mine.x = mine.y = 0; mine.dir = DIR_NORTH; mine.code = 0; mine.flags = FLAG_DEAD;
    if (lane < n_mine) nbr_cta_load<SLOTS>(E, curmask, a, g, o0, slot_row, c0 + warp + NBR_WARPS * lane, mine);
    const unsigned char *kplane = E.kind + (long)a * E.kplane;
    const unsigned lower = (1u << lane) - 1u;
    for (int u = 0; u < n_mine; ++u) {
        const int i = c0 + warp + NBR_WARPS * u;
        NbrObserver o;
        o.x = __shfl_sync(0xffffffffu, mine.x, u); o.y = __shfl_sync(0xffffffffu, mine.y, u);
        nbr_cta_take<SLOTS>(g, i, mine, u, o);
        const size_t row = (size_t)(out0 + i) * k;
        int found = 0;
        if (!(o.flags & FLAG_DEAD)) {
            const unsigned char *kp = kplane + (long)(o.y + E.kpad) * E.kw + o.x + E.kpad;
            const NbrCell *l = lut + (E.turn_mode ? o.dir * n_in : 0);
            // warp-uniform bounds: every lane takes part in every ballot
            for (int q0 = lane; q0 - lane < n_in && (count || found < k); q0 += 32 * NBR_ROUNDS) {
                int t[NBR_ROUNDS];
#pragma unroll
                for (int r = 0; r < NBR_ROUNDS; ++r) t[r] = q0 + 32 * r < n_in ? __ldg(kp + __ldg(&l[q0 + 32 * r].off)) : 0;
#pragma unroll
                for (int r = 0; r < NBR_ROUNDS; ++r) {
                    if (!count && found >= k) break;
                    int j = -1, cell = 0;
                    if (nbr_kind_of(t[r], of)) {
                        const int4 c = __ldg((const int4 *)(l + q0 + 32 * r));
                        j = nbr_nearest_at(E, curmask, a, g, of, o, o.x + (short)(c.y & 0xffff), o.y + (c.y >> 16), c.z);
                        cell = c.w;
                    }
                    const unsigned hits = __ballot_sync(0xffffffffu, j >= 0);
                    const int slot = found + __popc(hits & lower);
                    if (j >= 0 && slot < k) {
                        idx[row + slot] = nbr_cta_index<SLOTS>(E, curmask, a, of, base, j, T, S_of);
                        if (rel) { rel[2 * (row + slot)] = cell >> 16; rel[2 * (row + slot) + 1] = cell & 0xffff; }
                    }
                    found += __popc(hits);
                }
            }
        }
        for (int s = found + lane; s < k; s += 32) {              // unused slots
            idx[row + s] = -1;
            if (rel) { rel[2 * (row + s)] = -1; rel[2 * (row + s) + 1] = -1; }
        }
        if (count && lane == 0) count[out0 + i] = found;
    }
}

__global__ void __launch_bounds__(NBR_THREADS, 5) neighbours_kernel(const EngineDev *gE, const NbrCell *lut,
                                                                    unsigned curmask, int g, int of, int k, int *idx,
                                                                    int *rel, int *count, int n_total,
                                                                    int chunks_per_arena) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * NBR_OBS;
    const int o0 = E.off[(size_t)g * (E.A + 1) + a];
    int cta_cnt = min(NBR_OBS, E.off[(size_t)g * (E.A + 1) + a + 1] - o0 - c0);
    cta_cnt = min(cta_cnt, n_total - (o0 + c0));                 // never beyond the caller's buffers
    if (cta_cnt <= 0) return;
    neighbours_cta<false>(E, lut, curmask, g, of, k, idx, rel, count, a, c0, cta_cnt, o0, nullptr, o0, nullptr, 0);
}

void launch_neighbours(Ctx *c, const EngineDev *dE, const EngineDev &hE, const NbrCell *lut, unsigned curmask, int group,
                       int of, int k, int *idx, int *rel, int *count, int n_total) {
    DeviceGuard guard(c);
    const int cpa = (hE.grp[group].cap + NBR_OBS - 1) / NBR_OBS;
    neighbours_kernel<<<(unsigned)((size_t)hE.A * cpa), NBR_THREADS, 0, c->stream>>>(dE, lut, curmask, group, of, k, idx,
                                                                                    rel, count, n_total, cpa);
    post_launch("neighbours_kernel");
}

// ------------------------------------------------------------------------------------------------
// obs_prepare: the minimap of one observation state (GridWorld.cc:328-357): per (arena, group) the number of agents in
// every coarse cell of the OBSERVER's view-sized grid, divided by the group's size.  Dead-but-unculled agents count,
// absorbed ones do not when the observer's type can absorb (:343-347).  (The hp_norm plane the render also needs is
// kept current by the step kernels, step_phases.h hpn_set.)
//
// minimap_small_kernel: one CTA per (arena, group) when a group of an arena is at most a few thousand agents --
// histogram in shared memory, normalised row written directly.  Larger groups: obs_prepare_kernel histograms chunks of
// 4096 agents into global counters, minimap_norm_kernel normalises.
__global__ void __launch_bounds__(256) minimap_small_kernel(const EngineDev *gE, unsigned curmask, int og, float *mm_val, int stride) {
    extern __shared__ int hist[];
    __shared__ int counted_s;
    const EngineDev &E = *gE;
    const int ag = blockIdx.x;               // a * G + j
    const int a = ag / E.G, j = ag - a * E.G;
    const int vw = E.grp[og].view_w, vh = E.grp[og].view_h, cells = vw * vh;
    const int n = E.n[j * E.A + a];
    for (int k = threadIdx.x; k < cells; k += blockDim.x) hist[k] = 0;
    if (threadIdx.x == 0) counted_s = 0;
    __syncthreads();
    const GroupDev &G = E.grp[j];
    const AgentSoA &s = G.soa[(curmask >> j) & 1u];
    const int scale_h = (E.H + vh - 1) / vh, scale_w = (E.W + vw - 1) / vw;
    const bool skip_absorbed = E.grp[og].can_absorb != 0;
    int counted = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const long gi = (long)a * G.cap + i;
        if (skip_absorbed && (s.flags[gi] & FLAG_ABSORBED)) continue;
        atomicAdd(&hist[(s.y[gi] / scale_h) * vw + s.x[gi] / scale_w], 1);
        ++counted;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) counted += __shfl_xor_sync(0xffffffffu, counted, d);
    if ((threadIdx.x & 31) == 0 && counted) atomicAdd(&counted_s, counted);
    __syncthreads();
    const int tot = counted_s;
    float *out = mm_val + (size_t)a * stride + (size_t)j * cells;
    // an empty (or fully absorbed) group is 0/0 in the reference: x86 divss yields the default quiet NaN 0xFFC00000
    for (int k = threadIdx.x; k < cells; k += blockDim.x)
        out[k] = tot ? (float)hist[k] / (float)tot : __int_as_float((int)0xFFC00000u);
}

__global__ void __launch_bounds__(256) obs_prepare_kernel(const EngineDev *gE, unsigned curmask, int og, int chunk) {
    extern __shared__ int hist[];
    const EngineDev &E = *gE;
    const int ag = blockIdx.y;               // a * G + j
    const int a = ag / E.G, j = ag - a * E.G;
    const int vw = E.grp[og].view_w, vh = E.grp[og].view_h, cells = vw * vh;
    const int n = E.n[j * E.A + a];
    const int lo = blockIdx.x * chunk;
    if (lo >= n) return;
    const int hi = min(n, lo + chunk);
    for (int k = threadIdx.x; k < cells; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    const GroupDev &G = E.grp[j];
    const AgentSoA &s = G.soa[(curmask >> j) & 1u];
    const int scale_h = (E.H + vh - 1) / vh, scale_w = (E.W + vw - 1) / vw;
    const bool skip_absorbed = E.grp[og].can_absorb != 0;     // GridWorld.cc:343-347 (the OBSERVER's type decides)
    int counted = 0;
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        long gi = (long)a * G.cap + i;
        if (skip_absorbed && (s.flags[gi] & FLAG_ABSORBED)) continue;
        atomicAdd(&hist[(s.y[gi] / scale_h) * vw + s.x[gi] / scale_w], 1);
        ++counted;
    }
    if (counted) atomicAdd(&E.mm_total[ag], counted);
    __syncthreads();
    int *out = E.mm_count + (size_t)ag * cells;
    for (int k = threadIdx.x; k < cells; k += blockDim.x)
        if (hist[k]) atomicAdd(&out[k], hist[k]);
}

// normalised minimap, one padded row per arena: mm[a * stride + j * cells + cell]  (stride % 4 == 0 so that a row is a
// legal TMA bulk-copy source)
__global__ void __launch_bounds__(256) minimap_norm_kernel(const EngineDev *gE, int og, float *mm_val, int total, int stride) {
    const EngineDev &E = *gE;
    const int cells = E.grp[og].view_w * E.grp[og].view_h;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
        int ag = k / cells;
        // GridWorld.cc:350-357 (total_ct).  An empty (or fully absorbed) group is 0/0 in the reference: x86 divss
        // yields the default quiet NaN 0xFFC00000 whereas the GPU would give 0x7FFFFFFF, so emit the x86 payload.
        const int tot = E.mm_total[ag];
        const int a = ag / E.G;
        mm_val[(size_t)a * stride + (k - a * E.G * cells)] = tot ? (float)E.mm_count[k] / (float)tot : __int_as_float((int)0xFFC00000u);
    }
}

void launch_obs_prepare(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int og, float *mm_val) {
    if (!mm_val) return;                     // no minimap: nothing to prepare (the planes are kept current by the step)
    DeviceGuard guard(c);
    const int g_sms = c->sms;
    const int cells = hE.grp[og].view_w * hE.grp[og].view_h;
    const int total = hE.A * hE.G * cells;
    int cap_max = 0;
    for (int g = 0; g < hE.G; ++g) cap_max = cap_max > hE.grp[g].cap ? cap_max : hE.grp[g].cap;
    c->mm_stride = (hE.G * cells + 3) & ~3;
    const size_t need = (size_t)(hE.A + 1) * c->mm_stride;         // row A: the blank arena's (launch_obs_slots)
    if (need > c->mm_pad_n) {
        no_capture(c, "growing the minimap buffer");
        if (c->mm_pad) { CUDA_CHECK(cudaStreamSynchronize(c->stream)); CUDA_CHECK(cudaStreamSynchronize(c->copy)); cudaFree(c->mm_pad); }
        CUDA_CHECK(cudaMalloc(&c->mm_pad, need * sizeof(float)));
        CUDA_CHECK(cudaMemsetAsync(c->mm_pad, 0, need * sizeof(float), c->stream));
        c->mm_pad_n = need;
    }
    if (cap_max <= 8192 && smem_band(c, ATTR_MINIMAP_SMALL, minimap_small_kernel, (size_t)cells * sizeof(int)) == 0) {
        minimap_small_kernel<<<hE.A * hE.G, 256, cells * sizeof(int), c->stream>>>(dE, curmask, og, c->mm_pad, c->mm_stride);
        post_launch("minimap_small_kernel");
        return;
    }
    CUDA_CHECK(cudaMemsetAsync(hE.mm_count, 0, (size_t)total * 4, c->stream));
    CUDA_CHECK(cudaMemsetAsync(hE.mm_total, 0, (size_t)hE.A * hE.G * 4, c->stream));
    const int chunk = 4096;
    dim3 grid((cap_max + chunk - 1) / chunk, hE.A * hE.G);
    obs_prepare_kernel<<<grid, 256, cells * sizeof(int), c->stream>>>(dE, curmask, og, chunk);
    post_launch("obs_prepare_kernel");
    int g2 = (total + 255) / 256;
    if (g2 > 8 * g_sms) g2 = 8 * g_sms;
    minimap_norm_kernel<<<g2, 256, 0, c->stream>>>(dE, og, c->mm_pad, total, c->mm_stride);
    post_launch("minimap_norm_kernel");
}

// ------------------------------------------------------------------------------------------------
// obs_render_kernel: the observation gather (GridWorld.cc:292-401 + Map::extract_view Map.cc:129-207).
//
// The kernel is a stream of 4.7 KB records (battle) whose content is ~97 % zeros + the dense minimap channels +
// a handful of values gathered from the map.  Two ceilings matter: the TMA bulk-store stream itself and the L2
// throughput summed over reads and writes -- so every byte the kernel READS through L2 competes with the bytes it
// writes:
//   * tile = TA consecutive agents of the ABI concatenation = ONE CTA of TA warps, one warp per agent, one
//     shared-memory tile, 32 warps per SM (battle f32: 8 agents, 37.9 KB, 4 CTAs per SM), chunks of tiles dealt per
//     SM through device counters, so the CTAs of one SM compose neighbouring observers of one arena together (its
//     plane rows are shared in L1) and the whole grid works inside a window of a few arenas (planes / minimaps
//     L2-hot);
//   * the map is gathered from a ONE-BYTE kind plane (0 empty / 1 wall / 2+group; a view row is one 32-byte
//     sector) and only occupied cells (~5 %) take a second, dependent load from the hp_norm plane;
//   * the tile is composed entirely on the SM: each warp zero-fills its own record, copies the arena's
//     normalised minimap (G x cells floats, L1-resident) into the minimap channels, adds the self marker and
//     scatters the non-zero map values (n_channel-word stride => conflict-free for odd channel counts) --
//     no template tile is read through L2;
//   * the tile leaves the SM as ONE TMA bulk STORE (cp.async.bulk.global.shared::cta, SASS UBLKCP).  A tile's
//     byte range in the output is contiguous and 16-byte aligned because TA * sizeof(T) % 16 == 0.
//   * two tile widths (launch_obs_typed picks one per launch): the wide tile (8 f32 / 16 f16 agents) is 32 bytes
//     per record element, so its byte range is also 32-byte aligned for any record length -- a tile that starts
//     or ends inside a 32-byte sector shares that sector with a tile of another CTA.  It is used whenever it keeps
//     at least as many warps per SM as the narrow tile (4 f32 / 8 f16 agents), which also serves records too large
//     for a wide tile in shared memory.
// Algorithmic traffic per agent: sizeof(T)*(view_h*view_w*n_channel + feature) bytes written, plus one compulsory
// read of the occupancy plane per arena (DESIGN.md section 6).  No tensor cores: there is no contraction here.
#ifndef OBS_ABLATE
#define OBS_ABLATE 0                 // profiling experiments only: 1 no plane gather, 2 no tile
#endif                               // init (zero + minimap), 4 no feature rows, 8 no bulk store -- results are WRONG

// output element type of the observation: float = the reference ABI (env_get_observation); __half = the compact
// hand-off format of magent_b200_get_observation_f16 (each value is the f32 value rounded to nearest-even).
template <typename T> struct ObsOut;
template <> struct ObsOut<float> {
    static __device__ __forceinline__ float cv(float v) { return v; }
};
template <> struct ObsOut<__half> {
    static __device__ __forceinline__ __half cv(float v) {
        if (v != v) {                    // keep sign and top payload bits like a software f32->f16 cast does (numpy astype)
            const unsigned u = __float_as_uint(v);
            unsigned short r = (unsigned short)(0x7c00u + ((u & 0x7fffffu) >> 13));
            if (r == 0x7c00u) ++r;
            return __ushort_as_half((unsigned short)(r | ((u >> 16) & 0x8000u)));
        }
        return __float2half_rn(v);
    }
};

struct ObsParams {
    int A, W, H, G, C;
    int vw, vh, cells, rec, F;
    int ox, oy;                      // map offset of view cell (0,0) from the agent position
    int scale_w, scale_h, minimap;
    int cap, embedding, n_action, n_total;
    const unsigned char *mask;
    const int *off;
    const unsigned char *kind_plane; // [A][kplane] padded: 0 empty / 1 wall / 2+group (EngineDev::kind)
    const float *hpn_plane;          // [A][kplane] padded: hp / max_hp of the occupant (EngineDev::hpn)
    int kpad, kw;
    long kplane;
    int chunk;                       // consecutive tiles per CTA visit (<= OBS_CHUNK)
    unsigned *deal;                  // [sms + 1] chunk counters per SM + done counter (Ctx::obs_deal), or nullptr:
                                     // chunks round-robin over the CTAs
    int sms, deal_unit;              // the SMs that own chunk sequences; chunks per unit of a sequence
    int turn, body_w, body_l;        // turn_mode: 4 view LUTs (one per heading), the heading rides in the header
    const unsigned char *dir;
    const int *x, *y, *id, *act;
    const float *last_reward;
    const float *mm;                 // [A][mm_stride] normalised minimap rows (G x cells floats each), or nullptr
    int mm_stride;
    const int4 *hdr;                 // [n_total] per-agent header in ABI order (obs_headers_kernel)
    void *view, *feature;            // element type = the kernel's template argument
    int mm_ch[MG_MAX_GROUPS];        // observation channel of group j's minimap
    int grp_ch[MG_MAX_GROUPS];       // observation channel ('has'; hp is +1) of group j
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One observer of the pre-passes, agent i of arena a: returns its render header and writes the non-zeros of its
// feature row into f (F elements, zero-filled by the caller).
//   * header h = {x, y, arena, self minimap cell | heading << 16}: everything the render kernel needs about the observer itself, so
//     that its only dependent loads are kind plane -> hp_norm plane;
//   * the complete non-spatial feature row (GridWorld.cc:386-396): id bits LSB first, one-hot last action, last
//     reward, and x/W, y/H with the minimap.  A fresh agent's last_action == n_action ("dangerous", GridWorld.h:140)
//     lands on the reward slot and is overwritten by it -- here the reward simply wins.
template <typename T>
__device__ __forceinline__ int4 obs_observer(const ObsParams &P, int a, int i, T *f) {
    const long gi = (long)a * P.cap + i;
    const int x = P.x[gi], y = P.y[gi];
    const int self_cell = P.minimap ? (y / P.scale_h) * P.vw + x / P.scale_w : -1;  // GridWorld.cc:372-373
    const int heading = P.turn ? (int)P.dir[gi] : 0;
    unsigned id = (unsigned)P.id[gi];
    const int nbits = min(P.embedding, 31);
    id &= nbits >= 32 ? 0xffffffffu : ((1u << nbits) - 1u);
    while (id) {                                           // embedding: the set bits of the id, LSB first (GridWorld.h:155-164)
        const int bit = __ffs(id) - 1;
        f[bit] = ObsOut<T>::cv(1.0f);
        id &= id - 1;
    }
    T *g = f + P.embedding;
    const int act = P.act[gi];
    if (act >= 0 && act < P.n_action) g[act] = ObsOut<T>::cv(1.0f);
    g[P.n_action] = ObsOut<T>::cv(P.last_reward[gi]);       // also overwrites the "dangerous" fresh-agent one-hot slot
    if (P.minimap) {
        g[P.n_action + 1] = ObsOut<T>::cv((float)x / (float)P.W);               // GridWorld.cc:394-395
        g[P.n_action + 2] = ObsOut<T>::cv((float)y / (float)P.H);
    }
    return make_int4(x, y, a, (self_cell & 0xffff) | (heading << 16));
}

// the cnt * F elements of `rows` (shared memory) into out, coalesced
template <typename T>
__device__ __forceinline__ void obs_store_rows(T *out, const T *rows, int total) {
    if (sizeof(T) == 4 && ((((size_t)out) & 15) == 0)) {       // 16-byte body, scalar tail
        const int v4 = total >> 2;
        for (int q = threadIdx.x; q < v4; q += blockDim.x) ((float4 *)out)[q] = ((const float4 *)rows)[q];
        for (int q = (v4 << 2) + threadIdx.x; q < total; q += blockDim.x) out[q] = rows[q];
    } else {
        for (int q = threadIdx.x; q < total; q += blockDim.x) out[q] = rows[q];
    }
}

// pre-pass, one thread per observer, CTAs dealt per arena (no search for the arena: blockIdx says it): the header and
// feature row of every observer (obs_observer).  The rows of a CTA's observers are one contiguous block of the output:
// composed in shared memory (zero fill, then every thread its own handful of non-zeros), written out with coalesced
// stores.
template <typename T>
__global__ void __launch_bounds__(256) obs_headers_kernel(ObsParams P, int4 *hdr, int chunks_per_arena) {
    extern __shared__ __align__(16) unsigned char hdr_smem[];
    T *rows = (T *)hdr_smem;                                   // [blockDim.x][F]
    const int a = blockIdx.x / chunks_per_arena;
    const int i0 = (blockIdx.x - a * chunks_per_arena) * blockDim.x;
    const int o0 = P.off[a], n_a = P.off[a + 1] - o0;
    if (i0 >= n_a) return;
    int cnt = min((int)blockDim.x, n_a - i0);
    cnt = min(cnt, P.n_total - (o0 + i0));                     // never beyond the caller's buffers
    if (cnt <= 0) return;
    const int total = cnt * P.F;
    for (int q = threadIdx.x; q < total; q += blockDim.x) rows[q] = ObsOut<T>::cv(0.0f);
    __syncthreads();
    if ((int)threadIdx.x < cnt) {
        const int i = i0 + threadIdx.x;
        hdr[o0 + i] = obs_observer<T>(P, a, i, rows + (size_t)threadIdx.x * P.F);
    }
    __syncthreads();
    obs_store_rows<T>((T *)P.feature + (size_t)(o0 + i0) * P.F, rows, total);
}

// the slot-ordered pre-pass (magent_b200_get_observation_slots): the same header and feature row per slot, in [A][S]
// order.  slot_row ([A][S], slots_kernel) names the row in each slot, -1 when vacant; `off` are the group's device-side
// offsets (P.off is the render's count bound in a slot launch).  CTAs are dealt per arena, one thread per slot, so
// every header and every feature row is written exactly once and the stores are coalesced whatever the slots' order.
// A vacant slot gets the header of the blank arena A ({0, 0, A, 0}: see launch_obs_slots) and a zero feature row.
template <typename T>
__global__ void __launch_bounds__(256) obs_slot_headers_kernel(ObsParams P, const int *off, const int *slot_row, int S,
                                                               int4 *hdr, int chunks_per_arena) {
    extern __shared__ __align__(16) unsigned char hdr_smem[];
    T *rows = (T *)hdr_smem;                                   // [blockDim.x][F]
    const int a = blockIdx.x / chunks_per_arena;
    const int s0 = (blockIdx.x - a * chunks_per_arena) * blockDim.x;
    if (s0 >= S) return;
    const int cnt = min((int)blockDim.x, S - s0);
    const int total = cnt * P.F;
    const long o = (long)a * S + s0;                           // first slot of this CTA in [A][S] order
    for (int q = threadIdx.x; q < total; q += blockDim.x) rows[q] = ObsOut<T>::cv(0.0f);
    __syncthreads();
    if ((int)threadIdx.x < cnt) {
        const int r = __ldg(slot_row + o + threadIdx.x);
        hdr[o + threadIdx.x] = r >= 0 ? obs_observer<T>(P, a, r - __ldg(off + a), rows + (size_t)threadIdx.x * P.F)
                                      : make_int4(0, 0, P.A, 0);
    }
    __syncthreads();
    obs_store_rows<T>((T *)P.feature + o * P.F, rows, total);
}

#ifndef OBS_WARPS_PER_SM
#define OBS_WARPS_PER_SM 32          // resident render warps per SM the register budget is sized for: 64 per thread
#endif
// agents per tile (= warps per CTA) of the narrow and the wide render tile; TA * sizeof(T) % 16 == 0 keeps every
// tile's byte range 16-byte aligned, and the wide tile is 32 bytes per record element
template <typename T> constexpr int obs_tile_narrow() { return 16 / (int)sizeof(T); }
template <typename T> constexpr int obs_tile_wide() { return 32 / (int)sizeof(T); }
#ifndef OBS_CHUNK
#define OBS_CHUNK 4                  // consecutive tiles a CTA renders before it claims its next chunk
#endif
#ifndef OBS_DEAL_UNIT
#define OBS_DEAL_UNIT 4              // a unit of an SM's chunk sequence = OBS_DEAL_UNIT * (CTAs per SM) consecutive chunks
#endif
#ifndef OBS_DEAL_MIN_UNITS
#define OBS_DEAL_MIN_UNITS 4         // automatic launches deal per SM only with at least this many units per SM
#endif
// NIT = view cells per lane held in registers (NIT * 32 >= in-range cells of the view whenever that is <= 256;
// larger views take the unpipelined tail loop).
//
// The small-view instantiation (NIT = 4, no headings) is launched only for views of at most 4 * 32 in-range cells
// (launch_obs_dispatch, checked again in launch_obs_typed), so it keeps its whole LUT slice in registers and carries
// no tail loop at all: the dead tail alone cost it 84 bytes of spills per thread on sm_90a.
template <int NIT, bool TURN> constexpr bool obs_all_cells_in_regs() { return NIT <= 4 && !TURN; }
//
// The tile buffer is PERSISTENT: consecutive tiles of a CTA belong to the same arena (blocked tile assignment), so
// the zeros and the arena's minimap channels already in the buffer are still right for the next tile.  After the
// bulk store has read the buffer, each warp only UNDOES the few cells it marked for the previous observer (kinds
// remembered in one packed register) and restores the self-marker cell, then marks the new observer's cells.  A
// warp rebuilds its record (zero fill + minimap rows from L2) only when its observer's arena changes -- once or
// twice per launch.
template <typename T, int NIT, bool TURN, int TA>
__global__ void __launch_bounds__(32 * TA, OBS_WARPS_PER_SM / TA)
obs_render_kernel(const __grid_constant__ ObsParams P) {
    const int n_total = min(P.n_total, __ldg(P.off + P.A));   // the host may hold pre-cull counts (upper bounds)
    constexpr int OBS_TA = TA;
    constexpr int OBS_THREADS = 32 * OBS_TA;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    T *buf = (T *)smem_raw;                                   // one tile: OBS_TA records
    // in-range view cells only: lut[k] = {word offset of the cell inside a record, offset of the map cell in the
    // padded planes relative to the observer's own cell}
    int2 *lut = (int2 *)(buf + OBS_TA * P.rec);
    __shared__ int n_in_s;
    __shared__ int deal_s[4];                                 // claimed tiles: the first three, then the next chunk's start
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n_tiles = (n_total + OBS_TA - 1) / OBS_TA;

    // Tile assignment: chunks of P.chunk consecutive tiles; within a chunk the arena (almost) never changes, so the
    // persistent tile needs no rebuild.  With P.deal, the chunks are dealt per SM: units of P.deal_unit consecutive
    // chunks go round-robin to the SMs, and SM s's sequence of units is handed out chunk by chunk by counter s.  Every
    // CTA resident on SM s claims from counter s, so the CTAs of one SM compose neighbouring observers of one arena at
    // the same time and share its kind / hp plane rows in L1; all SMs still advance together through the output, inside
    // a window of about sms * unit chunks (a blocked assignment -- one contiguous region per CTA -- would spread the
    // stream over the whole output, beyond the TLB reach).  A CTA whose SM's sequence is drained claims from the other
    // counters in the order home + 1, home + 2, ..., so every chunk is rendered exactly once whatever the placement
    // of the CTAs (an SM without CTAs, an SM with more than the occupancy, a forced grid of 1), and the CTAs finish
    // together.  Without P.deal (a single round, or too few units per SM: launch_obs_render) the chunks go round-robin
    // over the CTAs: CTA b renders chunks b, b + grid, b + 2 * grid, ...
    // Warp 0 claims; a claim returns the first tile of the claimed chunk, n_tiles when there is none left.  The claim
    // of the chunk that follows tile i+2 is issued before tile i is composed and read after it (CLAIM_LATE), or before
    // it for the float NIT = 8 instantiations: they have no register to spare across the composition (holding the
    // claim there cost them 60 bytes of spills per thread).
    constexpr bool CLAIM_LATE = !(sizeof(T) == 4 && NIT == 8);
    const int chunk = P.chunk;
    // warp 0's claim state, in shared memory so that it holds no register across the tile loop: this CTA's SM (its
    // home counter; %smid need not be dense, and any counter is correct) and the counters drained so far, in the
    // order home, home + 1, ...
    __shared__ int home_s, drained_s;
    if (threadIdx.x == 0 && P.deal) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        home_s = (int)(smid % (unsigned)P.sms);
        drained_s = 0;
    }
    __syncwarp();
    auto seq_chunk = [&](int s, unsigned j, int n_chunks) -> int {   // chunk j of SM s's sequence (n_chunks: beyond its end)
        const long c = ((long)(j / P.deal_unit) * P.sms + s) * P.deal_unit + j % P.deal_unit;
        return c < n_chunks ? (int)c : n_chunks;
    };
    auto counter_of = [&](int home, int drained) -> int { return home + drained < P.sms ? home + drained : home + drained - P.sms; };
    // lane 0 of warp 0 takes a chunk index from the counter being drained; the atomic is issued ahead of claim() so
    // that its latency hides behind other work
    auto issue_claim = [&]() -> unsigned {
        return lane == 0 && drained_s < P.sms ? atomicAdd(P.deal + counter_of(home_s, drained_s), 1u) : 0u;
    };
    // warp 0, warp-uniform, P.deal only: the first tile of the claimed chunk (j = issue_claim()), n_tiles when none is left
    auto claim = [&](unsigned j) -> int {
        const int n_chunks = (n_tiles + chunk - 1) / chunk;
        const int home = home_s;
        int drained = drained_s, tile = n_tiles;
        __syncwarp();
        while (drained < P.sms) {
            const int c = __shfl_sync(0xffffffffu, lane == 0 ? seq_chunk(counter_of(home, drained), j, n_chunks) : 0, 0);
            if (c < n_chunks) { tile = c * chunk; break; }
            int next = P.sms;                             // this counter is drained: find the next live one, 32 at a time
            for (int base = drained + 1; base < P.sms; base += 32) {
                const int s = counter_of(home, base + lane);
                unsigned js = 0;
                if (base + lane < P.sms) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(js) : "l"(P.deal + s) : "memory");
                const unsigned b = __ballot_sync(0xffffffffu, base + lane < P.sms && seq_chunk(s, js, n_chunks) < n_chunks);
                if (b) { next = base + __ffs(b) - 1; break; }
            }
            drained = next;
            if (drained < P.sms && lane == 0) j = atomicAdd(P.deal + counter_of(home, drained), 1u);
        }
        if (lane == 0) drained_s = drained;
        __syncwarp();
        return tile;
    };
    // the tile after t: t + 1 inside its chunk, else nxt (the next claimed chunk) or the CTA's next round-robin chunk;
    // n_tiles past the end
    auto ends_chunk = [&](int t) -> bool { return t < n_tiles && (t + 1 == n_tiles || (t + 1) % chunk == 0); };
    auto next_tile = [&](int t, bool ends, int nxt) -> int {          // ends = ends_chunk(t)
        if (t >= n_tiles) return n_tiles;
        if (!ends) return t + 1;
        if (P.deal) return nxt;
        const long r = (long)t + 1 + (long)(gridDim.x - 1) * chunk;
        return r < n_tiles ? (int)r : n_tiles;
    };

    const int lut_stride = (P.cells + 1) & ~1;
    if (warp == 0) {                                          // compact the view mask (Range.h:104-189)
        int k = 0;                                            // order-preserving: ballot prefix per 32 cells
        for (int base = 0; base < P.cells; base += 32) {
            const int cell = base + lane;
            const bool in = cell < P.cells && P.mask[cell];
            const unsigned bal = __ballot_sync(0xffffffffu, in);
            if (in) {
                const int vy = cell / P.vw, vx = cell - vy * P.vw;
                const int q = k + __popc(bal & ((1u << lane) - 1u));
                if (!TURN) lut[q] = make_int2(cell * P.C, (P.oy + vy) * P.kw + P.ox + vx);
                else {
                    // the window is laid out in the observer's frame: one LUT per heading (Map.cc:140-146, 515-560)
                    for (int d = 0; d < 4; ++d) {
                        int rx = 0, ry = 0, dx, dy;                     // save_to_real
                        if (d == DIR_SOUTH) { rx = P.body_w - 1; ry = P.body_l - 1; }
                        else if (d == DIR_WEST) ry = P.body_w - 1;
                        else if (d == DIR_EAST) rx = P.body_l - 1;
                        const int ex = P.ox + vx, ey = P.oy + vy;       // rela_to_abs
                        if (d == DIR_NORTH) { dx = ex; dy = ey; }
                        else if (d == DIR_SOUTH) { dx = -ex; dy = -ey; }
                        else if (d == DIR_WEST) { dx = ey; dy = -ex; }
                        else { dx = -ey; dy = ex; }
                        lut[d * lut_stride + q] = make_int2(cell * P.C, (ry + dy) * P.kw + rx + dx);
                    }
                }
            }
            k += __popc(bal);
        }
        if (lane == 0) n_in_s = k;
        if (P.deal) {                                         // the pipeline starts with three tiles: claim their chunks
            const int t0 = claim(issue_claim());
            const int t1 = ends_chunk(t0) ? claim(issue_claim()) : next_tile(t0, false, n_tiles);
            const int t2 = ends_chunk(t1) ? claim(issue_claim()) : next_tile(t1, false, n_tiles);
            if (lane == 0) { deal_s[0] = t0; deal_s[1] = t1; deal_s[2] = t2; }
        }
    }
    __syncthreads();
    const int n_in = n_in_s;
    // this lane's slice of the view LUT never changes: small views keep it in registers, large ones re-read smem
    constexpr bool LUT_REGS = obs_all_cells_in_regs<NIT, TURN>();
    int2 lreg[LUT_REGS ? NIT : 1];
    if (LUT_REGS) {
#pragma unroll
        for (int it = 0; it < (LUT_REGS ? NIT : 1); ++it) lreg[it] = it * 32 + lane < n_in ? lut[it * 32 + lane] : make_int2(0, 0);
    }
    // hd = heading of the observer (always 0 without turn_mode)
    auto lutv = [&](int it, int hd) -> int2 {
        if (TURN) return it * 32 + lane < n_in ? lut[hd * lut_stride + it * 32 + lane] : make_int2(0, 0);
        return LUT_REGS ? lreg[LUT_REGS ? it : 0] : (it * 32 + lane < n_in ? lut[it * 32 + lane] : make_int2(0, 0));
    };
    // position of an observer's own cell in the padded planes (header word h = {x, y, arena, self cell | heading << 16})
    auto plane_base = [&](const int4 &h) -> long { return h.z * P.kplane + (long)(h.y + P.kpad) * P.kw + h.x + P.kpad; };

    // issue the kind-plane loads of one observer; the pad makes every view cell addressable.  Kinds are bytes: cell
    // `it` of a lane is byte it & 3 of kd[it >> 2].  The loads are unconditional (lanes past n_in read the observer's
    // own cell) and masked afterwards: per-cell predicates held across the tile loop were spilled on sm_90a.
    constexpr int KW = (NIT + 3) / 4;
    unsigned kmask[KW];                        // 0xff in the bytes of in-range cells
#pragma unroll
    for (int q = 0; q < KW; ++q) {
        kmask[q] = 0u;
#pragma unroll
        for (int b = 0; b < 4; ++b) if ((4 * q + b) * 32 + lane < n_in) kmask[q] |= 0xffu << (8 * b);
    }
    auto load_kinds = [&](const int4 &h, bool on, unsigned (&kd)[KW]) {
        const unsigned char *kp = P.kind_plane + plane_base(h);
        const int hd = TURN ? (h.w >> 16) & 3 : 0;
#pragma unroll
        for (int q = 0; q < KW; ++q) kd[q] = 0u;
#pragma unroll
        for (int it = 0; it < NIT; ++it) kd[it >> 2] |= (unsigned)__ldg(kp + lutv(it, hd).y) << ((it & 3) * 8);
#pragma unroll
        for (int q = 0; q < KW; ++q) kd[q] &= (on && !(OBS_ABLATE & 1)) ? kmask[q] : 0u;
    };
    auto kind_at = [](const unsigned (&kd)[KW], int it) -> int { return (kd[it >> 2] >> ((it & 3) * 8)) & 0xff; };
    // write (on = true) or erase what an occupied view cell shows: wall / food flag, or a group's {1, hp / max_hp}
    // channel of every kind, one byte each in two registers (byte k of chpack = channel of group k): no constant-bank
    // lookup and no branch ladder per marked cell
    unsigned long long chpack = 0ull;
#pragma unroll
    for (int j = 0; j < MG_MAX_GROUPS; ++j) chpack |= (unsigned long long)(P.grp_ch[j] & 0xff) << (8 * j);
    auto mark = [&](T *px, int t, float hp, bool on) {
        const bool agent = kind_is_agent(t);
        const int ch = agent ? (int)((chpack >> (8 * kind_group(t))) & 0xffull) : (t == KIND_FOOD ? 1 : 0);
        px[ch] = ObsOut<T>::cv(on ? 1.0f : 0.0f);                          // wall / food flag or the group's 'has' channel
        if (agent) px[ch + 1] = ObsOut<T>::cv(on ? hp : 0.0f);             // hp / max_hp (Map.cc:197)
    };

    // Software pipeline: while tile i is composed, the kind loads of tile i+1 and the header load of tile i+2 fly; the
    // chunk that follows tile i+2 is claimed during tile i and passed on at one of its barriers.
    int tile = (int)blockIdx.x < (n_tiles + chunk - 1) / chunk ? (int)blockIdx.x * chunk : n_tiles;
    int tile1 = next_tile(tile, ends_chunk(tile), n_tiles), tile2 = next_tile(tile1, ends_chunk(tile1), n_tiles);
    if (P.deal) { tile = deal_s[0]; tile1 = deal_s[1]; tile2 = deal_s[2]; }
    const int tile_end = n_tiles;
    const int4 zero4 = make_int4(0, 0, 0, 0);
    int4 hA = zero4, hA1 = zero4;             // headers of tile i and i+1
    unsigned kind[KW];
    // what this warp's record currently shows: the arena whose minimap rows it holds (-1: garbage), the previous
    // observer's heading, marked kinds (packed bytes; > 4 * 32 cells per lane never happens with NIT <= 8) and
    // self-marker cell with its unmarked minimap value per group lane
    int rec_arena = -1, prev_hd = 0, prev_self = -1;
    unsigned prev_kinds[KW];
#pragma unroll
    for (int q = 0; q < KW; ++q) prev_kinds[q] = 0u;
    float self_orig = 0.0f;
    bool prev_tail = false;                    // the previous observer had cells beyond NIT * 32 marked (large views)
    {
        const int o0 = tile * OBS_TA + warp, o1 = tile1 * OBS_TA + warp;
        const bool on0 = tile < tile_end && o0 < n_total;
        if (on0) hA = P.hdr[o0];
        if (o1 < n_total) hA1 = P.hdr[o1];
        load_kinds(hA, on0, kind);
    }
    for (int tile3; tile < tile_end; tile = tile1, tile1 = tile2, tile2 = tile3) {
        const int t0 = tile * OBS_TA;
        const int cnt = min(OBS_TA, n_total - t0);
        const bool active = warp < cnt;
        const int a = hA.z;
        // occupied cells only: the occupant's hp / max_hp (the kinds were loaded one tile ago)
        const float *hpnp = P.hpn_plane + plane_base(hA);
        const int hd = TURN ? (hA.w >> 16) & 3 : 0;
        float thp[NIT];
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int t = kind_at(kind, it);
            thp[it] = 0.0f;
            if (kind_is_agent(t)) thp[it] = (t & KIND_FULL) ? 1.0f : __ldg(hpnp + lutv(it, hd).y);   // full hp: no load
        }
        // next tile's kinds, next-next tile's header
        unsigned kind1[KW];
        const long o1 = (long)tile1 * OBS_TA + warp;
        load_kinds(hA1, o1 < n_total, kind1);
        int4 hA2 = zero4;
        {
            const long o2 = (long)tile2 * OBS_TA + warp;
            if (o2 < n_total) hA2 = P.hdr[o2];
        }
        // the previous tile's bulk store must have finished READING the buffer before it is touched.  One buffer per
        // CTA on purpose: a second would cost a CTA per SM, and at battle's size that loses more than the overlap
        // wins (DESIGN.md section 5, "Two tile slots per CTA").  The claim's atomic flies while the tile is composed.
        const bool ends2 = ends_chunk(tile2), claims = P.deal && ends2;
        const unsigned j = claims && warp == 0 ? issue_claim() : 0u;
        if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        if (!CLAIM_LATE && claims && warp == 0) {
            const int t = claim(j);
            if (lane == 0) deal_s[3] = t;
        }
        __syncthreads();
        if (!CLAIM_LATE) tile3 = next_tile(tile2, ends2, claims ? deal_s[3] : n_tiles);   // read before the next barrier
        if (active && !(OBS_ABLATE & 2)) {
            T *dst = buf + warp * P.rec;
            const int self = (int)(short)(hA.w & 0xffff);
            if (a != rec_arena) {
                // (re)build the record: zeros + the arena's minimap rows (GridWorld.cc:374-383), element stores because
                // f16 records share 32-bit words with their neighbours
                if (sizeof(T) == 4) {                              // 16-byte body, scalar head / tail
                    float *w = (float *)dst;
                    const int n = P.rec;
                    const int head = min(n, (int)((4u - ((unsigned)(warp * P.rec) & 3u)) & 3u));
                    const int body = (n - head) >> 2;
                    if (lane < head) w[lane] = 0.0f;
                    float4 *w4 = (float4 *)(w + head);
                    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                    for (int q = lane; q < body; q += 32) w4[q] = z;
                    const int tail0 = head + (body << 2);
                    if (tail0 + lane < n) w[tail0 + lane] = 0.0f;
                } else {
                    for (int q = lane; q < P.rec; q += 32) dst[q] = ObsOut<T>::cv(0.0f);
                }
                __syncwarp();
                if (P.minimap) {
                    const float *rows = P.mm + (size_t)a * P.mm_stride;
                    for (int j = 0; j < P.G; ++j) {
                        T *d = dst + P.mm_ch[j];
                        for (int cell = lane; cell < P.cells; cell += 32) d[cell * P.C] = ObsOut<T>::cv(__ldg(rows + j * P.cells + cell));
                    }
                }
                rec_arena = a;
                __syncwarp();
            } else {
                // undo the previous observer: its marked cells and its self marker
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const int t = kind_at(prev_kinds, it);
                    if (t != 0) mark(dst + lutv(it, prev_hd).x, t, 0.0f, false);
                }
                if (!LUT_REGS && prev_tail) {                                                   // large views: recompute which tail cells were marked
                    for (int k = NIT * 32 + lane; k < n_in; k += 32) {
                        T *px = dst + lut[(TURN ? prev_hd * lut_stride : 0) + k].x;
                        for (int ch = 0; ch < P.C; ++ch) {
                            bool mm_ch = false;
                            for (int j = 0; j < P.G; ++j) mm_ch |= P.minimap && ch == P.mm_ch[j];
                            if (!mm_ch) px[ch] = ObsOut<T>::cv(0.0f);
                        }
                    }
                }
                if (P.minimap && lane < P.G && prev_self >= 0) dst[prev_self * P.C + P.mm_ch[lane]] = ObsOut<T>::cv(self_orig);
                __syncwarp();
            }
            // the new observer: self marker (+1 at its coarse cell; NaN + 1 keeps the x86 payload in the reference)
            if (P.minimap && lane < P.G) {
                const float v = __ldg(P.mm + (size_t)a * P.mm_stride + lane * P.cells + self);
                self_orig = v;
                if (v == v) dst[self * P.C + P.mm_ch[lane]] = ObsOut<T>::cv(v + 1.0f);
            }
            prev_self = self;
            prev_hd = hd;
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                const int t = kind_at(kind, it);
                if (t != 0) mark(dst + lutv(it, hd).x, t, thp[it], true);
            }
#pragma unroll
            for (int q = 0; q < KW; ++q) prev_kinds[q] = kind[q];
            prev_tail = false;
            const unsigned char *kindp = P.kind_plane + plane_base(hA);
            for (int k = NIT * 32 + lane; !LUT_REGS && k < n_in; k += 32) {                          // views with > NIT * 32 in-range cells
                const int2 l = lut[(TURN ? hd * lut_stride : 0) + k];
                const int t = __ldg(kindp + l.y);
                if (t != 0) { mark(dst + l.x, t, kind_is_agent(t) ? ((t & KIND_FULL) ? 1.0f : __ldg(hpnp + l.y)) : 0.0f, true); }
                prev_tail = true;
            }
        }
        if (CLAIM_LATE && claims && warp == 0) {
            const int t = claim(j);
            if (lane == 0) deal_s[3] = t;
        }
        // make the generic-proxy writes visible to the async proxy, then one thread fires the bulk store
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (CLAIM_LATE) tile3 = next_tile(tile2, ends2, claims ? deal_s[3] : n_tiles);   // read before the next barrier: deal_s[3] is rewritten after it
        T *gout = (T *)P.view + (size_t)t0 * P.rec;
        const unsigned bytes = (unsigned)cnt * (unsigned)P.rec * (unsigned)sizeof(T);
        if ((bytes & 15u) == 0 && (((size_t)gout) & 15) == 0) {
            if (threadIdx.x == 0 && !(OBS_ABLATE & 8)) {
                // the output is a write-once stream far larger than L2: evict_first keeps it from pushing out the
                // planes, minimap rows and headers the composition reads (the policy is made here, not held in a
                // register across the loop)
                unsigned long long pol;
                asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                             :: "l"(gout), "r"(smem_u32(buf)), "r"(bytes), "l"(pol) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        } else {                                   // ragged last tile / unaligned caller buffer
            for (int q = threadIdx.x; q < cnt * P.rec; q += OBS_THREADS) gout[q] = buf[q];
            __syncthreads();
        }
        // rotate the pipeline
        hA = hA1; hA1 = hA2;
#pragma unroll
        for (int q = 0; q < KW; ++q) kind[q] = kind1[q];
    }
    if (threadIdx.x == 0) {
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        if (P.deal) {                          // the last CTA to finish (every claim is made) zeroes the counters for
            __threadfence();                   // the next launch: a replayed graph needs no memset node
            if (atomicAdd(P.deal + P.sms, 1u) == gridDim.x - 1)
                for (int s = 0; s <= P.sms; ++s) P.deal[s] = 0u;
        }
    }
}

// CTAs per SM of one render instantiation at this shared-memory size (0: it does not fit), cached per context slot
template <typename T, int NIT, bool TURN, int TA>
static int obs_ctas_per_sm(Ctx *c, int cfg_slot, size_t smem) {
    if (smem_band(c, ATTR_OBS0 + cfg_slot, obs_render_kernel<T, NIT, TURN, TA>, smem) < 0) return 0;
    Ctx::ObsCfg &cfg = c->obs_cfg[cfg_slot];
    ensure_dynamic_smem(c->device, ATTR_OBS0 + cfg_slot, obs_render_kernel<T, NIT, TURN, TA>, smem);
    if (smem != cfg.smem) {
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cfg.ctas_per_sm, obs_render_kernel<T, NIT, TURN, TA>, 32 * TA, smem));
        cfg.smem = smem;
    }
    return cfg.ctas_per_sm;
}

// O.grid / O.chunk > 0 replace the automatic grid and chunk (tests: CTAs that render many tiles at small sizes).
// Both are clamped: grid to [1, tiles], chunk to [1, ceil(tiles / grid)], so that no CTA is launched without a tile
// and no chunk is longer than a CTA's share.  The clamps never change the automatic values.
template <typename T, int NIT, bool TURN, int TA>
static void launch_obs_render(Ctx *c, const ObsArgs &O, ObsParams &P, int n_total, size_t smem, int ctas_per_sm) {
    const int g_sms = c->sms;
    const int tiles = (n_total + TA - 1) / TA;
    int grid = tiles < ctas_per_sm * g_sms ? tiles : ctas_per_sm * g_sms;
    P.chunk = tiles / (ctas_per_sm * g_sms);                            // keep every CTA busy before lengthening chunks
    if (P.chunk < 1) P.chunk = 1;
    const int max_chunk = sizeof(T) == 2 ? 2 * OBS_CHUNK : OBS_CHUNK;   // f16 tiles are rebuilt for twice the observers at once: longer chunks pay
    if (P.chunk > max_chunk) P.chunk = max_chunk;
    if (O.grid > 0) grid = O.grid;
    if (O.chunk > 0) P.chunk = O.chunk;
    grid = std::max(1, std::min(grid, tiles));
    P.chunk = std::max(1, std::min(P.chunk, (tiles + grid - 1) / grid));
    // more than one round of chunks: deal them per SM (obs_render_kernel) when every SM owns at least
    // OBS_DEAL_MIN_UNITS units, or when the grid is forced (tests: the claims and the stealing at small sizes);
    // otherwise round-robin.  With fewer units per SM the deal measured slower (DESIGN.md section 5, "Chunks dealt
    // per SM"): battle512 in float16 at 3.8 units per SM, gather64 at under 2.
    P.sms = g_sms;
    P.deal_unit = OBS_DEAL_UNIT * ctas_per_sm;
    const long chunks = (tiles + P.chunk - 1) / P.chunk;
    const bool rounds = (long)grid * P.chunk < tiles;
    P.deal = rounds && (O.grid > 0 || chunks >= (long)OBS_DEAL_MIN_UNITS * P.deal_unit * g_sms) ? c->obs_deal : nullptr;
    const int aligned = ((((size_t)P.view) | ((size_t)P.feature)) & 15) == 0;
    const int report[8] = {(int)sizeof(T), NIT, TURN ? 1 : 0, TA, grid, P.chunk, tiles, aligned};
    memcpy(c->obs_last, report, sizeof report);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    const bool timed = c->profile && !c->capturing;
    if (timed) { profile_pair(c, &e0, &e1); CUDA_CHECK(cudaEventRecord(e0, c->stream)); }
    obs_render_kernel<T, NIT, TURN, TA><<<grid, 32 * TA, smem, c->stream>>>(P);
    post_launch("obs_render_kernel");
    if (timed) CUDA_CHECK(cudaEventRecord(e1, c->stream));
}

// scratch owned by the context: the per-agent headers of n observers
static void grow_obs_hdr(Ctx *c, size_t n) {
    if (n <= c->obs_hdr_n) return;
    no_capture(c, "growing the observation header table");
    if (c->obs_hdr) { CUDA_CHECK(cudaStreamSynchronize(c->stream)); cudaFree(c->obs_hdr); }
    c->obs_hdr_n = n + n / 4 + 64;
    CUDA_CHECK(cudaMalloc(&c->obs_hdr, c->obs_hdr_n * sizeof(int4)));
}

// threads per CTA of the header pre-passes: as many observers as fit 48 KB of feature rows (*smem bytes)
static int obs_prepass_threads(int F, size_t elem, size_t *smem) {
    int threads = 256;
    while (threads > 32 && (size_t)threads * F * elem > 48 * 1024) threads >>= 1;
    *smem = (size_t)threads * F * elem;
    if (*smem > 48 * 1024) mg::fatal("feature row too long for the header kernel (%d elements)", F);
    return threads;
}

// cfg_slot: 0..5, one per (T, NIT, TURN); each owns two context slots, one per tile width
template <typename T, int NIT, bool TURN>
static void launch_obs_typed(Ctx *c, int cfg_slot, const EngineDev &hE, const ObsArgs &O, ObsParams &P, int n_total,
                             int view_count, bool with_headers = true, bool headers_only = false) {
    if (obs_all_cells_in_regs<NIT, TURN>() && view_count > NIT * 32)
        mg::fatal("render kernel NIT=%d chosen for a view of %d in-range cells", NIT, view_count);
    grow_obs_hdr(c, (size_t)n_total);
    P.hdr = c->obs_hdr;
    if (with_headers) {
        size_t hsm;
        const int threads = obs_prepass_threads(P.F, sizeof(T), &hsm);
        const int cpa = (P.cap + threads - 1) / threads;
        obs_headers_kernel<T><<<(unsigned)((size_t)P.A * cpa), threads, hsm, c->stream>>>(P, c->obs_hdr, cpa);
        post_launch("obs_headers_kernel");
    }
    if (headers_only) return;
    // the wide tile whenever it keeps at least as many warps per SM as the narrow one (always, for battle); the
    // narrow tile for records whose wide tile fits fewer warps or not at all.  O.tile forces a width: 1 narrow, 2 wide
    // (narrow when the wide tile does not fit).
    constexpr int TN = obs_tile_narrow<T>(), TW = obs_tile_wide<T>();
    const size_t lut_bytes = (size_t)(P.turn ? 4 : 1) * ((P.cells + 1) & ~1) * sizeof(int2);
    const size_t smem_n = (size_t)TN * P.rec * sizeof(T) + lut_bytes, smem_w = (size_t)TW * P.rec * sizeof(T) + lut_bytes;
    size_t need_n;
    if (smem_band(c, ATTR_OBS0 + 2 * cfg_slot, obs_render_kernel<T, NIT, TURN, TN>, smem_n, &need_n) < 0)
        mg::fatal("observation record too large for the render kernel (%zu bytes of shared memory, more than the %zu one "
                  "block may use)", need_n, c->smem_optin);
    const int ctas_w = obs_ctas_per_sm<T, NIT, TURN, TW>(c, 2 * cfg_slot + 1, smem_w);
    const int ctas_n = obs_ctas_per_sm<T, NIT, TURN, TN>(c, 2 * cfg_slot, smem_n);
    const bool wide = O.tile == 0 ? ctas_w >= 1 && ctas_w * TW >= ctas_n * TN : O.tile == 2 && ctas_w >= 1;
    if (wide) launch_obs_render<T, NIT, TURN, TW>(c, O, P, n_total, smem_w, ctas_w);
    else launch_obs_render<T, NIT, TURN, TN>(c, O, P, n_total, smem_n, ctas_n < 1 ? 1 : ctas_n);
}

static void fill_obs_params(Ctx *c, const EngineDev &hE, const ObsArgs &O, const float *mm_val, int n_total, ObsParams &P) {
    const int g = O.group;
    const GroupDev &G = hE.grp[g];
    memset(&P, 0, sizeof P);
    P.A = hE.A; P.W = hE.W; P.H = hE.H; P.G = hE.G; P.C = hE.n_channel;
    P.vw = G.view_w; P.vh = G.view_h; P.cells = G.view_w * G.view_h; P.rec = P.cells * P.C; P.F = G.feature_size;
    P.ox = G.view_xoff + G.view_x1; P.oy = G.view_yoff + G.view_y1;
    P.scale_w = (hE.W + G.view_w - 1) / G.view_w; P.scale_h = (hE.H + G.view_h - 1) / G.view_h;
    P.minimap = mm_val != nullptr;
    P.cap = G.cap; P.embedding = hE.embedding_size; P.n_action = G.n_action; P.n_total = n_total;
    P.mask = G.view_mask;
    P.off = hE.off + (size_t)g * (hE.A + 1);
    P.kind_plane = hE.kind; P.hpn_plane = hE.hpn; P.kpad = hE.kpad; P.kw = hE.kw; P.kplane = hE.kplane;
    const AgentSoA &s = G.soa[(O.curmask >> g) & 1u];
    P.x = s.x; P.y = s.y; P.id = s.id; P.act = s.act; P.last_reward = s.last_reward; P.dir = s.dir;
    P.turn = hE.turn_mode; P.body_w = G.body_w; P.body_l = G.body_l;
    P.mm = mm_val ? c->mm_pad : nullptr; P.mm_stride = mm_val ? c->mm_stride : 0;
    P.view = O.view; P.feature = O.feature;
    const int stride = 2 + (hE.minimap_mode ? 1 : 0);
    for (int j = 0; j < hE.G; ++j) {
        int rel = j - g; if (rel < 0) rel += hE.G;
        const int ch = hE.channel_base + rel * stride;                 // make_channel_trans, GridWorld.cc:897-913
        P.mm_ch[j] = ch + 2;
        P.grp_ch[j] = ch;
    }
}

static void launch_obs_dispatch(Ctx *c, const EngineDev &hE, const ObsArgs &O, ObsParams &P, int n_total, bool with_headers, bool headers_only) {
    const int vc = hE.grp[O.group].view_count;
    const bool small_view = vc <= 4 * 32;                       // in-range view cells held in registers: 4 or 8 per lane
    if (hE.turn_mode) {                                         // headings: per-heading LUTs in shared memory (NIT = 8 code path)
        if (O.half) launch_obs_typed<__half, 8, true>(c, 0, hE, O, P, n_total, vc, with_headers, headers_only);
        else launch_obs_typed<float, 8, true>(c, 1, hE, O, P, n_total, vc, with_headers, headers_only);
    } else if (O.half) {
        if (small_view) launch_obs_typed<__half, 4, false>(c, 2, hE, O, P, n_total, vc, with_headers, headers_only);
        else launch_obs_typed<__half, 8, false>(c, 3, hE, O, P, n_total, vc, with_headers, headers_only);
    } else {
        if (small_view) launch_obs_typed<float, 4, false>(c, 4, hE, O, P, n_total, vc, with_headers, headers_only);
        else launch_obs_typed<float, 8, false>(c, 5, hE, O, P, n_total, vc, with_headers, headers_only);
    }
}

void launch_obs(Ctx *c, const EngineDev *, const EngineDev &hE, const ObsArgs &O, const float *mm_val, int n_total) {
    DeviceGuard guard(c);
    ObsParams P;
    fill_obs_params(c, hE, O, mm_val, n_total, P);
    launch_obs_dispatch(c, hE, O, P, n_total, true, false);
}

void obs_launch_report(const Ctx *c, int out[8]) { memcpy(out, c->obs_last, sizeof c->obs_last); }
void step_launch_report(const Ctx *c, int out[10]) { memcpy(out, c->step_last, sizeof c->step_last); }

// ------------------------------------------------------------------------------------------------
// global state (magent_b200_get_global_state): state_compose_cell of every map cell of every arena, [A][H][W][C] in T.
// The output is one dense stream of 16-byte vectors, each written once.  A CTA takes tiles of GS_TILE consecutive
// output elements (16 KB of float32, 8 KB of half) and composes each tile in shared memory, one thread per map cell:
// consecutive threads read consecutive kind bytes of a plane row, and only agent cells below max hp load their hp_norm
// value.  Then the tile goes out with coalesced 16-byte stores; a warp's stores cover 512 contiguous bytes.  Only a
// ragged last vector (A*H*W*C not a multiple of the vector) is stored element by element.
//
// Composing per cell rather than per output vector keeps the work per element to one select chain and one shared store:
// an output vector of 4 or 8 elements straddles cells whenever C does not divide it (battle: C = 5), and composing it
// directly costs a kind and an hp lookup per element.
enum { GS_THREADS = 256, GS_TILE = 4096, GS_BATCH = 4 };
struct StateParams {
    const unsigned char *kind;       // EngineDev::kind, padded
    const float *hpn;                // EngineDev::hpn, padded
    int H, W, kpad, kw;
    long kplane;
    int C, base;                     // state_channels, state_base
    long long n_elem;                // A*H*W*C
    void *out;
};
template <typename T> constexpr int gs_vec_elems() { return 16 / (int)sizeof(T); }

template <typename T>
__global__ void __launch_bounds__(GS_THREADS) global_state_kernel(const __grid_constant__ StateParams P) {
    constexpr int VE = gs_vec_elems<T>(), TILE_V = GS_TILE / VE;
    __shared__ __align__(16) T s_out[GS_TILE];
    const long long n_tiles = (P.n_elem + GS_TILE - 1) / GS_TILE, n_full = P.n_elem / VE;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long e0 = tile * GS_TILE;
        const int ne = (int)min((long long)GS_TILE, P.n_elem - e0);
        const long long c0 = e0 / P.C;                            // first cell of the tile and the tile's offset inside it
        const int r0 = (int)(e0 - c0 * P.C);
        const int nc = (r0 + ne - 1) / P.C + 1;
        const int row0 = (int)(c0 / P.W), x0 = (int)(c0 - (long long)row0 * P.W);      // row = a * H + y
        for (int i0 = threadIdx.x; i0 < nc; i0 += GS_THREADS * GS_BATCH) {
            long pc[GS_BATCH];
            int t[GS_BATCH];
            float hp[GS_BATCH];
#pragma unroll
            for (int q = 0; q < GS_BATCH; ++q) {                  // the batch's kind loads are all in flight at once
                const int i = i0 + q * GS_THREADS;
                const int dr = (x0 + i) / P.W, x = x0 + i - dr * P.W;
                const int row = row0 + dr, a = row / P.H, y = row - a * P.H;
                pc[q] = a * P.kplane + (long)(y + P.kpad) * P.kw + x + P.kpad;
                t[q] = i < nc ? (int)__ldg(P.kind + pc[q]) : KIND_EMPTY;
            }
#pragma unroll
            for (int q = 0; q < GS_BATCH; ++q) hp[q] = state_needs_hpn(t[q]) ? __ldg(P.hpn + pc[q]) : 1.0f;
#pragma unroll
            for (int q = 0; q < GS_BATCH; ++q) {
                const int le = (i0 + q * GS_THREADS) * P.C - r0;  // tile element of the cell's channel 0
                for (int ch = 0; ch < P.C; ++ch)
                    if (le + ch >= 0 && le + ch < ne) s_out[le + ch] = ObsOut<T>::cv(state_cell_value(t[q], hp[q], ch, P.base));
            }
        }
        __syncthreads();
        const long long v0 = e0 / VE;
        for (int lv = threadIdx.x; lv < TILE_V; lv += GS_THREADS) {
            const long long v = v0 + lv;
            if (v < n_full) {
                ((uint4 *)P.out)[v] = ((const uint4 *)s_out)[lv];
            } else if (lv * VE < ne) {                            // the ragged end of the output
                for (int j = lv * VE; j < ne; ++j) ((T *)P.out)[e0 + j] = s_out[j];
            }
        }
        __syncthreads();
    }
}

template <typename T>
static void launch_global_state_typed(Ctx *c, const StateParams &P, int slot) {
    Ctx::ObsCfg &cfg = c->state_cfg[slot];
    if (cfg.smem != 0) {
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cfg.ctas_per_sm, global_state_kernel<T>, GS_THREADS, 0));
        if (cfg.ctas_per_sm < 1) mg::fatal("global_state_kernel does not fit an SM");
        cfg.smem = 0;
    }
    const long long tiles = (P.n_elem + GS_TILE - 1) / GS_TILE;
    const long long resident = (long long)cfg.ctas_per_sm * c->sms;
    const unsigned grid = (unsigned)(tiles < resident ? tiles : resident);
    if (grid == 0) return;
    global_state_kernel<T><<<grid, GS_THREADS, 0, c->stream>>>(P);
    post_launch("global_state_kernel");
}

void launch_global_state(Ctx *c, const EngineDev *, const EngineDev &hE, void *out, int half) {
    DeviceGuard guard(c);
    if ((uintptr_t)out & 15) mg::fatal("the global state buffer must be 16-byte aligned (got %p)", out);
    StateParams P;
    memset(&P, 0, sizeof P);
    P.kind = hE.kind; P.hpn = hE.hpn;
    P.H = hE.H; P.W = hE.W; P.kpad = hE.kpad; P.kw = hE.kw; P.kplane = hE.kplane;
    P.C = state_channels(hE); P.base = state_base(hE);
    P.n_elem = (long long)hE.A * hE.H * hE.W * P.C;
    P.out = out;
    if (half) launch_global_state_typed<__half>(c, P, 1);
    else launch_global_state_typed<float>(c, P, 0);
}

// ------------------------------------------------------------------------------------------------
// restore_kernel: arenas of a snapshot copied over live arenas (Engine::restore_arenas, DESIGN.md §5).
//
// Work items are (arena, chunk) pairs, K chunks of about RS_CHUNK_BYTES per arena, dealt grid-stride to at most one wave
// of CTAs.  Large chunks: an item walks some 30 segments one after the other, and a thread needs several vectors of each
// in flight (battle512 on H100: 16 KB chunks restore every arena in 1.14 ms, 512 KB chunks in 0.25 ms).  An item
// reads its arena's source (src[a], or a itself when src is null and the arena's last step reported done) and is
// finished at once when there is none, so a restore of nothing costs one launch of idle CTAs.  Otherwise chunk k copies
// the k-th of K slices of every segment of the arena: the occ, kind, hp_norm and food planes, the snapshot's n[g][s]
// records of every SoA field, and the -1 fill of claim_head.  A segment's slices are 16-byte vectors where source and
// destination agree modulo 16 bytes (SoA capacities are multiples of 64; a plane does when its per-arena size is a
// multiple of 16 bytes or the arena restores itself), else words or bytes; the unaligned head and the ragged tail go
// to chunk 0.  Chunk 0 also copies counts and header.
//
// The done words are written by restore_finish_kernel afterwards: with a null src every chunk of an arena reads its
// arena's done word to decide, so no chunk may change it.
enum { RS_THREADS = 256, RS_CHUNK_BYTES = 512 << 10, RS_MAX_CHUNKS = 256, RS_SOA_FIELDS = 11, RS_SOA_WORDS = 8 };
static_assert(sizeof(AgentSoA) == RS_SOA_FIELDS * sizeof(void *), "AgentSoA: 8 four-byte fields, then 3 byte fields");
static_assert(offsetof(ArenaHdr, rng) == 0 && offsetof(ArenaHdr, rng_next) == 4 && sizeof(ArenaHdr) % 4 == 0,
              "keep_rng skips the first two words of the header");

struct RestoreParams {
    const int *src;                  // device int32[A] or nullptr (done-driven)
    const int *done;                 // EngineDev::done
    int A, G, K, keep_rng;
    long cells, kplane;              // W*H, padded plane
    int *occ, *claim; unsigned char *kind; float *hpn, *food;
    ArenaHdr *hdr; int *n, *dead_ct;
    int cap[MG_MAX_GROUPS];
    AgentSoA soa[MG_MAX_GROUPS];     // the live ping-pong buffer
    SnapDev S;
};

// slice k of K of a copy in units of T; dst and src agree modulo sizeof(T)
template <typename T>
__device__ __forceinline__ void rs_copy_as(unsigned char *dst, const unsigned char *src, long bytes, int k, int K) {
    constexpr long U = sizeof(T);
    const long head = min(bytes, (long)((U - ((uintptr_t)dst & (U - 1))) & (U - 1)));
    const long nv = (bytes - head) / U;
    if (k == 0) {
        for (long i = threadIdx.x; i < head; i += RS_THREADS) dst[i] = src[i];
        for (long i = head + nv * U + threadIdx.x; i < bytes; i += RS_THREADS) dst[i] = src[i];
    }
    T *d = (T *)(dst + head);
    const T *s = (const T *)(src + head);
    const long v1 = nv * (k + 1) / K;
#pragma unroll 4
    for (long v = nv * k / K + threadIdx.x; v < v1; v += RS_THREADS) d[v] = __ldg(s + v);
}

// 16-byte vectors where source and destination agree modulo 16 (every SoA field, and the planes of a restore from the
// same arena or of maps whose plane size is a multiple of 16 bytes), else words or bytes
__device__ __forceinline__ void rs_copy(unsigned char *dst, const unsigned char *src, long bytes, int k, int K) {
    const unsigned rel = (unsigned)((uintptr_t)dst - (uintptr_t)src) & 15u;
    if (rel == 0) rs_copy_as<uint4>(dst, src, bytes, k, K);
    else if ((rel & 3u) == 0) rs_copy_as<unsigned>(dst, src, bytes, k, K);
    else rs_copy_as<unsigned char>(dst, src, bytes, k, K);
}

__device__ __forceinline__ void rs_fill_ff(unsigned char *dst, long bytes, int k, int K) {
    const long head = min(bytes, (long)((16 - ((uintptr_t)dst & 15)) & 15));
    const long nv = (bytes - head) >> 4;
    if (k == 0) {
        for (long i = threadIdx.x; i < head; i += RS_THREADS) dst[i] = 0xff;
        for (long i = head + (nv << 4) + threadIdx.x; i < bytes; i += RS_THREADS) dst[i] = 0xff;
    }
    uint4 *d = (uint4 *)(dst + head);
    const long v1 = nv * (k + 1) / K;
    for (long v = nv * k / K + threadIdx.x; v < v1; v += RS_THREADS) d[v] = make_uint4(~0u, ~0u, ~0u, ~0u);
}

__device__ __forceinline__ int restore_source(const int *src, const int *done, int A, int a) {
    const int s = src ? __ldg(src + a) : ((__ldg(done + a) & 1) ? a : -1);
    return s >= 0 && s < A ? s : -1;
}

__global__ void __launch_bounds__(RS_THREADS, 4) restore_kernel(const __grid_constant__ RestoreParams P) {
    const long items = (long)P.A * P.K;
    for (long item = blockIdx.x; item < items; item += gridDim.x) {
        const int a = (int)(item / P.K), k = (int)(item - (long)a * P.K);
        const int s = restore_source(P.src, P.done, P.A, a);
        if (s < 0) continue;
        rs_copy((unsigned char *)(P.occ + a * P.cells), (const unsigned char *)(P.S.occ + s * P.cells), P.cells * 4, k, P.K);
        rs_fill_ff((unsigned char *)(P.claim + a * P.cells), P.cells * 4, k, P.K);
        rs_copy(P.kind + a * P.kplane, P.S.kind + s * P.kplane, P.kplane, k, P.K);
        rs_copy((unsigned char *)(P.hpn + a * P.kplane), (const unsigned char *)(P.S.hpn + s * P.kplane), P.kplane * 4, k, P.K);
        if (P.food)
            rs_copy((unsigned char *)(P.food + a * P.cells), (const unsigned char *)(P.S.food + s * P.cells), P.cells * 4, k, P.K);
        for (int g = 0; g < P.G; ++g) {
            const long ns = __ldg(P.S.n + g * P.A + s);
            unsigned char *const *dst = (unsigned char *const *)&P.soa[g];
            const unsigned char *const *from = (const unsigned char *const *)&P.S.soa[g];
#pragma unroll                                            // (a rolled loop keeps a stack frame and spills)
            for (int f = 0; f < RS_SOA_FIELDS; ++f) {
                const long esz = f < RS_SOA_WORDS ? 4 : 1;
                rs_copy(dst[f] + (long)a * P.cap[g] * esz, from[f] + (long)s * P.S.cap[g] * esz, ns * esz, k, P.K);
            }
            if (k == 0 && threadIdx.x == 0) {
                P.n[g * P.A + a] = (int)ns;
                P.dead_ct[g * P.A + a] = __ldg(P.S.dead_ct + g * P.A + s);
            }
        }
        if (k == 0) {
            int *h = (int *)(P.hdr + a);
            const int *hs = (const int *)(P.S.hdr + s);
            for (int w = threadIdx.x + (P.keep_rng ? 2 : 0); w < (int)(sizeof(ArenaHdr) / 4); w += RS_THREADS) h[w] = __ldg(hs + w);
        }
    }
}

// the done words of the restored arenas, then the offset table (offsets_kernel's scan, every group in one CTA)
__global__ void __launch_bounds__(1024) restore_finish_kernel(const EngineDev *gE, const int *src, const int *snap_done) {
    const int A = gE->A;
    for (int a = threadIdx.x; a < A; a += blockDim.x) {
        const int s = restore_source(src, gE->done, A, a);      // this thread alone reads and writes done[a]
        if (s >= 0) gE->done[a] = snap_done[s];
    }
    __syncthreads();
    for (int g = 0; g < gE->G; ++g) offsets_group(gE, g);
}

void launch_restore(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, const SnapDev &S, const int *src,
                    int keep_rng) {
    DeviceGuard guard(c);
    if (c->restore_ctas_per_sm == 0) {
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c->restore_ctas_per_sm, restore_kernel, RS_THREADS, 0));
        if (c->restore_ctas_per_sm < 1) mg::fatal("restore_kernel does not fit an SM");
    }
    RestoreParams P;
    memset(&P, 0, sizeof P);
    P.src = src; P.done = hE.done;
    P.A = hE.A; P.G = hE.G; P.keep_rng = keep_rng ? 1 : 0;
    P.cells = (long)hE.W * hE.H; P.kplane = hE.kplane;
    P.occ = hE.occ; P.claim = hE.claim_head; P.kind = hE.kind; P.hpn = hE.hpn; P.food = hE.food;
    P.hdr = hE.hdr; P.n = hE.n; P.dead_ct = hE.dead_ct;
    // chunks per arena from the bytes a restored arena moves at most (the SoA part at the snapshot's capacity)
    long bytes = P.cells * (P.food ? 12 : 8) + P.kplane * 5;
    for (int g = 0; g < hE.G; ++g) {
        P.cap[g] = hE.grp[g].cap;
        P.soa[g] = hE.grp[g].soa[(curmask >> g) & 1u];
        bytes += (long)S.cap[g] * (4 * RS_SOA_WORDS + (RS_SOA_FIELDS - RS_SOA_WORDS));
    }
    const long K = (bytes + RS_CHUNK_BYTES - 1) / RS_CHUNK_BYTES;
    P.K = (int)(K < 1 ? 1 : K > RS_MAX_CHUNKS ? RS_MAX_CHUNKS : K);
    P.S = S;
    const long items = (long)P.A * P.K, resident = (long)c->restore_ctas_per_sm * c->sms;
    restore_kernel<<<(unsigned)(items < resident ? items : resident), RS_THREADS, 0, c->stream>>>(P);
    post_launch("restore_kernel");
    restore_finish_kernel<<<1, 1024, 0, c->stream>>>(dE, src, S.done);
    post_launch("restore_finish_kernel");
}

// ------------------------------------------------------------------------------------------------
// stable slots (magent_b200_get_slots, slot_phases.h).  One CTA per arena: the arena's [S] block of slot_row is filled
// with -1, then every row of the arena (the device-side offsets say how many) looks its agent's id up in the slot table,
// writes a * S + slot to row_slot and scatters its row into slot_row.  Consecutive threads take consecutive rows and
// slots, so the fill and the row_slot stores are coalesced, and so is the scatter while slots still follow the rows
// (culls only open gaps).  The rows from the device-side total up to n_bound get -1, dealt over every CTA.
constexpr int SLOT_THREADS = 256;

__global__ void __launch_bounds__(SLOT_THREADS) slots_kernel(const int *off, const int *ids, int cap, const SlotDev *T,
                                                             int A, int S, int *row_slot, int *slot_row, int n_bound) {
    const int a = blockIdx.x;
    const int *tab = T->tab;
    const int id_cap = T->id_cap;
    if (slot_row) {
        for (int q = threadIdx.x; q < S; q += SLOT_THREADS) slot_row[(long)a * S + q] = -1;
        __syncthreads();
    }
    const int o0 = off[a];
    const int cnt = min(off[a + 1] - o0, n_bound - o0);         // never beyond the caller's buffer
    const int *id = ids + (long)a * cap;
    for (int i = threadIdx.x; i < cnt; i += SLOT_THREADS) {
        const int flat = slot_flat(tab, id_cap, a, __ldg(id + i), S);
        if (row_slot) row_slot[o0 + i] = flat;
        if (slot_row && flat >= 0) slot_row[flat] = o0 + i;
    }
    if (row_slot)
        for (int r = off[A] + a * SLOT_THREADS + threadIdx.x; r < n_bound; r += A * SLOT_THREADS) row_slot[r] = -1;
}

void launch_slots(Ctx *c, const EngineDev *, const EngineDev &hE, const SlotDev *T, unsigned curmask, int group, int S,
                  int *row_slot, int *slot_row, int n_bound) {
    DeviceGuard guard(c);
    const GroupDev &D = hE.grp[group];
    slots_kernel<<<(unsigned)hE.A, SLOT_THREADS, 0, c->stream>>>(hE.off + (size_t)group * (hE.A + 1),
                                                                 D.soa[(curmask >> group) & 1u].id, D.cap, T, hE.A, S,
                                                                 row_slot, slot_row, n_bound);
    post_launch("slots_kernel");
}

// the slot rows of the arenas a restore is about to replace (restore_source decides, before restore_finish_kernel
// rewrites the done words): the snapshot row's counters and id -> slot entries, at most the live table's width
__global__ void __launch_bounds__(SLOT_THREADS) restore_slots_kernel(const SlotDev *T, const int *snap_tab,
                                                                     int snap_id_cap, const int *src, const int *done,
                                                                     int A) {
    const int a = blockIdx.x;
    const int s = restore_source(src, done, A, a);
    if (s < 0) return;
    const int id_cap = T->id_cap;
    int *dst = T->tab + (long)a * slot_row_stride(id_cap);
    const int *from = snap_tab + (long)s * slot_row_stride(snap_id_cap);
    const long n = slot_row_stride(min(id_cap, snap_id_cap));
    for (long q = threadIdx.x; q < n; q += SLOT_THREADS) dst[q] = __ldg(from + q);
}

void launch_restore_slots(Ctx *c, const EngineDev *, const EngineDev &hE, const SlotDev *T, const int *snap_tab,
                          int snap_id_cap, const int *src) {
    DeviceGuard guard(c);
    restore_slots_kernel<<<(unsigned)hE.A, SLOT_THREADS, 0, c->stream>>>(T, snap_tab, snap_id_cap, src, hE.done, hE.A);
    post_launch("restore_slots_kernel");
}

__global__ void __launch_bounds__(256) arena_done_kernel(const EngineDev *gE, int *out) {
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < gE->A; a += gridDim.x * blockDim.x) out[a] = gE->done[a] & 1;
}

void launch_arena_done(Ctx *c, const EngineDev *dE, const EngineDev &hE, int *out) {
    DeviceGuard guard(c);
    arena_done_kernel<<<(hE.A + 255) / 256, 256, 0, c->stream>>>(dE, out);
    post_launch("arena_done_kernel");
}

// ------------------------------------------------------------------------------------------------
// env_step's done word
__global__ void __launch_bounds__(256) done_reduce_kernel(const EngineDev *gE, int *out) {
    __shared__ int all_s;
    if (threadIdx.x == 0) all_s = 1;
    __syncthreads();
    int all = 1;
    for (int a = threadIdx.x; a < gE->A; a += blockDim.x) all &= gE->done[a] & 1;
    if (!all) all_s = 0;
    __syncthreads();
    if (threadIdx.x == 0) *out = all_s;
}

void read_done(Ctx *c, const EngineDev &hE, int *done_words) {
    no_capture(c, "env_step with a host `done`");
    DeviceGuard guard(c);
    if ((size_t)hE.A > c->pin_done_n) {
        if (c->pin_done) cudaFreeHost(c->pin_done);
        c->pin_done_n = (size_t)hE.A + 64;
        CUDA_CHECK(cudaHostAlloc((void **)&c->pin_done, c->pin_done_n * sizeof(int), cudaHostAllocDefault));
    }
    CUDA_CHECK(cudaMemcpyAsync(c->pin_done, hE.done, (size_t)hE.A * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    memcpy(done_words, c->pin_done, (size_t)hE.A * sizeof(int));
}

void counts_fetch_begin(Ctx *c, const int *dev_off, size_t n_ints) {
    no_capture(c, "the asynchronous count fetch");
    DeviceGuard guard(c);
    if (n_ints > c->pin_counts_n) {
        if (c->pin_counts) { CUDA_CHECK(cudaStreamSynchronize(c->stream)); cudaFreeHost(c->pin_counts); }
        c->pin_counts_n = n_ints + 64;
        CUDA_CHECK(cudaHostAlloc((void **)&c->pin_counts, c->pin_counts_n * sizeof(int), cudaHostAllocDefault));
    }
    CUDA_CHECK(cudaMemcpyAsync(c->pin_counts, dev_off, n_ints * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaEventRecord(c->ev_counts, c->stream));
}
const int *counts_fetch_wait(Ctx *c) {
    DeviceGuard guard(c);
    CUDA_CHECK(cudaEventSynchronize(c->ev_counts));
    return c->pin_counts;
}

void launch_done_to_device(Ctx *c, const EngineDev *dE, const EngineDev &, int *dev_done) {
    DeviceGuard guard(c);
    done_reduce_kernel<<<1, 256, 0, c->stream>>>(dE, dev_done);
    post_launch("done_reduce_kernel");
}

// ------------------------------------------------------------------------------------------------
// Host-buffer observations: the wire format (backend.h WireHdr / WireMark, DESIGN.md 6b).
//
// The reference ABI wants one dense float32 record per observer in HOST memory (4732 B for battle, 97 % zeros).
// PCIe moves ~55 GB/s; the host's memory system takes several times that.  So the GPU does the gather -- which cells of
// the view window show something, and what (Map::extract_view, Map.cc:129-207) -- and ships the answer as a compact
// record of ~60 B per observer; host threads then write the dense bytes (host_expand.cc).
//
// obs_wire_kernel: one warp per observer, ABI order.  Lanes stride over the in-range view cells (same LUT as the render
// kernel), load the kind byte and, for occupied cells, hp / max_hp; a ballot compacts the non-empty cells into the
// observer's slot row (worst-case sized, written sparsely).  Lane 0 writes the header and adds the count to the
// observer's chunk total.  wire_scan_kernel turns chunk totals into chunk bases; wire_compact_kernel copies the slot
// rows of a chunk into the contiguous mark stream the host reads.
__global__ void __launch_bounds__(256) obs_wire_kernel(const __grid_constant__ ObsParams P, WireHdr *whdr, WireMark *slots,
                                                       int slot_stride, int *chunk_total) {
    extern __shared__ __align__(16) unsigned char wire_smem[];
    int2 *lut = (int2 *)wire_smem;
    __shared__ int n_in_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lut_stride = (P.cells + 1) & ~1;
    if (warp == 0) {                                          // compact the view mask (Range.h:104-189), as obs_render_kernel does
        int k = 0;
        for (int base = 0; base < P.cells; base += 32) {
            const int cell = base + lane;
            const bool in = cell < P.cells && P.mask[cell];
            const unsigned bal = __ballot_sync(0xffffffffu, in);
            if (in) {
                const int vy = cell / P.vw, vx = cell - vy * P.vw;
                const int q = k + __popc(bal & ((1u << lane) - 1u));
                if (!P.turn) lut[q] = make_int2(cell * P.C, (P.oy + vy) * P.kw + P.ox + vx);
                else {
                    for (int d = 0; d < 4; ++d) {                       // one LUT per heading (Map.cc:140-146, 515-560)
                        int rx = 0, ry = 0, dx, dy;
                        if (d == DIR_SOUTH) { rx = P.body_w - 1; ry = P.body_l - 1; }
                        else if (d == DIR_WEST) ry = P.body_w - 1;
                        else if (d == DIR_EAST) rx = P.body_l - 1;
                        const int ex = P.ox + vx, ey = P.oy + vy;
                        if (d == DIR_NORTH) { dx = ex; dy = ey; }
                        else if (d == DIR_SOUTH) { dx = -ex; dy = -ey; }
                        else if (d == DIR_WEST) { dx = ey; dy = -ex; }
                        else { dx = -ey; dy = ex; }
                        lut[d * lut_stride + q] = make_int2(cell * P.C, (ry + dy) * P.kw + rx + dx);
                    }
                }
            }
            k += __popc(bal);
        }
        if (lane == 0) n_in_s = k;
    }
    __syncthreads();
    const int n_in = n_in_s;
    const int warps = gridDim.x * (blockDim.x >> 5);
    for (int o = blockIdx.x * (blockDim.x >> 5) + warp; o < P.n_total; o += warps) {
        const int4 h = P.hdr[o];                              // {x, y, arena, self cell | heading << 16}
        const long pb = h.z * P.kplane + (long)(h.y + P.kpad) * P.kw + h.x + P.kpad;
        const unsigned char *kp = P.kind_plane + pb;
        const float *hpnp = P.hpn_plane + pb;
        const int2 *l = lut + (P.turn ? ((h.w >> 16) & 3) * lut_stride : 0);
        WireMark *row = slots + (size_t)o * slot_stride;
        int running = 0;
        for (int base = 0; base < n_in; base += 32) {
            const int k = base + lane;
            int t = 0;
            int2 lk = make_int2(0, 0);
            if (k < n_in) { lk = l[k]; t = __ldg(kp + lk.y); }
            const unsigned bal = __ballot_sync(0xffffffffu, t != 0);
            if (t != 0) {
                WireMark m;
                if (t == KIND_WALL) { m.off = (unsigned)lk.x; m.val = 0.0f; }
                else if (t == KIND_FOOD) { m.off = (unsigned)lk.x + 1u; m.val = 0.0f; }
                else { m.off = (unsigned)(lk.x + P.grp_ch[kind_group(t)]) | WIRE_HAS_HP; m.val = (t & KIND_FULL) ? 1.0f : __ldg(hpnp + lk.y); }
                row[running + __popc(bal & ((1u << lane) - 1u))] = m;
            }
            running += __popc(bal);
        }
        if (lane == 0) {
            WireHdr w;
            w.arena = h.z;
            w.self_cell = (unsigned short)(h.w & 0xffff);
            w.count = (unsigned short)running;
            whdr[o] = w;
            if (running) atomicAdd(&chunk_total[o / WIRE_CHUNK], running);
        }
    }
}

// dynamic shared memory of obs_wire_kernel: the view LUT of the group, one per heading in turn_mode.  The kernel does not
// opt in to more than the default per-block limit: a larger view takes the dense path (smem_fits SMEM_OBS_WIRE).
static size_t wire_dyn_smem(const EngineDev &hE, int group) {
    const GroupDev &G = hE.grp[group];
    return (size_t)(hE.turn_mode ? 4 : 1) * ((G.view_w * G.view_h + 1) & ~1) * sizeof(int2);
}

__global__ void __launch_bounds__(1024) wire_scan_kernel(const int *chunk_total, long long *base, int n_chunks) {
    __shared__ long long carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int tile = 0; tile < n_chunks; tile += blockDim.x) {
        const int cidx = tile + threadIdx.x;
        const int v = cidx < n_chunks ? chunk_total[cidx] : 0;
        int tot;
        const int ex = block_excl_scan(v, tot);
        const long long carry = carry_s;
        if (cidx < n_chunks) base[cidx] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) base[n_chunks] = carry_s;
}

__global__ void __launch_bounds__(256) wire_compact_kernel(const WireHdr *whdr, const WireMark *slots, int slot_stride,
                                                           const long long *base, WireMark *stream, int n_total, int n_chunks) {
    __shared__ int off_s[WIRE_CHUNK];
    __shared__ unsigned short cnt_s[WIRE_CHUNK];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        const int o0 = ch * WIRE_CHUNK, cnt_obs = min(WIRE_CHUNK, n_total - o0);
        int running = 0;
        for (int tile = 0; tile < WIRE_CHUNK; tile += blockDim.x) {
            const int i = tile + threadIdx.x;
            const int v = i < cnt_obs ? (int)whdr[o0 + i].count : 0;
            int tot;
            const int ex = block_excl_scan(v, tot);
            off_s[i] = running + ex;
            cnt_s[i] = (unsigned short)v;
            running += tot;
        }
        __syncthreads();
        WireMark *dst = stream + base[ch];
        for (int i = warp; i < cnt_obs; i += nw) {
            const int n = cnt_s[i], off = off_s[i];
            const WireMark *src = slots + (size_t)(o0 + i) * slot_stride;
            for (int k = lane; k < n; k += 32) dst[off + k] = src[k];
        }
        __syncthreads();
    }
}

template <class T>
static void grow_dev(Ctx *c, T *&p, size_t &have, size_t need) {
    if (need <= have) return;
    if (p) { CUDA_CHECK(cudaStreamSynchronize(c->stream)); CUDA_CHECK(cudaStreamSynchronize(c->copy)); cudaFree(p); }
    have = need + need / 4 + 64;
    CUDA_CHECK(cudaMalloc((void **)&p, have * sizeof(T)));
}
template <class T>
static void grow_pinned(Ctx *c, T *&p, size_t &have, size_t need) {
    if (need <= have) return;
    if (p) { CUDA_CHECK(cudaStreamSynchronize(c->copy)); cudaFreeHost(p); }
    have = need + need / 2 + 1024;
    CUDA_CHECK(cudaHostAlloc((void **)&p, have * sizeof(T), cudaHostAllocDefault));
}

void obs_wire_begin(Ctx *c, const EngineDev *, const EngineDev &hE, const ObsArgs &O, const float *mm_val, int n_total,
                    WireDesc *out) {
    no_capture(c, "an observation into host memory");
    DeviceGuard guard(c);
    ObsParams P;
    fill_obs_params(c, hE, O, mm_val, n_total, P);
    launch_obs_dispatch(c, hE, O, P, n_total, true, true);               // headers + feature rows (into O.feature)
    const int n_in = hE.grp[O.group].view_count;
    const int n_chunks = (n_total + WIRE_CHUNK - 1) / WIRE_CHUNK;
    grow_dev(c, c->wire_slots, c->wire_slots_n, (size_t)n_total * n_in);
    grow_dev(c, c->wire_hdr, c->wire_hdr_n, (size_t)n_total);
    {
        size_t have = c->wire_base_n;
        grow_dev(c, c->wire_base, c->wire_base_n, (size_t)n_chunks + 1);
        if (c->wire_base_n != have) {
            if (c->wire_chunk_total) cudaFree(c->wire_chunk_total);
            CUDA_CHECK(cudaMalloc((void **)&c->wire_chunk_total, c->wire_base_n * sizeof(int)));
        }
    }
    CUDA_CHECK(cudaMemsetAsync(c->wire_chunk_total, 0, (size_t)n_chunks * sizeof(int), c->stream));
    {
        const size_t smem = wire_dyn_smem(hE, O.group);
        if (smem_band(c, ATTR_WIRE, obs_wire_kernel, smem) != 0)
            mg::fatal("view too large for the wire kernel (%zu bytes of shared memory)", smem);
        int grid = (n_total + 7) / 8;
        if (grid > 8 * c->sms) grid = 8 * c->sms;
        obs_wire_kernel<<<grid, 256, smem, c->stream>>>(P, c->wire_hdr, c->wire_slots, n_in, c->wire_chunk_total);
        post_launch("obs_wire_kernel");
        wire_scan_kernel<<<1, 1024, 0, c->stream>>>(c->wire_chunk_total, c->wire_base, n_chunks);
        post_launch("wire_scan_kernel");
    }
    grow_pinned(c, c->h_wire_base, c->h_wire_base_n, (size_t)n_chunks + 1);
    CUDA_CHECK(cudaMemcpyAsync(c->h_wire_base, c->wire_base, ((size_t)n_chunks + 1) * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaEventRecord(c->ev_done, c->stream));                  // totals on their way
    if (mm_val) {
        grow_pinned(c, c->h_mm, c->h_mm_n, (size_t)hE.A * c->mm_stride);
        CUDA_CHECK(cudaMemcpyAsync(c->h_mm, c->mm_pad, (size_t)hE.A * c->mm_stride * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    grow_pinned(c, c->h_wire_hdr, c->h_wire_hdr_n, (size_t)n_total);
    // the mark stream cannot be longer than every in-range cell of every observer; it is sized from the real total below
    CUDA_CHECK(cudaEventSynchronize(c->ev_done));
    const long long total_marks = c->h_wire_base[n_chunks];
    grow_dev(c, c->wire_stream, c->wire_stream_n, (size_t)total_marks + 1);
    grow_pinned(c, c->h_wire_marks, c->h_wire_marks_n, (size_t)total_marks + 1);
    {
        int grid = n_chunks < 8 * c->sms ? n_chunks : 8 * c->sms;
        wire_compact_kernel<<<grid, 256, 0, c->stream>>>(c->wire_hdr, c->wire_slots, n_in, c->wire_base, c->wire_stream, n_total, n_chunks);
        post_launch("wire_compact_kernel");
    }
    CUDA_CHECK(cudaEventRecord(c->ev_wire, c->stream));
    // queue the copies wave by wave on the copy stream
    CUDA_CHECK(cudaStreamWaitEvent(c->copy, c->ev_wire, 0));
    int cpw = (n_chunks + 7) / 8;
    if (cpw < 4) cpw = 4;
    const int n_waves = (n_chunks + cpw - 1) / cpw;
    while ((int)c->wave_events.size() < n_waves) {
        cudaEvent_t e; CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->wave_events.push_back(e);
    }
    for (int q = 0; q < n_waves; ++q) {
        const int half = (n_waves + 1) / 2;
        const int w = (q & 1) ? half + (q >> 1) : (q >> 1);             // 0, half, 1, half + 1, ...
        out->wave_order[q] = w;
        const int c0 = w * cpw, c1 = (c0 + cpw < n_chunks) ? c0 + cpw : n_chunks;
        const size_t o0 = (size_t)c0 * WIRE_CHUNK, o1 = (size_t)c1 * WIRE_CHUNK < (size_t)n_total ? (size_t)c1 * WIRE_CHUNK : (size_t)n_total;
        CUDA_CHECK(cudaMemcpyAsync(c->h_wire_hdr + o0, c->wire_hdr + o0, (o1 - o0) * sizeof(WireHdr), cudaMemcpyDeviceToHost, c->copy));
        const long long m0 = c->h_wire_base[c0], m1 = c->h_wire_base[c1];
        if (m1 > m0) CUDA_CHECK(cudaMemcpyAsync(c->h_wire_marks + m0, c->wire_stream + m0, (size_t)(m1 - m0) * sizeof(WireMark), cudaMemcpyDeviceToHost, c->copy));
        CUDA_CHECK(cudaEventRecord(c->wave_events[w], c->copy));
    }
    c->waves_queued = n_waves;
    out->hdr = c->h_wire_hdr; out->marks = c->h_wire_marks; out->chunk_base = c->h_wire_base;
    out->mm = mm_val ? c->h_mm : nullptr; out->mm_stride = mm_val ? c->mm_stride : 0;
    out->n_total = n_total; out->n_chunks = n_chunks; out->n_waves = n_waves; out->chunks_per_wave = cpw;
}

void obs_wire_wait(Ctx *c, int wave) {
    DeviceGuard guard(c);
    CUDA_CHECK(cudaEventSynchronize(c->wave_events[wave]));
}

void dma_d2h_async(Ctx *c, void *dst, const void *src, size_t bytes) {
    DeviceGuard guard(c);
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->copy));
    if (c->dma_events.size() < 64) {
        while (c->dma_events.size() < 64) { cudaEvent_t e; CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->dma_events.push_back(e); }
    }
    if (c->dma_tail - c->dma_head >= c->dma_events.size()) {             // ring full: retire the oldest
        CUDA_CHECK(cudaEventSynchronize(c->dma_events[c->dma_head % c->dma_events.size()]));
        ++c->dma_head;
    }
    CUDA_CHECK(cudaEventRecord(c->dma_events[c->dma_tail % c->dma_events.size()], c->copy));
    ++c->dma_tail;
}

void dma_wait(Ctx *c, int keep_in_flight) {
    DeviceGuard guard(c);
    while ((long long)(c->dma_tail - c->dma_head) > (long long)keep_in_flight) {
        CUDA_CHECK(cudaEventSynchronize(c->dma_events[c->dma_head % c->dma_events.size()]));
        ++c->dma_head;
    }
}

// ------------------------------------------------------------------------------------------------
// slot-ordered observations (magent_b200_get_observation_slots): record a * S + s is the record env_get_observation
// writes for the row in slot s of arena a, all zeros where the slot is vacant.  Only the pre-pass knows about slots:
// slots_kernel writes the [A][S] slot -> row map into scratch, obs_slot_headers_kernel one header and one feature row
// per slot, and the unchanged obs_render_kernel renders the A * S headers as it renders rows.  A vacant slot's header
// names the blank arena A at (0, 0), self cell 0:
//   * its kind plane is the zeroed window the engine keeps after the last arena's plane in EngineDev::kind: (2 kpad + 1)
//     rows of kw bytes, which hold every view cell of an observer at (0, 0).  No cell is marked, so the hp_norm plane is
//     never read;
//   * its minimap row is row A of mm_pad: zeros, but -1 at cell 0 of every group, so the self marker (+1 at cell 0)
//     leaves +0 there and the undo between two vacant records puts the -1 back.
// A vacant record next to a live one in a CTA's chunk is an arena change, so the render rebuilds the record.  The
// render bounds its record count by the device-side total of the rows (P.off[P.A]); here every one of the A * S headers
// is valid whatever the counts, so P.off points at [A + 1] words of INT_MAX.
__global__ void __launch_bounds__(256) obs_blank_minimap_kernel(float *row, int G, int cells) {
    for (int k = threadIdx.x; k < G * cells; k += blockDim.x) row[k] = k % cells == 0 ? -1.0f : 0.0f;
}

void launch_obs_slots(Ctx *c, const EngineDev *, const EngineDev &hE, const SlotDev *T, const ObsArgs &O,
                      const float *mm_val, int S) {
    DeviceGuard guard(c);
    const size_t n = (size_t)hE.A * S;
    if (n == 0) return;
    if (n > 0x7fffffff) mg::fatal("%zu slot-ordered observation records are more than one launch renders", n);
    grow_obs_hdr(c, n);
    if (n > c->obs_slot_row_n) {
        no_capture(c, "growing the slot table of the observation pre-pass");
        grow_dev(c, c->obs_slot_row, c->obs_slot_row_n, n);
    }
    if ((size_t)hE.A + 1 > c->obs_slot_bound_n) {
        no_capture(c, "growing the observation count bound");
        if (c->obs_slot_bound) { CUDA_CHECK(cudaStreamSynchronize(c->stream)); cudaFree(c->obs_slot_bound); }
        c->obs_slot_bound_n = (size_t)hE.A + 1;
        CUDA_CHECK(cudaMalloc(&c->obs_slot_bound, c->obs_slot_bound_n * sizeof(int)));
        const std::vector<int> bound(c->obs_slot_bound_n, 0x7fffffff);
        CUDA_CHECK(cudaMemcpyAsync(c->obs_slot_bound, bound.data(), bound.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    }
    ObsParams P;
    fill_obs_params(c, hE, O, mm_val, (int)n, P);
    const int g = O.group;
    const GroupDev &D = hE.grp[g];
    const int *off = P.off;
    slots_kernel<<<(unsigned)hE.A, SLOT_THREADS, 0, c->stream>>>(off, D.soa[(O.curmask >> g) & 1u].id, D.cap, T, hE.A, S,
                                                                 nullptr, c->obs_slot_row, 0x7fffffff);
    post_launch("slots_kernel");
    if (mm_val) {
        obs_blank_minimap_kernel<<<1, 256, 0, c->stream>>>(c->mm_pad + (size_t)hE.A * c->mm_stride, hE.G, P.cells);
        post_launch("obs_blank_minimap_kernel");
    }
    size_t hsm;
    const int threads = obs_prepass_threads(P.F, O.half ? 2 : 4, &hsm);
    const int cps = (S + threads - 1) / threads;
    const unsigned grid = (unsigned)((size_t)hE.A * cps);
    if (O.half) obs_slot_headers_kernel<__half><<<grid, threads, hsm, c->stream>>>(P, off, c->obs_slot_row, S, c->obs_hdr, cps);
    else obs_slot_headers_kernel<float><<<grid, threads, hsm, c->stream>>>(P, off, c->obs_slot_row, S, c->obs_hdr, cps);
    post_launch("obs_slot_headers_kernel");
    P.off = c->obs_slot_bound;
    launch_obs_dispatch(c, hE, O, P, (int)n, false, false);
}

// ------------------------------------------------------------------------------------------------
// the slot-ordered step loop (magent_b200_set_action_slots, _get_reward_slots, _get_action_mask_slots), slot_phases.h.
// Actions: one thread per row, CTAs dealt per arena like info_kernel; each row looks its agent's id up in the slot table
// and loads its action from the [A][S] buffer.  Reward and status: one CTA per arena like slots_kernel, which fills the
// arena's [S] blocks, then scatters its rows; no scratch, so the call records into a graph from its first use.
__global__ void __launch_bounds__(256) set_action_slots_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                               const SlotDev *T, int S, const int *act,
                                                               int chunks_per_arena) {
    const EngineDev &E = *gE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = E.grp[g].soa[(curmask >> g) & 1u];
    const int a = blockIdx.x / chunks_per_arena;
    const int i = (blockIdx.x - a * chunks_per_arena) * blockDim.x + threadIdx.x;
    if (i >= off[a + 1] - off[a]) return;
    const long gi = (long)a * E.grp[g].cap + i;
    const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gi], S);
    if (flat >= 0) s.act[gi] = __ldg(act + flat);
}

void launch_set_action_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, unsigned curmask,
                             int group, int S, const int *act) {
    DeviceGuard guard(c);
    const int cap = hE.grp[group].cap;
    const int threads = cap >= 256 ? 256 : ((cap + 31) & ~31);
    const int cpa = (cap + threads - 1) / threads;
    set_action_slots_kernel<<<(unsigned)((size_t)hE.A * cpa), threads, 0, c->stream>>>(dE, curmask, group, T, S, act, cpa);
    post_launch("set_action_slots_kernel");
}

__global__ void __launch_bounds__(SLOT_THREADS) reward_slots_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                                    const SlotDev *T, int S, float *reward,
                                                                    unsigned char *status) {
    const EngineDev &E = *gE;
    const int a = blockIdx.x;
    for (int q = threadIdx.x; q < S; q += SLOT_THREADS) {
        if (reward) reward[(long)a * S + q] = 0.0f;
        if (status) status[(long)a * S + q] = 0;
    }
    __syncthreads();
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = E.grp[g].soa[(curmask >> g) & 1u];
    const int o0 = off[a], cnt = off[a + 1] - o0;
    const float shared_reward = E.hdr[a].grp_reward[g];
    const long base = (long)a * E.grp[g].cap;
    for (int i = threadIdx.x; i < cnt; i += SLOT_THREADS) {
        const int flat = slot_flat(T->tab, T->id_cap, a, s.id[base + i], S);
        if (flat < 0) continue;
        if (reward) reward[flat] = s.next_reward[base + i] + shared_reward;        // info_kernel's INFO_REWARD
        if (status) status[flat] = (s.flags[base + i] & FLAG_DEAD) ? 2 : 1;
    }
}

void launch_reward_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, unsigned curmask, int group,
                         int S, float *reward, unsigned char *status) {
    DeviceGuard guard(c);
    reward_slots_kernel<<<(unsigned)hE.A, SLOT_THREADS, 0, c->stream>>>(dE, curmask, group, T, S, reward, status);
    post_launch("reward_slots_kernel");
}

// the [A][S] slot -> row map of `group` in c->obs_slot_row (grown outside a capture only)
static void slot_rows_scratch(Ctx *c, const EngineDev &hE, const SlotDev *T, unsigned curmask, int group, int S,
                              const char *what) {
    const size_t n = (size_t)hE.A * S;
    if (n > c->obs_slot_row_n) {
        no_capture(c, what);
        grow_dev(c, c->obs_slot_row, c->obs_slot_row_n, n);
    }
    const GroupDev &D = hE.grp[group];
    slots_kernel<<<(unsigned)hE.A, SLOT_THREADS, 0, c->stream>>>(hE.off + (size_t)group * (hE.A + 1),
                                                                 D.soa[(curmask >> group) & 1u].id, D.cap, T, hE.A, S,
                                                                 nullptr, c->obs_slot_row, 0x7fffffff);
    post_launch("slots_kernel");
}

// Mask: slots_kernel writes the [A][S] slot -> row map into the scratch of the slot-ordered observation, then
// action_mask_slots_kernel takes MASK_THREADS consecutive slots of one arena per CTA, so an arena gets several CTAs
// whatever its population (a one-arena batch is not one CTA).  It is action_mask_kernel with the lanes' agents looked up
// through the map: a vacant slot's lane holds a dead agent, which action_legal refuses every action, so its row is zero.
// The CTA's rows are one contiguous byte range of the output, stored as action_mask_kernel stores its rows.
__global__ void __launch_bounds__(MASK_THREADS) action_mask_slots_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                                        const int *slot_row, int S, unsigned char *out,
                                                                        int chunks_per_arena) {
    __shared__ EngineDev sE;
    extern __shared__ __align__(16) unsigned char mask_smem[];
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * MASK_THREADS;
    const int cta_cnt = min(MASK_THREADS, S - c0);
    const int cnt = min(32, cta_cnt - 32 * warp);
    MaskAgent mine;
    mine.x = mine.y = 0; mine.dir = DIR_NORTH; mine.code = 0; mine.flags = FLAG_DEAD;
    if (lane < cnt) {
        const int r = slot_row[(long)a * S + c0 + 32 * warp + lane];
        if (r >= 0) mine = mask_agent(E, curmask, a, g, r - E.off[(size_t)g * (E.A + 1) + a]);
    }
    const int na = E.grp[g].n_action;
    unsigned char *dst = out + ((size_t)a * S + c0) * na;
    unsigned char *rows = mask_smem + ((size_t)dst & 15);
    const int *occ = E.occ + (long)a * E.W * E.H;
    for (int j = 0; j < cnt; ++j) {
        MaskAgent m;
        m.x = __shfl_sync(0xffffffffu, mine.x, j); m.y = __shfl_sync(0xffffffffu, mine.y, j);
        m.dir = __shfl_sync(0xffffffffu, mine.dir, j); m.code = __shfl_sync(0xffffffffu, mine.code, j);
        m.flags = (unsigned char)__shfl_sync(0xffffffffu, (int)mine.flags, j);
        unsigned char *row = rows + (size_t)(32 * warp + j) * na;
        for (int k = lane; k < na; k += 32) row[k] = action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
    }
    __syncthreads();
    mask_rows_store(dst, rows, cta_cnt * na);
}

void launch_action_mask_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, unsigned curmask,
                              int group, int S, unsigned char *mask) {
    DeviceGuard guard(c);
    const size_t n = (size_t)hE.A * S;
    if (n == 0) return;
    const size_t smem = mask_dyn_smem(hE, group);
    smem_prepare(c, ATTR_MASK_SLOTS, action_mask_slots_kernel, smem, "action_mask_slots_kernel");
    slot_rows_scratch(c, hE, T, curmask, group, S, "growing the slot table of the slot-ordered action mask");
    const int cps = (S + MASK_THREADS - 1) / MASK_THREADS;
    action_mask_slots_kernel<<<(unsigned)((size_t)hE.A * cps), MASK_THREADS, smem, c->stream>>>(dE, curmask, group,
                                                                                               c->obs_slot_row, S, mask, cps);
    post_launch("action_mask_slots_kernel");
}

// Mean action and neighbours in slot order (magent_b200_get_mean_action_slots, _get_neighbours_slots): slots_kernel
// writes the group's [A][S] slot -> row map into the same scratch as for the mask, then the kernels run the CTAs of
// mean_action_kernel and neighbours_kernel under the slot policy (nbr_cta_load): a CTA takes MEAN_OBS / NBR_OBS
// consecutive slots of one arena, so a one-arena batch still gets many CTAs, and writes its rows at a * S + slot, one
// contiguous range.  A vacant slot's lane holds the dead placeholder, so the dead-observer path writes its zero / -1 row.
__global__ void __launch_bounds__(MEAN_THREADS, 5) mean_action_slots_kernel(const EngineDev *gE, unsigned curmask, int g,
                                                                        int of, const int *slot_row, int S, float *mean,
                                                                        int *count, int chunks_per_arena) {
    __shared__ EngineDev sE;
    __shared__ int n_in_s;
    extern __shared__ __align__(16) unsigned char mean_smem[];
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * MEAN_OBS;
    const int o0 = E.off[(size_t)g * (E.A + 1) + a];
    mean_action_cta<true>(E, curmask, g, of, mean, count, a, c0, min(MEAN_OBS, S - c0), o0, slot_row + (size_t)a * S,
                          a * S, mean_smem, n_in_s);
}

__global__ void __launch_bounds__(NBR_THREADS, 5) neighbours_slots_kernel(const EngineDev *gE, const NbrCell *lut,
                                                                          unsigned curmask, int g, int of, int k,
                                                                          const int *slot_row, int S, const SlotDev *T,
                                                                          int S_of, int *idx, int *rel, int *count,
                                                                          int chunks_per_arena) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * NBR_OBS;
    const int o0 = E.off[(size_t)g * (E.A + 1) + a];
    neighbours_cta<true>(E, lut, curmask, g, of, k, idx, rel, count, a, c0, min(NBR_OBS, S - c0), o0,
                         slot_row + (size_t)a * S, a * S, T, S_of);
}

void launch_mean_action_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, unsigned curmask,
                              int group, int of, int S, float *mean, int *count) {
    DeviceGuard guard(c);
    const size_t n = (size_t)hE.A * S;
    if (n == 0) return;
    if (n > 0x7fffffff) mg::fatal("%zu slots are more than one launch covers (rows a * S + slot are ints)", n);
    const size_t smem = mean_dyn_smem(hE, group, of);
    smem_prepare(c, ATTR_MEAN_SLOTS, mean_action_slots_kernel, smem, "mean_action_slots_kernel");
    slot_rows_scratch(c, hE, T, curmask, group, S, "growing the slot table of the slot-ordered mean action");
    const int cps = (S + MEAN_OBS - 1) / MEAN_OBS;
    mean_action_slots_kernel<<<(unsigned)((size_t)hE.A * cps), MEAN_THREADS, smem, c->stream>>>(
        dE, curmask, group, of, c->obs_slot_row, S, mean, count, cps);
    post_launch("mean_action_slots_kernel");
}

void launch_neighbours_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, const NbrCell *lut,
                             unsigned curmask, int group, int of, int k, int S, int S_of, int *idx, int *rel,
                             int *count) {
    DeviceGuard guard(c);
    const size_t n = (size_t)hE.A * S;
    if (n == 0) return;
    if (n > 0x7fffffff) mg::fatal("%zu slots are more than one launch covers (rows a * S + slot are ints)", n);
    slot_rows_scratch(c, hE, T, curmask, group, S, "growing the slot table of the slot-ordered neighbours");
    const int cps = (S + NBR_OBS - 1) / NBR_OBS;
    neighbours_slots_kernel<<<(unsigned)((size_t)hE.A * cps), NBR_THREADS, 0, c->stream>>>(
        dE, lut, curmask, group, of, k, c->obs_slot_row, S, T, S_of, idx, rel, count, cps);
    post_launch("neighbours_slots_kernel");
}

// ------------------------------------------------------------------------------------------------
// built-in scripted opponents (magent_b200_rule_actions, _get_rule_actions, _get_rule_actions_slots): rule_phases.h
// for every agent of a group.  CTAs are dealt per arena like random_legal_actions_kernel (blockIdx says which arena, the
// device-side offsets decide how many agents it has, the host's count is only an upper bound); a thread holds one agent.
// Attacks, moves and the fallback draw are decided per lane (rule_attack, rule_move, rule_fallback: a handful of `occ`
// cells each).  The view walk of step 2 (rule_nearest) is made by the whole warp, one agent at a time for the lanes
// that need it: the lanes take 32 consecutive cells of the view LUT (key order, L1-resident), and the lowest lane whose
// cell lists a target in the first round that has one gives the cell, as neighbours_kernel finds its first neighbour.
// A walk of one lane at a time measured about 1.24 ms per call on battle512 against 0.19 ms for the neighbours at k = 1
// (DESIGN.md §5).  The slot kernel takes RULE_THREADS consecutive slots of one arena per CTA and looks each slot's row up
// in slots_kernel's [A][S] map, as action_mask_slots_kernel does; a vacant slot gets -1.
constexpr int RULE_THREADS = 256;
// __launch_bounds__(RULE_THREADS, 4) leaves them 64 registers: 61-63 without spills (a bare bound allows 48, and spills).

// The action of this lane's agent m (ABI ordinal o; `live` false: no agent, the result is not used).  Every lane of the
// warp calls it.
__device__ __forceinline__ int rule_warp(const EngineDev &E, const NbrCell *lut, unsigned curmask, int a, int g, int t,
                                         int policy, const MaskAgent &m, bool live, unsigned long long seed, int o) {
    const int lane = threadIdx.x & 31;
    const int *occ = E.occ + (long)a * E.W * E.H;
    int act = -1;                                             // -1: not decided yet
    if (!live || (m.flags & FLAG_DEAD)) act = 0;
    else if (policy == RULE_RUSH) act = rule_attack(E, curmask, a, occ, g, t, m);
    const int n = E.grp[g].view_count;
    bool seen = false;
    int cx = 0, cy = 0;
    for (unsigned need = __ballot_sync(0xffffffffu, act < 0); need; need &= need - 1) {
        const int u = __ffs(need) - 1;
        NbrObserver w;
        w.x = __shfl_sync(0xffffffffu, m.x, u); w.y = __shfl_sync(0xffffffffu, m.y, u);
        w.dir = __shfl_sync(0xffffffffu, m.dir, u); w.code = __shfl_sync(0xffffffffu, m.code, u);
        w.flags = (unsigned char)__shfl_sync(0xffffffffu, (int)m.flags, u);
        const NbrCell *l = lut + (E.turn_mode ? w.dir * n : 0);
        const unsigned char *kp = E.kind + (long)a * E.kplane + (long)(w.y + E.kpad) * E.kw + w.x + E.kpad;
        for (int q0 = 0; q0 < n; q0 += 32) {                  // warp-uniform bounds: every lane takes every ballot
            const int q = q0 + lane;
            int x = 0, y = 0;
            bool hit = false;
            if (q < n && nbr_kind_of(__ldg(kp + __ldg(&l[q].off)), t)) {
                const int d = __ldg(&l[q].delta);
                x = w.x + (short)(d & 0xffff); y = w.y + (d >> 16);
                hit = nbr_nearest_at(E, curmask, a, g, t, w, x, y, __ldg(&l[q].key)) >= 0;
            }
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (hits) {
                const int f = __ffs(hits) - 1;
                x = __shfl_sync(0xffffffffu, x, f); y = __shfl_sync(0xffffffffu, y, f);
                if (lane == u) { seen = true; cx = x; cy = y; }
                break;
            }
        }
    }
    if (act < 0 && seen) act = rule_move(E, curmask, a, occ, g, m, cx, cy, policy == RULE_FLEE);
    if (act < 0) act = rule_fallback(E, curmask, a, occ, g, m, seed, E.counters[CNT_STEPS], o);
    return act;
}

__global__ void __launch_bounds__(RULE_THREADS, 4) rule_actions_kernel(const EngineDev *gE, const NbrCell *lut,
                                                                      unsigned curmask, int g, int t, int policy,
                                                                      unsigned long long seed, int *out, int n_total,
                                                                      int chunks_per_arena) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const int a = blockIdx.x / chunks_per_arena;
    const int c0 = (blockIdx.x - a * chunks_per_arena) * RULE_THREADS;
    const int o0 = off[a];
    if (c0 >= off[a + 1] - o0 || o0 + c0 >= n_total) return;     // the whole CTA: the warps below stay converged
    const int i = c0 + threadIdx.x, o = o0 + i;
    const bool live = i < off[a + 1] - o0 && o < n_total;
    MaskAgent m;
    m.x = m.y = 0; m.dir = DIR_NORTH; m.code = 0; m.flags = FLAG_DEAD;
    if (live) m = mask_agent(E, curmask, a, g, i);
    const int act = rule_warp(E, lut, curmask, a, g, t, policy, m, live, seed, o);
    if (!live) return;
    if (out) out[o] = act;
    else cur_soa(E, curmask, g).act[gidx(E, a, g, i)] = act;
}

__global__ void __launch_bounds__(RULE_THREADS, 4) rule_actions_slots_kernel(const EngineDev *gE, const NbrCell *lut,
                                                                            unsigned curmask, int g, int t, int policy,
                                                                            unsigned long long seed, const int *slot_row,
                                                                            int S, int *out, int chunks_per_arena) {
    __shared__ EngineDev sE;
    load_engine(&sE, gE);
    const EngineDev &E = sE;
    const int a = blockIdx.x / chunks_per_arena;
    const int s = (blockIdx.x - a * chunks_per_arena) * RULE_THREADS + threadIdx.x;
    const int r = s < S ? slot_row[(long)a * S + s] : -1;
    const int o0 = E.off[(size_t)g * (E.A + 1) + a];
    MaskAgent m;
    m.x = m.y = 0; m.dir = DIR_NORTH; m.code = 0; m.flags = FLAG_DEAD;
    if (r >= 0) m = mask_agent(E, curmask, a, g, r - o0);
    const int act = rule_warp(E, lut, curmask, a, g, t, policy, m, r >= 0, seed, r);
    if (s < S) out[(long)a * S + s] = r >= 0 ? act : -1;
}

void launch_rule_actions(Ctx *c, const EngineDev *dE, const EngineDev &hE, const NbrCell *lut, unsigned curmask,
                         int group, int target, int policy, unsigned long long seed, int *out, int n_total) {
    DeviceGuard guard(c);
    const int cpa = (hE.grp[group].cap + RULE_THREADS - 1) / RULE_THREADS;
    rule_actions_kernel<<<(unsigned)((size_t)hE.A * cpa), RULE_THREADS, 0, c->stream>>>(dE, lut, curmask, group, target,
                                                                                      policy, seed, out, n_total, cpa);
    post_launch("rule_actions_kernel");
}

void launch_rule_actions_slots(Ctx *c, const EngineDev *dE, const EngineDev &hE, const SlotDev *T, const NbrCell *lut,
                               unsigned curmask, int group, int target, int policy, unsigned long long seed, int S,
                               int *out) {
    DeviceGuard guard(c);
    const size_t n = (size_t)hE.A * S;
    if (n == 0) return;
    if (n > 0x7fffffff) mg::fatal("%zu slots are more than one launch covers (rows a * S + slot are ints)", n);
    slot_rows_scratch(c, hE, T, curmask, group, S, "growing the slot table of the slot-ordered rule actions");
    const int cps = (S + RULE_THREADS - 1) / RULE_THREADS;
    rule_actions_slots_kernel<<<(unsigned)((size_t)hE.A * cps), RULE_THREADS, 0, c->stream>>>(
        dE, lut, curmask, group, target, policy, seed, c->obs_slot_row, S, out, cps);
    post_launch("rule_actions_slots_kernel");
}

// ------------------------------------------------------------------------------------------------
// replay recorder (replay_phases.h).  Every kernel covers agents, not arenas: a thread per flat row (GroupDev::foff + i)
// of a recorded arena, blockIdx.y the arena, so one arena of 800k agents spreads over the whole GPU like 64 small ones.
constexpr int REP_THREADS = 256;
constexpr unsigned REP_MAX_Y = 65535;

__global__ void __launch_bounds__(REP_THREADS) replay_events_kernel(const EngineDev *gE, unsigned curmask, RepArena *rep,
                                                                    RepEvent *ev, const int *arenas, int n_arenas) {
    const EngineDev &E = *gE;
    const int f = blockIdx.x * REP_THREADS + threadIdx.x;
    if (f >= E.cap_total) return;
    const int g = replay_group_of(E, f);
    if (g < 0) return;
    const GroupDev &G = E.grp[g];
    const int i = f - G.foff;
    const AgentSoA &s = G.soa[(curmask >> g) & 1u];
    for (int k = blockIdx.y; k < n_arenas; k += gridDim.y) {
        const int a = __ldg(arenas + k);
        if (a < 0) continue;
        const int n = E.n[(long)g * E.A + a];
        if (i == 0) rep[a].ev_n[g] = n;
        if (i >= n) continue;
        const long gi = (long)a * G.cap + i;
        ev[(long)a * E.cap_total + f] = replay_event(G, s, E.turn_mode, gi, G.ev_rank[gi]);
    }
}

void launch_replay_events(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, RepArena *rep,
                          RepEvent *ev, const int *arenas, int n_arenas) {
    if (n_arenas <= 0 || hE.cap_total <= 0) return;
    DeviceGuard guard(c);
    const dim3 grid((unsigned)((hE.cap_total + REP_THREADS - 1) / REP_THREADS), std::min((unsigned)n_arenas, REP_MAX_Y));
    replay_events_kernel<<<grid, REP_THREADS, 0, c->stream>>>(dE, curmask, rep, ev, arenas, n_arenas);
    post_launch("replay_events_kernel");
}

__global__ void __launch_bounds__(REP_THREADS) replay_restore_kernel(RepArena *rep, const int *src, const int *done, int A) {
    const int a = blockIdx.x * REP_THREADS + threadIdx.x;
    if (a >= A || restore_source(src, done, A, a) < 0) return;
    rep[a].episode += 1;
    for (int g = 0; g < MG_MAX_GROUPS; ++g) rep[a].ev_n[g] = 0;
}

void launch_replay_restore(Ctx *c, const EngineDev &hE, RepArena *rep, const int *src) {
    DeviceGuard guard(c);
    replay_restore_kernel<<<(unsigned)((hE.A + REP_THREADS - 1) / REP_THREADS), REP_THREADS, 0, c->stream>>>(rep, src, hE.done, hE.A);
    post_launch("replay_restore_kernel");
}

// items of a recorded arena: cap_total agent rows, cap_total event rows, wall_words bitmap words.  Every CTA reads the
// frame counter and the last episodes first; the last CTA to finish (ticket) advances them, so no CTA of this launch
// sees them change.
__global__ void __launch_bounds__(REP_THREADS) replay_record_kernel(const EngineDev *gE, unsigned curmask,
                                                                    const RepArena *rep, const RepEvent *ev,
                                                                    const RepRecord R) {
    const EngineDev &E = *gE;
    const int frame = *(volatile const int *)&R.ctl->n_frames;
    if (frame < R.max_frames) {
        const int item = blockIdx.x * REP_THREADS + threadIdx.x;
        const int ct = R.L.cap_total;
        const long cells = (long)E.W * E.H;
        const long agent_base = R.L.agent_base(), event_base = R.L.event_base(), wall_base = R.L.wall_base();
        const long frame_ints = R.L.frame_ints();
        for (int k = blockIdx.y; k < R.n_arenas; k += gridDim.y) {
            const int a = __ldg(R.arenas + k);
            const int episode = rep[a].episode;
            const bool walls = episode != R.last_ep[k];
            int *F = R.frames + ((long)frame * R.n_arenas + k) * frame_ints;
            if (item == 0) {
                F[REP_H_EPISODE] = episode;
                F[REP_H_WALLS] = walls ? 1 : 0;
                for (int g = 0; g < MG_MAX_GROUPS; ++g) {
                    F[REP_H_N + g] = g < E.G ? E.n[(long)g * E.A + a] : 0;
                    F[REP_H_EV_N + g] = g < E.G ? rep[a].ev_n[g] : 0;
                }
            }
            if (item < 2 * ct) {
                const int f = item < ct ? item : item - ct;
                const int g = replay_group_of(E, f);
                if (g < 0) continue;
                const GroupDev &G = E.grp[g];
                const int i = f - G.foff;
                if (item < ct) {
                    if (i >= E.n[(long)g * E.A + a]) continue;
                    const RepAgent r = replay_agent(G.soa[(curmask >> g) & 1u], E.turn_mode, (long)a * G.cap + i);
                    int *o = F + agent_base + (long)f * (sizeof(RepAgent) / 4);
                    o[0] = r.id; o[1] = r.x; o[2] = r.y; o[3] = __float_as_int(r.hp); o[4] = r.dir_flags;
                } else {
                    if (i >= rep[a].ev_n[g]) continue;
                    const int4 e = *reinterpret_cast<const int4 *>(ev + (long)a * ct + f);
                    reinterpret_cast<int4 *>(F + event_base)[f] = e;
                }
            } else if (walls && item - 2 * ct < R.L.wall_words) {
                const int w = item - 2 * ct;
                F[wall_base + w] = (int)replay_wall_word(E.occ + (long)a * cells, cells, w);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned last = gridDim.x * gridDim.y - 1;
        if (atomicAdd(&R.ctl->ticket, 1u) == last) {
            if (frame < R.max_frames) {
                for (int k = 0; k < R.n_arenas; ++k) R.last_ep[k] = rep[__ldg(R.arenas + k)].episode;
                R.ctl->n_frames = frame + 1;
            } else {
                R.ctl->dropped += 1;
            }
            R.ctl->ticket = 0;
            __threadfence();
        }
    }
}

void launch_replay_record(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, const RepArena *rep,
                          const RepEvent *ev, const RepRecord &R) {
    DeviceGuard guard(c);
    const long items = 2L * R.L.cap_total + R.L.wall_words;
    const dim3 grid((unsigned)std::max(1L, (items + REP_THREADS - 1) / REP_THREADS), std::min((unsigned)R.n_arenas, REP_MAX_Y));
    replay_record_kernel<<<grid, REP_THREADS, 0, c->stream>>>(dE, curmask, rep, ev, R);
    post_launch("replay_record_kernel");
}

bool smem_fits(Ctx *c, const EngineDev &hE, int which, int group, int of, std::string *why) {
    DeviceGuard guard(c);
    size_t dyn = 0, need = 0;
    int band = 0;
    switch (which) {
    case SMEM_ACTION_MASK:
        band = smem_band(c, ATTR_MASK, action_mask_kernel, dyn = mask_dyn_smem(hE, group), &need); break;
    case SMEM_ACTION_MASK_SLOTS:
        band = smem_band(c, ATTR_MASK_SLOTS, action_mask_slots_kernel, dyn = mask_dyn_smem(hE, group), &need); break;
    case SMEM_MEAN_ACTION:
        band = smem_band(c, ATTR_MEAN, mean_action_kernel, dyn = mean_dyn_smem(hE, group, of), &need); break;
    case SMEM_MEAN_ACTION_SLOTS:
        band = smem_band(c, ATTR_MEAN_SLOTS, mean_action_slots_kernel, dyn = mean_dyn_smem(hE, group, of), &need); break;
    case SMEM_OBS_WIRE:                                      // no opt-in: the default limit is the wire kernel's
        band = smem_band(c, ATTR_WIRE, obs_wire_kernel, dyn = wire_dyn_smem(hE, group), &need);
        if (band > 0) band = -1;
        break;
    default: mg::fatal("smem_fits: no kernel %d", which);
    }
    if (band >= 0) return true;
    if (why) {
        char buf[256];
        snprintf(buf, sizeof buf, "%zu bytes of shared memory per block (%zu of them the kernel's own), more than the %zu "
                 "the device allows", need, need - dyn, which == SMEM_OBS_WIRE ? c->smem_block : c->smem_optin);
        *why = buf;
    }
    return false;
}

}  // namespace be
}  // namespace mg
