// backend.h -- the thin seam between the host engine (engine.cc, plain C++) and the device.
//
// The product library links backend_cuda.cu (CUDA runtime + the sm_90a kernels).  tests/emu/ links
// backend_emu.cc instead, which runs the same phase functions single-threaded on the host so the
// parallel formulations can be debugged without a GPU.  There is exactly one backend per library;
// nothing selects between them at run time.
//
// Every engine owns one be::Ctx: the CUDA device it lives on, its private streams, events and device-side scratch
// buffers.  Nothing device-related is process-global, so engines on different devices (or driven from different
// threads) do not interfere -- like the reference, which keeps one heap object per handle (src/runtime_api.cc:15-32).
#pragma once
#include <stddef.h>
#include <string>
#include "dev_types.h"

namespace mg {
namespace be {

struct Ctx;                              // per-engine device context (opaque to the engine)

const char *name();
int device_count();
// Create a context on `device` (or the current one when < 0).  Returns nullptr and fills *err when no usable device.
Ctx *create(int device, std::string *err);
void destroy(Ctx *);
int device_of(const Ctx *);
int sm_count(const Ctx *);
void *stream_handle(const Ctx *);        // the cudaStream_t every kernel of this engine is launched on

void *dmalloc(Ctx *, size_t bytes);
void dfree(Ctx *, void *p);
void dmemset(Ctx *, void *p, int byte, size_t bytes);
void h2d(Ctx *, void *dst, const void *src, size_t bytes);          // blocking
void d2h(Ctx *, void *dst, const void *src, size_t bytes);          // blocking
void d2d(Ctx *, void *dst, const void *src, size_t bytes);
void *host_alloc(size_t bytes);          // page-locked
void host_free(void *p);
bool host_register(void *p, size_t bytes);   // page-lock existing host memory (DMA target); false when not possible
void host_unregister(void *p);
bool is_device_ptr(const void *p);
bool is_pinned_host_ptr(const void *p);  // page-locked host memory known to the CUDA driver (DMA target)
void sync(Ctx *);

// dE: device copy of the EngineDev block; hE: the host copy it was uploaded from (for sizes)
void launch_step(Ctx *, const EngineDev *dE, const EngineDev &hE, const StepArgs &S, int max_agents_per_arena);
void launch_cull(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int max_agents_per_arena);
void launch_offsets(Ctx *, const EngineDev *dE, const EngineDev &hE);
// per-call preparation of get_observation: normalised minimap into mm_val ([A][G][view cells]; nullptr when
// minimap_mode is off) plus whatever the backend wants to precompute for the render kernel
void launch_obs_prepare(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int obs_group, float *mm_val);
void launch_obs(Ctx *, const EngineDev *dE, const EngineDev &hE, const ObsArgs &O, const float *mm_val, int n_total);
// the last obs_render_kernel launch of this context: {sizeof(T), NIT, turn, TA (agents per tile), grid, chunk, tiles,
// view and feature buffers both 16-byte aligned}; all zero before the first launch.  Declared weak like
// launch_global_state: a backend without it loads, and the engine refuses the "obs_launch" info key.
__attribute__((weak)) void obs_launch_report(const Ctx *, int out[8]);
// the last step and cull launches of this context, five ints each (step first, then cull): {mode (0 CTA per arena,
// 1 whole-grid team), grid, threads, dynamic shared-memory bytes, step scratch in shared memory (0 for the cull)}; all
// zero before the first launch.  Weak like obs_launch_report: the engine refuses the "step_launch" info key without it.
__attribute__((weak)) void step_launch_report(const Ctx *, int out[10]);
// whole-map state of every arena into `out` ([A][H][W][state_channels], obs_phases.h state_compose_cell): float32, or
// IEEE half (the float32 value rounded to nearest-even) when `half`.  A device buffer, 16-byte aligned.
// Declared weak: the CUDA backend always defines it, a test backend may leave it out (the engine then refuses
// magent_b200_get_global_state instead of failing to load).
__attribute__((weak)) void launch_global_state(Ctx *, const EngineDev *dE, const EngineDev &hE, void *out, int half);
// Restore arenas from a snapshot (Engine::restore_arenas): live arena a becomes snapshot arena s = src[a] (src: device
// int32[A]), or s = a where bit 0 of EngineDev::done[a] is set when src is nullptr; s outside [0, A) leaves the arena
// untouched.  Copies occ, kind, hp_norm, food, the first S.n[g][s] records of every SoA field of the live buffer
// (curmask), n, dead_ct, done and the header (but the RNG when keep_rng), fills claim_head with -1, then recomputes the
// offset table (launch_offsets).  Needs no host synchronisation.
// launch_arena_done: bit 0 of EngineDev::done into out[A] (a device buffer).
// Declared weak like launch_global_state: a backend without them loads, and the engine refuses the calls.
__attribute__((weak)) void launch_restore(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask,
                                          const SnapDev &S, const int *src, int keep_rng);
__attribute__((weak)) void launch_arena_done(Ctx *, const EngineDev *dE, const EngineDev &hE, int *out);
void launch_info(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int kind, int group,
                 void *buf, int n_total);
void launch_random_actions(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group,
                           unsigned long long seed, int n_total);
// Legal actions of every agent of `group` (mask_phases.h action_legal).  launch_action_mask: uint8 [n][n_action] into
// `out`, a device buffer; launch_random_legal_actions: AgentSoA::act of every agent drawn uniformly from its legal actions
// (mask_phases.h legal_draw; 0 when it has none).  n_total is the host's count, an upper bound: the device-side offsets
// decide.  Declared weak like launch_global_state: a backend without them loads, and the engine refuses the calls.
__attribute__((weak)) void launch_action_mask(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group,
                                              unsigned char *out, int n_total);
__attribute__((weak)) void launch_random_legal_actions(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask,
                                                       int group, unsigned long long seed, int n_total);
// Mean neighbour action of every agent of `group` over its neighbours of group `of` (nbr_phases.h): float
// [n][n_action(of)] into `mean` and, unless null, int [n] into `count`, both device buffers.  n_total is the host's count,
// an upper bound: the device-side offsets decide.  Weak like launch_action_mask: the engine refuses the call without it.
__attribute__((weak)) void launch_mean_action(Ctx *, const EngineDev *dE, const EngineDev &hE, unsigned curmask, int group,
                                              int of, float *mean, int *count, int n_total);
// The first k (1..32) neighbours of group `of`, nearest first (nbr_phases.h nbr_cell_key), of every agent of `group`: int
// [n][k] rows of `of` into `idx`, unless null int [n][k][2] (vy, vx) into `rel` and int [n] |N(i)| into `count`, all
// device buffers; unused slots -1.  `lut` is the group's view LUT in key order (struct NbrCell, one run of view_count
// entries per heading in turn_mode), a device buffer.  n_total is the host's count, an upper bound: the device-side
// offsets decide.  Weak like launch_mean_action: the engine refuses the call without it.
__attribute__((weak)) void launch_neighbours(Ctx *, const EngineDev *dE, const EngineDev &hE, const NbrCell *lut,
                                             unsigned curmask, int group, int of, int k, int *idx, int *rel, int *count,
                                             int n_total);
// Stable slots of `group` (slot_phases.h): row_slot[r] = a * S + slot for every row r below the device-side total, -1
// from there up to n_bound, and slot_row[a][slot] = the row of the agent in that slot, -1 where none is; either may be
// null, both are device buffers.  `T` is the engine's SlotDev block, a device pointer.  n_bound is the host's bound of
// the rows (num_bound): the device-side offsets decide.  launch_restore_slots copies, for every arena launch_restore
// (same src and done rules) is about to restore, the first SLOT_HDR + snap_id_cap words of the snapshot table's row s
// into the live row; it runs before launch_restore, which changes the done words.  Weak like launch_neighbours: the
// engine refuses get_slots without them.
__attribute__((weak)) void launch_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                        unsigned curmask, int group, int S, int *row_slot, int *slot_row, int n_bound);
__attribute__((weak)) void launch_restore_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                const int *snap_tab, int snap_id_cap, const int *src);
// Observation O of group O.group in slot order (magent_b200_get_observation_slots): O.view [A][S] records and O.feature
// [A][S] rows, both device buffers; record a * S + s is the one launch_obs writes for the row in slot s of arena a
// (slot_phases.h, the device-side offsets decide the rows), all zeros where no row is.  mm_val as for launch_obs (the
// engine ran launch_obs_prepare for this group).  The kind plane must be followed by the blank window of
// EngineDev::kind.  Weak like launch_slots: the engine refuses the call without it.
__attribute__((weak)) void launch_obs_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                            const ObsArgs &O, const float *mm_val, int S);
// The slot-ordered step loop of `group` (slot_phases.h, the device-side offsets decide the rows; all buffers are device
// buffers of [A][S] entries).  launch_set_action_slots: every row's AgentSoA::act = act[its slot], nothing else is read.
// launch_reward_slots: reward[slot] = the row's env_get_reward value and status[slot] = 1 alive, 2 dead (not culled yet),
// +0.0 and 0 where no row is; either may be null.  launch_action_mask_slots: mask [A][S][n_action], the row
// launch_action_mask writes for the row in each slot (mask_phases.h action_legal), all zero where no row is.  Weak like
// launch_slots: the engine refuses the calls without them.
__attribute__((weak)) void launch_set_action_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                   unsigned curmask, int group, int S, const int *act);
__attribute__((weak)) void launch_reward_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                               unsigned curmask, int group, int S, float *reward, unsigned char *status);
__attribute__((weak)) void launch_action_mask_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                    unsigned curmask, int group, int S, unsigned char *mask);
// The mean action and the neighbours of `group` in slot order (slot_phases.h, the device-side offsets decide the rows; all
// buffers are device buffers).  launch_mean_action_slots: mean [A][S][n_action(of)] and, unless null, count [A][S], the
// rows launch_mean_action writes for the row in each slot, +0.0 and 0 where no row is.  launch_neighbours_slots: idx
// [A][S][k] and, unless null, rel [A][S][k][2] and count [A][S], the rows launch_neighbours writes for the row in each
// slot with every stored idx entry the neighbour's a * S_of + slot in group `of` (S_of = of's slot space) instead of its
// row; all -1 and count 0 where no row is.  `lut` as for launch_neighbours.  Weak like launch_slots: the engine refuses
// the calls without them.
__attribute__((weak)) void launch_mean_action_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                    unsigned curmask, int group, int of, int S, float *mean, int *count);
__attribute__((weak)) void launch_neighbours_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                   const NbrCell *lut, unsigned curmask, int group, int of, int k, int S,
                                                   int S_of, int *idx, int *rel, int *count);
// The built-in scripted opponent (rule_phases.h rule_action) for every agent of `group` against group `target` under
// `policy` (RULE_RUSH, RULE_FLEE); `seed` and the device step counter as legal_draw takes them, `lut` as for
// launch_neighbours.  launch_rule_actions: int [n] in row order into `out`, or AgentSoA::act of every agent when `out` is
// null; n_total is the host's count, an upper bound: the device-side offsets decide.  launch_rule_actions_slots: int
// [A][S] into `out`, the action of the row in each slot (slot_phases.h, the device-side offsets decide the rows), -1
// where no row is.  All buffers are device buffers.  Weak like launch_neighbours: the engine refuses the calls without
// them.
__attribute__((weak)) void launch_rule_actions(Ctx *, const EngineDev *dE, const EngineDev &hE, const NbrCell *lut,
                                               unsigned curmask, int group, int target, int policy,
                                               unsigned long long seed, int *out, int n_total);
__attribute__((weak)) void launch_rule_actions_slots(Ctx *, const EngineDev *dE, const EngineDev &hE, const SlotDev *T,
                                                     const NbrCell *lut, unsigned curmask, int group, int target,
                                                     int policy, unsigned long long seed, int S, int *out);
// Whether kernel `which` fits the device's shared memory for `group` (and, for the mean action, the histograms of group
// `of`'s actions): its static shared memory plus what the view or the action space asks for, against the device's
// opt-in limit per block (the default limit for the wire kernel, which does not opt in).  When it does not, *why (unless
// null) says how many bytes it would need and what the device allows.  The engine asks before anything is staged or
// written: it refuses the mask and mean-action calls with -1, and takes the dense path instead of the wire records.
// Weak like launch_slots: without it nothing is refused (the test emulation has no shared-memory limit).
enum { SMEM_ACTION_MASK, SMEM_ACTION_MASK_SLOTS, SMEM_MEAN_ACTION, SMEM_MEAN_ACTION_SLOTS, SMEM_OBS_WIRE };
__attribute__((weak)) bool smem_fits(Ctx *, const EngineDev &hE, int which, int group, int of, std::string *why);
// clear_dead: asynchronous read-back of the [G][A+1] offset table (launch_offsets) into page-locked memory
void counts_fetch_begin(Ctx *, const int *dev_off, size_t n_ints);
const int *counts_fetch_wait(Ctx *);     // blocks until the fetch has landed; valid until the next counts_fetch_begin
// env_step's result: *all_done = AND over arenas of the done bit, *any_dead = OR of bit 1 (EngineDev::done), and the
// per-arena words into done_words[A] when not null.  One small pinned read-back on the engine's stream.
void read_done(Ctx *, const EngineDev &hE, int *done_words);
// the same reduction written to a DEVICE int (env_step called with a device pointer): no host synchronisation
void launch_done_to_device(Ctx *, const EngineDev *dE, const EngineDev &hE, int *dev_done);

// ---- host-buffer observations (DESIGN.md §6b): compact wire records over PCIe, expanded by host threads
// One wire record per observer in ABI order: header + the observer's marks (non-zero view values other than the
// minimap channels).  Marks of WIRE_CHUNK consecutive observers are contiguous in `marks`, chunk c starting at
// chunk_base[c]; inside a chunk the marks of consecutive observers follow each other (count in the header).
enum { WIRE_CHUNK = 1024 };
enum : unsigned { WIRE_HAS_HP = 0x80000000u };
struct WireHdr {
    int arena;                           // whose minimap rows the record carries
    unsigned short self_cell;            // coarse minimap cell of the observer (0xffff: none)
    unsigned short count;                // marks of this observer
};
struct WireMark {
    unsigned off;                        // word offset inside the record: rec[off] = 1; bit 31: rec[off + 1] = val as well
    float val;                           // hp / max_hp of the occupant (Map.cc:197)
};
struct WireDesc {
    const WireHdr *hdr;                  // [n_total]            (page-locked staging owned by the context)
    const WireMark *marks;               // [chunk_base[n_chunks]]
    const long long *chunk_base;         // [n_chunks + 1]
    const float *mm;                     // [A][mm_stride] normalised minimap rows, or nullptr
    int mm_stride;
    int n_total, n_chunks;
    int n_waves, chunks_per_wave;        // the staging fills wave by wave (obs_wire_wait): wave w = chunks [w * cpw, (w + 1) * cpw)
    int wave_order[16];                  // the order the waves were queued in (front and back half alternate, so that the
                                         // threads of every NUMA part of the caller's buffer find work early)
};
// Launch the wire kernels for observation O (feature rows into O.feature, device staging), read the totals back and queue
// the device->host copies of headers and marks, wave by wave.
void obs_wire_begin(Ctx *, const EngineDev *dE, const EngineDev &hE, const ObsArgs &O, const float *mm_val, int n_total,
                    WireDesc *out);
void obs_wire_wait(Ctx *, int wave);     // returns once wave `wave` is in host memory
// asynchronous device->host copies on the context's copy stream (feature rows of a host-buffer observation)
void dma_d2h_async(Ctx *, void *dst, const void *src, size_t bytes);
void dma_wait(Ctx *, int keep_in_flight);   // wait until at most `keep_in_flight` of the queued copies are outstanding

// ---- CUDA graphs for launch-bound (small) workloads: everything the engine queues on its stream between begin and end
// becomes one graph; a replay costs one launch.  While capturing, the backend refuses anything that cannot be captured
// (allocation growth, host synchronisation).  Returns false when the backend has no graph support (test emulation).
bool capture_begin(Ctx *);
int capture_end(Ctx *);                  // instantiates; returns the graph's id (>= 0)
bool capturing(const Ctx *);
void graph_launch(Ctx *, int id);
void graph_destroy_all(Ctx *);

// instrumentation: kernel launch counter and optional CUDA-event timing of the obs-render kernel
long long launch_count();
void profile_enable(Ctx *, bool on);
void profile_read(Ctx *, double *obs_ms_total, long long *obs_launches);

}  // namespace be
}  // namespace mg
