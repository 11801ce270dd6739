/*
 * magent_b200_ext.h -- entry points the B200 engine adds next to the reference ABI.
 * None of them exists in the reference library; a caller that never uses them is a pure drop-in.
 */
#ifndef MAGENT_B200_EXT_H
#define MAGENT_B200_EXT_H
#include <stddef.h>
#include "magent_runtime_api.h"

#ifdef __cplusplus
extern "C" {
#endif

int magent_b200_version(void);                 /* 1000*major + minor */
const char *magent_b200_last_error(void);
int magent_b200_device_count(void);            /* 0 when no CUDA device is visible */

/* page-locked host memory for observation / reward receive buffers.  Blocks of 64 MB and more on a multi-socket host are
 * striped over the NUMA nodes (32 MB stripes, each resident on its node and written by that node's threads in
 * env_get_observation). */
void *magent_b200_host_alloc(size_t bytes);
int magent_b200_host_free(void *p);
int magent_b200_numa_nodes(void);              /* NUMA nodes the host threads are spread over (1 = not NUMA) */

int magent_b200_sync(EnvHandle game);          /* wait for all queued device work of this game */
/* env_step(game, done) also accepts a CUDA device pointer for `done`: the flag is written on the device and the call
 * returns without waiting for the step (device-resident loops; reference src/runtime_api.h:31 takes a host int). */
/* route the following setup calls (add_agents, seed) to one arena of the batch; -1 = all arenas */
int magent_b200_select_arena(EnvHandle game, int arena);
/* set_action with uniform random actions generated on the device (throughput runs; not part of parity).
 * `unused` must be NULL. */
int magent_b200_random_actions(EnvHandle game, GroupHandle group, void *unused, unsigned long long seed);
/* compact observation hand-off (SURVEY.md 8f rank 2): same call, layout and pointer rules as env_get_observation
 * (reference src/runtime_api.h:35), but every element is an IEEE binary16 = the float32 value rounded to
 * nearest-even.  buffer[0] = view [n][view_h][view_w][n_channel], buffer[1] = feature [n][feature_size];
 * host or CUDA device pointers.  Halves the HBM / PCIe bytes per observation. */
int magent_b200_get_observation_f16(EnvHandle game, GroupHandle group, void **buffer);
/* global state (centralised critics): the whole map of every arena as one image, [num_arenas][H][W][C] with
 * C = 1 + food_mode + 2 * n_group; env_get_info(game, -1, "state_space", int[3]) gives (H, W, C).  Per map cell:
 *   channel 0                   1.0 on a wall (border walls included)
 *   channel 1 (food_mode only)  1.0 on food
 *   channel base + 2g           1.0 where an agent of group g stands (every cell of its body), base = 1 + food_mode
 *   channel base + 2g + 1       that agent's hp / max_hp
 * and 0 elsewhere.  Every value is the one a view covering the cell shows; groups are in absolute order (group 0
 * first), not in the observer-relative order of the views, and there are no minimap channels.  Covers every arena
 * whatever magent_b200_select_arena says.  half = 0: float32; half = 1: IEEE binary16, the float32 value rounded to
 * nearest-even.  `buffer` is host memory or a 16-byte aligned CUDA device pointer.  With a device pointer the call
 * needs no agent counts: it neither synchronises nor allocates once the game runs on the device, so it can be
 * recorded into a CUDA graph. */
int magent_b200_get_global_state(EnvHandle game, void *buffer, int half);
/* int64 event counters since construction: agent_steps, attacks, hits, kills, starved, moves_ok,
 * moves_blocked, steps.  Returns the number written. */
int magent_b200_get_counters(EnvHandle game, long long *out, int capacity);

/* instrumentation: kernels launched by this library in this process; optional CUDA-event timing of the
 * obs-render kernel of one game (total milliseconds and launches since enabled; read after the fact, no sync added). */
long long magent_b200_launch_count(void);
int magent_b200_set_profiling(EnvHandle game, int on);
int magent_b200_get_profile(EnvHandle game, double *obs_ms_total, long long *obs_launches);
/* bytes moved by the step-loop calls of this game so far: [0] device->host over PCIe, [1] host->device, [2] written into
 * caller host buffers by the engine's host threads (env_get_observation with host pointers); [3..5] microseconds the
 * host-buffer observation calls spent producing wire records / expanding them / finishing the feature rows.
 * Returns the number written. */
int magent_b200_get_io_stats(EnvHandle game, long long *out, int capacity);
/* CUDA graphs for launch-bound (small) workloads.  Every step-loop call made with CUDA device pointers between begin and
 * end is recorded instead of executed (actions, rewards, observations and `done` in caller-owned device buffers); the
 * recorded sequence must contain an even number of gridworld_clear_dead calls (two steps).  graph_launch replays it
 * `times` times: one launch per replay instead of one per kernel.  The caller refills its action buffers between
 * replays; counts / ids / positions are read with the usual calls after a replay. */
int magent_b200_graph_begin(EnvHandle game);
int magent_b200_graph_end(EnvHandle game);     /* returns the graph id */
int magent_b200_graph_launch(EnvHandle game, int graph_id, int times);
/* the cudaStream_t all kernels of this game are launched on (a blocking stream: work on the legacy default stream is
 * ordered with it both ways, so CUDA-pointer consumers on the default stream need no extra synchronisation) */
void *magent_b200_stream(EnvHandle game);
/* host threads env_get_observation uses to write host buffers (MAGENT_B200_HOST_THREADS overrides) */
int magent_b200_host_threads(void);
int magent_b200_set_host_threads(int n);       /* 0 = default (usable cores, at most 16; 24 on hosts with 48+ usable cores) */

#ifdef __cplusplus
}
#endif
#endif
