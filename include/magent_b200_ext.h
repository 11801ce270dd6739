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
/* legal-action mask: uint8 [n][n_action] in ABI order (the rows of env_set_action, un-culled dead agents included).
 * Byte [i][k] is 1 iff action k, taken by agent i alone on the state as it is now, would succeed:
 *   move    the target footprint is inside the board by the reference's own test, free of walls and food, and every cell
 *           is empty or the mover's own (the centre move of a live agent is therefore always 1); or the first other
 *           agent in the blocked footprint is an absorbing type that has not absorbed yet (the mover would be swallowed)
 *   turn    (turn_mode) the rotated footprint is free or the agent's own
 *   attack  the aimed cell is on the board and holds an agent of another group, of the own group when the type has
 *           attack_in_group, or food (food_mode)
 * What other agents do in the same step is not anticipated.  A dead, un-culled agent has an all-zero row; an absorbed
 * absorber has no legal move (its turns and attacks are decided as for anyone else).  Returns -1 for a bad group handle,
 * and returns -1, sets magent_b200_last_error and writes nothing when 256 rows of n_action bytes do not fit the device's
 * shared memory per block (on an H100: more than 881 actions; DESIGN.md §5 "Shared-memory limits").
 * Host pointer or CUDA device pointer.  With a device pointer: no synchronisation, no allocation, recordable into a CUDA
 * graph; rows are sized by the device-side counts, at most "num_bound" of them are written.  magent_b200_select_arena
 * does not apply. */
int magent_b200_get_action_mask(EnvHandle game, GroupHandle group, unsigned char *buffer);
/* set_action with an action drawn uniformly from the legal actions (the mask above) of every agent, on the device; an
 * agent without a legal action gets action 0, which the step ignores for it.  Same seeding discipline as
 * magent_b200_random_actions: the call counter of both calls and the device step counter ride in the seed, so a replayed
 * graph draws fresh actions.  Not part of parity.  Returns -1 for a bad group handle. */
int magent_b200_random_legal_actions(EnvHandle game, GroupHandle group, unsigned long long seed);
/* mean neighbour action (mean-field Q-learning / actor-critic): for every agent i of `group`, in ABI order (the rows of
 * env_set_action, arenas concatenated), the mean one-hot action of its neighbours of group `of` (`of` == `group` is
 * allowed).  The neighbours N(i) are the distinct agents j != i of `of`, in i's arena, whose presence i's own view shows:
 * some in-range cell of i's view window (turn_mode: laid out in i's frame, as env_get_observation does) is a map cell
 * that j's body covers.  A body larger than 1 x 1 counts once however many of its cells are in view.
 *   count[i]   = |N(i)|                                                             int32 [n], may be NULL
 *   mean[i][k] = (float)#{j in N(i): act_j == k} / (float)count[i], k < n_action(of)   float32 [n][n_action(of)]
 * with IEEE round-to-nearest division.  act_j is the action j holds now: the one set_action / random_actions /
 * random_legal_actions last gave it, which is the one the last env_step executed until the next set.  So called after
 * env_step and before the next set_action it gives the previous step's mean action (what mean-field methods condition on);
 * called after set_action it gives the actions just set.  A neighbour whose action is outside [0, n_action(of)) (added
 * since the last step, or an id the step ignores) is counted in count and in no bin: its row sums to less than 1.  A row
 * without neighbours is all zero; a dead, un-culled agent has an all-zero row and count 0.  Returns -1 for a bad `group`
 * or `of` handle, or when one pointer is host memory and the other a CUDA device pointer; and returns -1, sets
 * magent_b200_last_error and writes nothing when the view LUT of `group` (one per heading in turn_mode) and eight
 * histograms of n_action(of) ints do not fit the device's shared memory per block (on an H100 with 21 actions: circle
 * views of radius 95 and more, 48 and more in turn_mode; DESIGN.md §5 "Shared-memory limits").  Both host pointers: the call
 * waits for the counts.  Both CUDA device pointers: no synchronisation, no allocation, recordable into a CUDA graph; rows
 * are sized by the device-side counts, at most "num_bound" of them are written.  magent_b200_select_arena does not
 * apply. */
int magent_b200_get_mean_action(EnvHandle game, GroupHandle group, GroupHandle of, float *mean, int *count);
/* nearest visible neighbours (graph-convolutional and attention policies): for every agent i of `group`, in ABI order,
 * the first k of its neighbours N(i) in group `of`, nearest first.  N(i) is exactly the neighbour set of
 * magent_b200_get_mean_action (`of` == `group` allowed).  Every view cell (vx, vy) of i's window (turn_mode: laid out in
 * i's frame) has the key (d2, vy * view_w + vx), compared in that order: d2 is the squared Euclidean distance, in map
 * cells, from the map cell it shows to i's footprint [x, x + bw) x [y, y + bh) (body dimensions rotated by i's heading;
 * 0 on the footprint itself).  The distance is to the body, not to the window centre, because sector views do not centre
 * the window on the observer.  A neighbour's key is the smallest key among the in-range, on-board cells of i's window that
 * its body covers (a body larger than 1 x 1 appears once, at its nearest visible cell).  Neighbours are ordered by key
 * and the first min(k, |N(i)|) are written:
 *   idx[i][r]    = j's row in group `of`'s ABI concatenation now (its arena's offset + its index): its row in
 *                  get_observation(of), get_pos(of) and any per-agent tensor kept in that order     int32 [n][k]
 *   rel[i][r][:] = (vy, vx), the view cell where that nearest visible cell lies: where i's own observation shows j
 *                                                                                 int32 [n][k][2], may be NULL
 *   count[i]     = |N(i)|, not capped by k (= get_mean_action's count)            int32 [n], may be NULL
 * Unused slots hold -1 (rel: (-1, -1)).  A dead, un-culled observer has an all -1 row and count 0; dead neighbours have
 * left the map.  The indices go stale with the next clear_dead, restore_arenas or add_agents, like every row-ordered
 * output.  1 <= k <= 32.  Returns -1, sets magent_b200_last_error and writes nothing for a bad `group` or `of` handle, k
 * out of range, a NULL idx, pointers that mix host and CUDA device memory, or a backend without the kernel.  Host
 * pointers: the call waits for the counts.  CUDA device pointers: no synchronisation, no allocation, recordable into a
 * CUDA graph; rows are sized by the device-side counts, at most "num_bound" of them are written.
 * magent_b200_select_arena does not apply. */
int magent_b200_get_neighbours(EnvHandle game, GroupHandle group, GroupHandle of, int k, int *idx, int *rel, int *count);
/* stable agent slots (rollout buffers, recurrent state, mixers: anything that needs one fixed index per agent for the
 * whole episode, and fixed-shape CUDA-graph training steps).  Every row-ordered output keeps its row order; this call
 * serves the two index maps between rows and slots.
 *   The slot of an agent is the number of agents of its group that were placed into its arena before it since that
 *   arena's last env_reset.  Placement is add_agents in any method, including mid-episode and through
 *   magent_b200_select_arena.  So right after placement the slot equals the agent's index within its arena and group.  A
 *   slot is never reused within an episode, and clear_dead keeps it.  A restored arena's agents take the slots they have
 *   in the snapshot arena, and the arena's slot counters come from the snapshot too.  env_reset starts over at 0.
 *   The slot space S(g) is the largest slot count of group g over all arenas in their current episode and over every
 *   live snapshot's arenas.  It is therefore a bound that no device-side restore can exceed.  Only host-side calls change
 *   it: env_reset, add_agents, snapshot_arenas and free_snapshot.  Read it with env_get_info(game, -1, "slot_space",
 *   int[n_group]), which never waits, like "num_bound".
 *   row_slot[r] = a * S + slot                int32 [num_bound(group)], may be NULL
 *                 for each row r (the rows of env_set_action) below the device-side total of the group, a being the row's
 *                 arena; -1 from the device-side total up to num_bound: the valid-row mask of a device consumer
 *   slot_row[a][slot] = r                     int32 [num_arenas][S], may be NULL
 *                 the row of the agent occupying the slot, or -1 when the slot is vacant (never placed in this episode,
 *                 or its agent was culled).  A dead agent that has not been culled keeps its row.
 * Either pointer may be NULL, but not both.  Both host pointers: the call waits for the counts.  Both CUDA device
 * pointers: no synchronisation, no allocation, recordable into a CUDA graph, also after a restore from a device src
 * inside the graph.  Returns -1, sets magent_b200_last_error and writes nothing for a bad group handle, two NULL
 * pointers, pointers that mix host and CUDA device memory, or a backend without the kernel.  magent_b200_select_arena
 * does not apply. */
int magent_b200_get_slots(EnvHandle game, GroupHandle group, int *row_slot, int *slot_row);
/* the observation of one group in the stable [arena, slot] layout of magent_b200_get_slots, rendered in that order:
 *   buffer[0] = view [num_arenas][S][view_h][view_w][n_channel], buffer[1] = feature [num_arenas][S][feature_size],
 *   S = env_get_info(game, -1, "slot_space", int[n_group])[group].
 * An occupied slot (a, s) holds, bit for bit, the view record and feature row env_get_observation (half = 1:
 * magent_b200_get_observation_f16) writes at the same moment for row slot_row[a][s]; a dead agent that has not been culled
 * keeps its slot and its record.  A vacant slot holds an all-zero view record and feature row (+0.0).  half = 0:
 * float32; half = 1: IEEE binary16, the float32 value rounded to nearest-even.  Covers every arena whatever
 * magent_b200_select_arena says; S == 0 writes nothing.  Both CUDA device pointers: no synchronisation and, once a
 * first call has sized the engine's tables, no allocation, so the call can be recorded into a CUDA graph, also after a
 * restore from a device src inside the graph (the device decides which slots hold rows).  Both host pointers: rendered
 * into device staging and copied back (counted in the d2h figure of magent_b200_get_io_stats).  Returns -1, sets
 * magent_b200_last_error and writes nothing for a bad group handle, half other than 0 or 1, a NULL pointer, pointers that
 * mix host and CUDA device memory, or a backend without the kernel. */
int magent_b200_get_observation_slots(EnvHandle game, GroupHandle group, void **buffer, int half);
/* The rest of a fixed-shape step loop in the [arena, slot] layout of magent_b200_get_slots: actions in, rewards, agent
 * status and legal-action masks out.  S = env_get_info(game, -1, "slot_space", int[n_group])[group], A = num_arenas.
 * The shapes are known on the host and the device decides which slots hold rows (the device-side offsets and the slot
 * table), so none of the three calls waits for the agent counts, whatever the pointer kind.  Both CUDA device pointers:
 * no synchronisation and no allocation (get_action_mask_slots: once a first call has sized the engine's tables), so
 * the calls can be recorded into a CUDA graph, also after a restore from a device src inside the graph.  They cover
 * every arena whatever magent_b200_select_arena says.
 *
 * set_action_slots: act is int32 [A][S].  Every agent of the group, at its row r below the device-side count, takes
 * act[a * S + slot] as its action, (a, slot) being its arena and slot.  Values in vacant slots are never read, so they
 * may be anything, out-of-range ids included.  The engine state afterwards is bit for bit what env_set_action(game, group,
 * rows) leaves with rows[r] = act[row_slot[r]], including every later step output and magent_b200_get_mean_action.  The
 * call is the group's set_action for this step: it takes the same place in the step's action order, makes
 * magent_b200_restore_arenas refuse until env_step as set_action does, and a second call for the group in the same step
 * (this one or env_set_action) overwrites.  S == 0: only registers the group's action, reads nothing, act may be NULL.
 * A host act is copied in (A * S * 4 bytes, counted in the h2d figure of magent_b200_get_io_stats).  Returns -1, sets
 * magent_b200_last_error, writes nothing and registers nothing for a bad group handle, a NULL act when S > 0, or a
 * backend without the kernel. */
int magent_b200_set_action_slots(EnvHandle game, GroupHandle group, const int *act);
/* reward[a][s] = bit for bit the value env_get_reward gives the row in slot (a, s), +0.0 in a vacant slot
 *                                                                                 float32 [A][S], may be NULL
 * status[a][s] = 0 vacant, 1 the row's env_get_info("alive") is 1, 2 occupied by a dead agent that has not been culled
 *                yet: between env_step and gridworld_clear_dead, 2 is the per-agent terminal signal; after the cull
 *                those slots read 0                                               uint8 [A][S], may be NULL
 * Either pointer may be NULL, but not both.  Host pointers are copied back and counted in the d2h figure, exactly the
 * bytes asked for.  Returns -1, sets magent_b200_last_error and writes nothing for a bad group handle, two NULL pointers,
 * pointers that mix host and CUDA device memory, or a backend without the kernel. */
int magent_b200_get_reward_slots(EnvHandle game, GroupHandle group, float *reward, unsigned char *status);
/* mask uint8 [A][S][n_action]: an occupied slot's row is bit for bit the row magent_b200_get_action_mask gives its
 * agent's row (a dead, un-culled agent's row is all zero); a vacant slot's row is all zero.  Host pointer: copied back
 * and counted in the d2h figure.  Returns -1, sets magent_b200_last_error and writes nothing for a bad group handle, a
 * NULL mask, a backend without the kernel, or an action space magent_b200_get_action_mask refuses. */
int magent_b200_get_action_mask_slots(EnvHandle game, GroupHandle group, unsigned char *mask);
/* The mean neighbour action and the nearest visible neighbours in the [arena, slot] layout of magent_b200_get_slots.
 * S = slot_space(group), S_of = slot_space(of) (env_get_info "slot_space"), A = num_arenas; slot_row and row_slot are the
 * maps magent_b200_get_slots serves at the same moment, row_slot_of those of group `of`.
 *   get_mean_action_slots: mean float32 [A][S][n_action(of)], count int32 [A][S] (may be NULL).  An occupied slot (a, s)
 *     holds, bit for bit, the row magent_b200_get_mean_action gives row slot_row[a][s] (a dead, un-culled agent's row is
 *     zero and its count 0, as there); a vacant slot a +0.0 row and count 0.
 *   get_neighbours_slots: idx int32 [A][S][k], rel int32 [A][S][k][2] and count int32 [A][S] (rel and count may be
 *     NULL), 1 <= k <= 32.  An occupied slot holds the row magent_b200_get_neighbours gives row slot_row[a][s], with every
 *     used idx entry the neighbour's flat slot row_slot_of[its row] = a * S_of + slot_of instead of its row: gather
 *     slot-ordered features of `of` with hid_s.view(A * S_of, d)[idx.clamp(min=0)].  rel and count are the row call's;
 *     unused entries are -1.  A vacant slot holds -1 everywhere and count 0.  Unlike row indices, these stay valid for the
 *     whole episode: after a clear_dead one may point at a vacant slot (its agent was culled), never at another agent.
 * Neither call waits for the agent counts, whatever the pointer kind.  Both CUDA device pointers: no synchronisation and,
 * once a first call has sized the engine's tables, no allocation, so the calls can be recorded into a CUDA graph, also
 * after a restore from a device src inside the graph.  Host pointers: computed into device staging and copied back,
 * counted in the d2h figure (exactly the bytes asked for).  They cover every arena whatever magent_b200_select_arena
 * says; S == 0 writes nothing.  Returns -1, sets magent_b200_last_error and writes nothing for a bad `group` or `of`
 * handle, k out of range, a NULL mean / idx, pointers that mix host and CUDA device memory, a view too large to order
 * its cells by an int key (as magent_b200_get_neighbours refuses it), a mean action magent_b200_get_mean_action refuses
 * for its shared memory, or a backend without the kernel. */
int magent_b200_get_mean_action_slots(EnvHandle game, GroupHandle group, GroupHandle of, float *mean, int *count);
int magent_b200_get_neighbours_slots(EnvHandle game, GroupHandle group, GroupHandle of, int k, int *idx, int *rel,
                                     int *count);
/* Built-in scripted opponents: a fixed, non-trivial policy to train against or to measure progress by, decided on the
 * device.  For every agent i of `group` and a target group `target` (t; t == group allowed), on the state as it is now:
 *   MAGENT_B200_RULE_RUSH
 *     1. attack: among the attack actions k that magent_b200_get_action_mask allows i and whose aimed cell holds an agent
 *        of t other than i, the one whose target agent has the lowest hp now (env_get_info "hp"); ties to the lowest k.
 *     2. approach: otherwise, when i sees an agent of t, let c be the map cell that magent_b200_get_neighbours(group,
 *        of = t, k = 1) lists for i (its nearest visible target, at its smallest-key cell; turn_mode headings, sector
 *        views and longer bodies as stated there).  Among the move actions k < n_move that the mask allows (turn actions
 *        never count), the one whose moved footprint [nx, nx + bw) x [ny, ny + bh) (the body after the move, rotated by
 *        i's heading) has the smallest squared distance to c: ex^2 + ey^2, ex = nx - cx when cx < nx, cx - (nx + bw - 1)
 *        when cx >= nx + bw, else 0 (ey likewise), as the neighbours' key measures d2.  Ties to the lowest k.
 *     3. fallback: otherwise, the action magent_b200_random_legal_actions(game, group, seed) would set for i if it were
 *        called in this call's place.  This call does not count as one of its calls: it leaves the call counter that
 *        random_actions and random_legal_actions share where it was.
 *   MAGENT_B200_RULE_FLEE: step 2 with the largest distance instead of the smallest, when i sees an agent of t; otherwise
 *     step 3.
 * Step 2 with no legal move falls through to step 3.  A dead, un-culled agent and an agent with no legal action take
 * action 0, which the step ignores for it.  Food cells (food_mode) are never targets; an absorber is one like any agent.
 * Typical targets: the enemy in battle, the prey for pursuit's predators (rush), the predators for pursuit's prey (flee),
 * the food group in gather.  The fallback, like random_legal_actions, folds the device step counter into the seed, so
 * a replayed CUDA graph draws afresh.
 *   rule_actions: sets the decisions as the group's actions for this step; it counts as the group's set_action (same
 *     place in the step's action order, blocks magent_b200_restore_arenas until env_step).  No synchronisation and no
 *     allocation: recordable into a CUDA graph.
 *   get_rule_actions: int32 [n] in row order (the rows of env_set_action), the actions rule_actions would set.  Host
 *     pointer: the call waits for the counts.  CUDA device pointer: no synchronisation, no allocation, recordable into a
 *     CUDA graph; rows are sized by the device-side counts, at most "num_bound" of them are written.
 *   get_rule_actions_slots: int32 [A][S] in the [arena, slot] layout of magent_b200_get_slots: an occupied slot holds the
 *     row call's action for row slot_row[a][s], a vacant slot -1.  Does not wait for the counts, whatever the pointer
 *     kind; CUDA device pointer: no synchronisation and, once a first call has sized the engine's tables, no allocation.
 * None of them sets or reads anything else.  They cover every arena whatever magent_b200_select_arena says.  Returns -1,
 * sets magent_b200_last_error and writes or registers nothing for a bad `group` or `target` handle, a policy other than
 * the two below, a NULL act where something is to be written, a view of `group` too large to order its cells by an int key
 * (as magent_b200_get_neighbours refuses it), or a backend without the kernel. */
#define MAGENT_B200_RULE_RUSH 0
#define MAGENT_B200_RULE_FLEE 1
int magent_b200_rule_actions(EnvHandle game, GroupHandle group, GroupHandle target, int policy, unsigned long long seed);
int magent_b200_get_rule_actions(EnvHandle game, GroupHandle group, GroupHandle target, int policy,
                                 unsigned long long seed, int *act);
int magent_b200_get_rule_actions_slots(EnvHandle game, GroupHandle group, GroupHandle target, int policy,
                                       unsigned long long seed, int *act);
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
/* reset pool: restart finished arenas of the batch without leaving the device.  Take a snapshot once, after placement
 * (placement itself stays on the host, bit-exact with the reference), and later restore any subset of arenas from it.
 * The calls below return -1 and set magent_b200_last_error when they refuse; the state is then unchanged.
 *
 * snapshot_arenas copies the current state of every arena into new device memory of its own and returns the
 * snapshot's id (>= 0).  Ids are not reused; free_snapshot releases one.  A snapshot restored inside a recorded CUDA
 * graph lives as long as the game. */
int magent_b200_snapshot_arenas(EnvHandle game);
int magent_b200_free_snapshot(EnvHandle game, int snapshot);
/* src: int32[num_arenas], host or CUDA device pointer.  src[a] = -1 keeps arena a byte for byte; src[a] = s in
 * [0, num_arenas) makes it exactly arena s of the snapshot: map, food, every agent with its order, ids, hp, rewards,
 * last op and heading, the per-arena counters and reward state, the done flag, the agent id counter, and, when
 * keep_rng = 0, the RNG state (keep_rng = 1: the arena keeps its own minstd stream).  src == NULL: every arena whose
 * last env_step reported done is replaced by its own index (src[a] = a), decided on the device.  On the device,
 * values outside [0, num_arenas) mean -1; a host src holding one is refused.  magent_b200_select_arena does not apply.
 * Refused: actions set for the current step (call env_step first), rendering started, an unknown or freed snapshot,
 * a snapshot taken under another geometry (map size, groups, agent types, food_mode, turn_mode).
 * With a device pointer or NULL the call neither synchronises nor allocates, so it can be recorded into a CUDA graph.
 *
 * Counts: env_get_info "num" stays exact (it waits for the counts, as after gridworld_clear_dead).  Without waiting,
 * env_get_info(game, -1, "num_bound", int[n_group]) gives per group the most records a device-pointer call can write
 * before the counts next settle.  While any snapshot exists, a CUDA graph sizes every count-dependent launch it records
 * (before or after a restore) for the counts a restore can produce: size the device buffers of such a graph by
 * "num_bound".  env_get_info(game, -1, "arena_rng", uint32[num_arenas]) gives each arena's minstd state (a value for
 * the "seed" key would have to be this to continue the stream). */
int magent_b200_restore_arenas(EnvHandle game, int snapshot, const int *src, int keep_rng);
/* per-arena done flags of the last env_step into int32[num_arenas], host or CUDA device pointer; with a device pointer
 * nothing is waited for */
int magent_b200_get_arena_done(EnvHandle game, int *out);
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

/* ---- extension keys of the reference calls env_config_game / env_get_info (no entry point of their own) ----
 *
 * Render launch shape of one game (tests and measurement; the defaults are the tuned choice).  env_config_game keys,
 * int values, changeable between calls, 0 = automatic: "obs_grid" CTAs (clamped to [1, tiles]), "obs_chunk" consecutive
 * tiles per CTA visit (clamped to [1, ceil(tiles / grid)]), "obs_tile" 1 = narrow, 2 = wide (narrow when the wide tile
 * does not fit in shared memory).  A negative value or obs_tile > 2 is refused: env_config_game returns -1 and nothing
 * changes.  env_get_info(game, -1, "obs_override", int[3]) reads the three keys back.
 * env_get_info(game, -1, "obs_launch", int[8]) reports the last obs_render_kernel launch of the game: {sizeof(T), NIT,
 * turn, agents per tile, grid, chunk, tiles, view and feature buffers both 16-byte aligned}, zeros before the first.
 * env_get_info(game, -1, "step_launch", int[10]) reports the last step and clear_dead launches of the game, five ints
 * each (step first): {mode (0 a CTA per arena, 1 the whole-grid team), grid, threads, dynamic shared-memory bytes, step
 * scratch in shared memory}, zeros before the first. */

#ifdef __cplusplus
}
#endif
#endif
