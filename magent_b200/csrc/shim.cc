// shim.cc -- the extern "C" boundary (include/magent_runtime_api.h) over mg::Engine.
// Same role as the reference src/runtime_api.cc:15-163: cast the opaque handle, forward, return 0.
#include <stdio.h>
#include <string.h>
#include <string>

#include "../../include/magent_b200_ext.h"
#include "backend.h"
#include "engine.h"
#include "host_expand.h"

namespace mg { const char *last_error(); void set_last_error(const std::string &s); }

#define MG_API extern "C" __attribute__((visibility("default")))
static inline mg::Engine *E(EnvHandle h) { return (mg::Engine *)h; }

MG_API int env_new_game(EnvHandle *game, const char *name) {
    if (strcmp(name, "GridWorld") != 0) {
        mg::set_last_error(std::string("unsupported game for the B200 engine: ") + name);
        fprintf(stderr, "[magent_b200] %s\n", mg::last_error());
        *game = nullptr;
        return -1;
    }
    std::string err;
    if (mg::be::device_count() <= 0) {
        mg::set_last_error("no CUDA device visible: the B200 engine has no CPU fallback");
        fprintf(stderr, "[magent_b200] %s\n", mg::last_error());
        *game = nullptr;
        return -1;
    }
    *game = new mg::Engine();
    return 0;
}
MG_API int env_delete_game(EnvHandle game) { delete E(game); return 0; }
MG_API int env_config_game(EnvHandle game, const char *name, void *p_value) { return E(game)->set_config(name, p_value); }
MG_API int env_reset(EnvHandle game) { E(game)->reset(); return 0; }
MG_API int env_get_observation(EnvHandle game, GroupHandle group, float **buffer) { E(game)->get_observation(group, (void **)buffer, 0); return 0; }
MG_API int env_set_action(EnvHandle game, GroupHandle group, const int *actions) { E(game)->set_action(group, actions); return 0; }
MG_API int env_step(EnvHandle game, int *done) { E(game)->step(done); return 0; }
MG_API int env_get_reward(EnvHandle game, GroupHandle group, float *buffer) { E(game)->get_reward(group, buffer); return 0; }
MG_API int env_get_info(EnvHandle game, GroupHandle group, const char *name, void *buffer) { return E(game)->get_info(group, name, buffer); }
MG_API int env_render(EnvHandle game) { E(game)->render(); return 0; }
MG_API int env_render_next_file(EnvHandle game) { E(game)->render_next_file(); return 0; }

MG_API int gridworld_register_agent_type(EnvHandle game, const char *name, int n, const char **keys, float *values) {
    E(game)->register_agent_type(name, n, keys, values); return 0;
}
MG_API int gridworld_new_group(EnvHandle game, const char *agent_type_name, GroupHandle *group) {
    E(game)->new_group(agent_type_name, group); return 0;
}
MG_API int gridworld_add_agents(EnvHandle game, GroupHandle group, int n, const char *method,
                                const int *pos_x, const int *pos_y, const int *dir) {
    E(game)->add_agents(group, n, method, pos_x, pos_y, dir); return 0;
}
MG_API int gridworld_clear_dead(EnvHandle game) { E(game)->clear_dead(); return 0; }
MG_API int gridworld_set_goal(EnvHandle game, GroupHandle group, const char *method, const int *linear_buffer) {
    E(game)->set_goal(group, method, linear_buffer); return 0;
}
MG_API int gridworld_define_agent_symbol(EnvHandle game, int no, int group, int index) {
    E(game)->define_agent_symbol(no, group, index); return 0;
}
MG_API int gridworld_define_event_node(EnvHandle game, int no, int op, int *inputs, int n_inputs) {
    E(game)->define_event_node(no, op, inputs, n_inputs); return 0;
}
MG_API int gridworld_add_reward_rule(EnvHandle game, int on, int *receiver, float *value, int n_receiver,
                                     bool is_terminal, bool auto_value) {
    E(game)->add_reward_rule(on, receiver, value, n_receiver, is_terminal, auto_value); return 0;
}

MG_API int discrete_snake_clear_dead(EnvHandle) {
    mg::fatal("DiscreteSnake is not part of the B200 engine (SURVEY.md §2 row 11)");
}
MG_API int discrete_snake_add_object(EnvHandle, int, int, const char *, const int *) {
    mg::fatal("DiscreteSnake is not part of the B200 engine (SURVEY.md §2 row 11)");
}

// ---- extensions
MG_API int magent_b200_version(void) { return 1000 * 0 + 1; }
MG_API const char *magent_b200_last_error(void) { return mg::last_error(); }
MG_API int magent_b200_device_count(void) { return mg::be::device_count(); }
// Receive buffers for observations.  Large ones on a multi-socket host are split over the NUMA nodes (one part per node,
// written by that node's threads: host_expand.h) and page-locked in place; everything else is plain page-locked memory.
MG_API void *magent_b200_host_alloc(size_t bytes) {
    if (mg::be::device_count() <= 0) return nullptr;
    if (bytes >= ((size_t)64 << 20) && mg::numa_nodes() > 1) {
        if (void *p = mg::numa_split_alloc(bytes)) {
            mg::be::host_register(p, mg::numa_split_size(p));
            return p;
        }
    }
    return mg::be::host_alloc(bytes);
}
MG_API int magent_b200_host_free(void *p) {
    if (mg::numa_split_size(p)) { mg::be::host_unregister(p); mg::numa_split_free(p); return 0; }
    mg::be::host_free(p);
    return 0;
}
MG_API int magent_b200_numa_nodes(void) { return mg::numa_nodes(); }
MG_API int magent_b200_sync(EnvHandle game) { E(game)->sync(); return 0; }
MG_API int magent_b200_select_arena(EnvHandle game, int arena) { E(game)->select_arena(arena); return 0; }
MG_API int magent_b200_random_actions(EnvHandle game, GroupHandle group, void *, unsigned long long seed) {
    E(game)->random_actions(group, seed); return 0;
}
MG_API int magent_b200_get_action_mask(EnvHandle game, GroupHandle group, unsigned char *buffer) {
    return E(game)->get_action_mask(group, buffer);
}
MG_API int magent_b200_random_legal_actions(EnvHandle game, GroupHandle group, unsigned long long seed) {
    return E(game)->random_legal_actions(group, seed);
}
MG_API int magent_b200_get_mean_action(EnvHandle game, GroupHandle group, GroupHandle of, float *mean, int *count) {
    return E(game)->get_mean_action(group, of, mean, count);
}
MG_API int magent_b200_get_neighbours(EnvHandle game, GroupHandle group, GroupHandle of, int k, int *idx, int *rel,
                                      int *count) {
    return E(game)->get_neighbours(group, of, k, idx, rel, count);
}
MG_API int magent_b200_get_slots(EnvHandle game, GroupHandle group, int *row_slot, int *slot_row) {
    return E(game)->get_slots(group, row_slot, slot_row);
}
MG_API int magent_b200_get_observation_slots(EnvHandle game, GroupHandle group, void **buffer, int half) {
    return E(game)->get_observation_slots(group, buffer, half);
}
MG_API int magent_b200_set_action_slots(EnvHandle game, GroupHandle group, const int *act) {
    return E(game)->set_action_slots(group, act);
}
MG_API int magent_b200_get_reward_slots(EnvHandle game, GroupHandle group, float *reward, unsigned char *status) {
    return E(game)->get_reward_slots(group, reward, status);
}
MG_API int magent_b200_get_action_mask_slots(EnvHandle game, GroupHandle group, unsigned char *mask) {
    return E(game)->get_action_mask_slots(group, mask);
}
MG_API int magent_b200_get_mean_action_slots(EnvHandle game, GroupHandle group, GroupHandle of, float *mean, int *count) {
    return E(game)->get_mean_action_slots(group, of, mean, count);
}
MG_API int magent_b200_get_neighbours_slots(EnvHandle game, GroupHandle group, GroupHandle of, int k, int *idx, int *rel,
                                            int *count) {
    return E(game)->get_neighbours_slots(group, of, k, idx, rel, count);
}
MG_API int magent_b200_rule_actions(EnvHandle game, GroupHandle group, GroupHandle target, int policy,
                                    unsigned long long seed) {
    return E(game)->rule_actions(group, target, policy, seed);
}
MG_API int magent_b200_get_rule_actions(EnvHandle game, GroupHandle group, GroupHandle target, int policy,
                                        unsigned long long seed, int *act) {
    return E(game)->get_rule_actions(group, target, policy, seed, act);
}
MG_API int magent_b200_get_rule_actions_slots(EnvHandle game, GroupHandle group, GroupHandle target, int policy,
                                              unsigned long long seed, int *act) {
    return E(game)->get_rule_actions_slots(group, target, policy, seed, act);
}
MG_API int magent_b200_get_observation_f16(EnvHandle game, GroupHandle group, void **buffer) {
    E(game)->get_observation(group, buffer, 1);
    return 0;
}
MG_API int magent_b200_get_global_state(EnvHandle game, void *buffer, int half) {
    E(game)->get_global_state(buffer, half);
    return 0;
}
MG_API int magent_b200_snapshot_arenas(EnvHandle game) { return E(game)->snapshot_arenas(); }
MG_API int magent_b200_free_snapshot(EnvHandle game, int snapshot) { return E(game)->free_snapshot(snapshot); }
MG_API int magent_b200_restore_arenas(EnvHandle game, int snapshot, const int *src, int keep_rng) {
    return E(game)->restore_arenas(snapshot, src, keep_rng);
}
MG_API int magent_b200_replay_new(EnvHandle game, const int *arenas, int n_arenas, int max_frames) {
    return E(game)->replay_new(arenas, n_arenas, max_frames);
}
MG_API int magent_b200_replay_record(EnvHandle game, int replay) { return E(game)->replay_record(replay); }
MG_API int magent_b200_replay_write(EnvHandle game, int replay, const char *dir, long long *dropped) {
    return E(game)->replay_write(replay, dir, dropped);
}
MG_API int magent_b200_replay_free(EnvHandle game, int replay) { return E(game)->replay_free(replay); }
MG_API int magent_b200_get_arena_done(EnvHandle game, int *out) { return E(game)->get_arena_done(out); }
MG_API int magent_b200_get_counters(EnvHandle game, long long *out, int capacity) { return E(game)->get_counters(out, capacity); }
MG_API long long magent_b200_launch_count(void) { return mg::be::launch_count(); }
MG_API int magent_b200_set_profiling(EnvHandle game, int on) { E(game)->set_profiling(on != 0); return 0; }
MG_API int magent_b200_get_profile(EnvHandle game, double *ms, long long *n) { E(game)->get_profile(ms, n); return 0; }
MG_API int magent_b200_get_io_stats(EnvHandle game, long long *out, int capacity) { E(game)->get_io_stats(out, capacity); return capacity < 6 ? capacity : 6; }
MG_API int magent_b200_graph_begin(EnvHandle game) { E(game)->graph_begin(); return 0; }
MG_API int magent_b200_graph_end(EnvHandle game) { return E(game)->graph_end(); }
MG_API int magent_b200_graph_launch(EnvHandle game, int id, int times) { E(game)->graph_launch(id, times); return 0; }
MG_API void *magent_b200_stream(EnvHandle game) { return E(game)->stream(); }
MG_API int magent_b200_host_threads(void) { return mg::host_threads(); }
MG_API int magent_b200_set_host_threads(int n) { mg::set_host_threads(n); return 0; }
