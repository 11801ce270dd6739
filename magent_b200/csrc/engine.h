// engine.h -- host side of the B200 grid-world engine (plain C++, no CUDA headers).
//
// Mirrors the reference GridWorld class surface (src/gridworld/GridWorld.h:38-128) behind the C ABI in
// shim.cc.  Setup-time work (agent types and range tables, reward-rule compilation, episode placement
// with the engine RNG) runs on the host against a host image of the arenas; the first hot-path call
// uploads the image to HBM and from then on every step-loop call is a kernel launch (backend.h).
#pragma once
#include <stdint.h>
#include <iosfwd>
#include <map>
#include <string>
#include <vector>
#include "dev_types.h"

namespace mg {
namespace be { struct Ctx; }

[[noreturn]] void fatal(const char *fmt, ...);

// Range tables (reference src/gridworld/Range.h:104-190)
struct RangeTab {
    int width = 0, height = 0, count = 0;
    int x1 = 0, y1 = 0, x2 = 0, y2 = 0;
    std::vector<unsigned char> mask;    // is_in_range, row-major [height][width]
    std::vector<int> dx, dy;            // num2delta
};
RangeTab make_circle_range(float radius, float inner_radius, int parity);
RangeTab make_sector_range(float angle, float radius, int parity);

// reference src/gridworld/AgentType.h:17-48
struct AgentTypeDef {
    std::string name;
    int width = 1, length = 1;
    float speed = 1.0f, hp = 1.0f;
    float view_radius = 1, view_angle = 360, attack_radius = 0, attack_angle = 0;
    float hear_radius = 0, speak_radius = 0;
    int speak_ability = 0;
    float damage = 0, trace = 0, eat_ability = 0, step_recover = 0, kill_supply = 0, food_supply = 0;
    bool attack_in_group = false, can_absorb = false;
    float step_reward = 0, kill_reward = 0, dead_penalty = 0, attack_penalty = 0;
    int view_x_offset = 0, view_y_offset = 0, att_x_offset = 0, att_y_offset = 0;
    RangeTab view, attack, move;
    int move_base = 0, turn_base = 0, attack_base = 0, n_action = 0;
};

struct HostGroup {                      // one group of one arena, in vector order
    std::vector<int> x, y, id, act, op_obj;
    std::vector<float> hp, next_reward, last_reward;
    std::vector<unsigned char> last_op, flags, dir;
    int dead_ct = 0;
    int n_cull = 0;                     // size after the last clear_dead (reference Agent::index is refreshed only there)
    float grp_reward = 0.0f;
    int size() const { return (int)x.size(); }
    void clear();
    void resize(int n);
};

struct HostArena {
    std::vector<int> occ;
    std::vector<float> food;            // food_mode: amount per OCC_FOOD cell
    std::vector<HostGroup> groups;
    uint32_t rng = 1;
    int id_counter = 0;
    int done = 0;
    // stable slots (slot_phases.h): slot_of_id[id] for every id handed out since the last reset (size id_counter), and
    // per group the slots handed out
    std::vector<int> slot_of_id;
    int slot_ct[MG_MAX_GROUPS] = {0};
};

// a copy of every arena's state in HBM (Engine::snapshot_arenas): its own allocations, outside dev_allocs_, so that
// neither free_device nor a capacity-growing re-upload frees it
struct ArenaSnapshot {
    bool live = false;
    bool in_graph = false;              // recorded into a CUDA graph: lives as long as the engine
    // the geometry it was taken under; a restore needs the same
    int W = 0, H = 0, kpad = 0;
    bool food_mode = false, turn_mode = false;
    std::vector<const AgentTypeDef *> types;
    std::vector<int> n;                 // [G][A] agents per group and arena
    std::vector<int> max_n;             // [G] largest per-arena count
    SnapDev dev;
    // the slot table at the time ([A][SLOT_HDR + slot_id_cap], in allocs) and what a restore from it can bring in: the
    // largest id counter and per group the largest slot count of its arenas
    int *slot_tab = nullptr;
    int slot_id_cap = 0, max_ids = 0;
    std::vector<int> slot_max;
    std::vector<void *> allocs;
};

// a replay recorder (Engine::replay_new): frames of chosen arenas buffered in its own device memory, written out in the
// reference viewer's format by Engine::replay_write
struct ReplayRec {
    bool live = false;
    bool in_graph = false;              // recorded into a CUDA graph: lives as long as the engine
    std::vector<int> arenas;
    int max_frames = 0;
    std::vector<int> cap;               // [G] per-arena capacity the frames are sized for
    RepLayout L = {0, 0};
    int W = 0, H = 0;
    int *d_arenas = nullptr, *frames = nullptr, *last_ep = nullptr;
    RepCtl *ctl = nullptr;
    // writer state per recorded arena: the open file (0: none yet), frames in it, the walls of its episode
    std::vector<int> file_ct, frame_ct;
    std::vector<std::vector<int>> walls;
};

struct SymbolDef { int group = 0, index = 0; };
struct NodeDef { int op = OP_NULL; std::vector<int> raw; };
struct RuleDef { int on = 0; std::vector<int> recv; std::vector<float> values; bool is_terminal = false, auto_value = false; };

class Engine {
public:
    Engine();
    ~Engine();

    // ---- reference Environment / GridWorld surface
    int set_config(const char *key, void *p_value);     // -1: refused (extension keys; last_error says why)
    void register_agent_type(const char *name, int n, const char **keys, float *values);
    void new_group(const char *type_name, int *handle);
    void define_agent_symbol(int no, int group, int index);
    void define_event_node(int no, int op, int *inputs, int n_inputs);
    void add_reward_rule(int on, int *receivers, float *values, int n_receiver, bool is_terminal, bool auto_value);

    void reset();
    void add_agents(int group, int n, const char *method, const int *pos_x, const int *pos_y, const int *dir);
    void get_observation(int group, void **bufs, int half = 0);     // half: compact f16 hand-off (extension)
    void set_action(int group, const int *actions);
    void step(int *done);
    void get_reward(int group, float *buf);
    void clear_dead();
    int get_info(int group, const char *name, void *buf);   // -1: refused (extension keys)
    void set_goal(int group, const char *method, const int *buf);
    void render();

    void render_next_file();

    // ---- extensions
    void select_arena(int a) { sel_arena_ = a; }
    void random_actions(int group, unsigned long long seed);
    // whole-map state of every arena, [A][H][W][state_channels()] (obs_phases.h state_compose_cell); half: IEEE binary16
    void get_global_state(void *buf, int half);
    // reset pool: snapshot every arena on the device, later restore any subset of arenas from it.  These return -1 and
    // set the last error when they refuse (the state is then unchanged).
    int snapshot_arenas();
    int free_snapshot(int id);
    int restore_arenas(int id, const int *src, int keep_rng);
    int get_arena_done(int *out);
    // legal actions (mask_phases.h): uint8 [n][n_action] of one group / actions drawn uniformly from them on the device.
    // -1 and the last error when refused.
    int get_action_mask(int group, unsigned char *buf);
    int random_legal_actions(int group, unsigned long long seed);
    // mean neighbour action (nbr_phases.h): float [n][n_action(of)] and int [n] (count may be null) of one group.
    // -1 and the last error when refused.
    int get_mean_action(int group, int of, float *mean, int *count);
    // the first k neighbours of group `of`, nearest first (nbr_phases.h nbr_cell_key): int [n][k] rows of `of`, int
    // [n][k][2] view cells and int [n] neighbour counts (rel and count may be null).  -1 and the last error when refused.
    int get_neighbours(int group, int of, int k, int *idx, int *rel, int *count);
    // stable slots (slot_phases.h): int [num_bound] row -> a * S + slot and int [A][S] slot -> row of one group, S =
    // slot_space(group); either may be null, not both.  -1 and the last error when refused.
    int get_slots(int group, int *row_slot, int *slot_row);
    // the observation of one group in slot order: bufs[0] view [A][S][view_h][view_w][n_channel], bufs[1] feature
    // [A][S][feature_size], the records get_observation writes for the row in each slot, all zeros in vacant slots;
    // half: IEEE binary16.  -1 and the last error when refused.
    int get_observation_slots(int group, void **bufs, int half);
    // the slot-ordered step loop (S = slot_space(group), [A][S] buffers; neither waits for the counts).  set_action_slots:
    // set_action with act[slot] for every row, registered in the step's action order like set_action (act may be null
    // when S == 0).  get_reward_slots: float reward and uint8 status (0 vacant, 1 alive, 2 dead, not culled yet) per
    // slot, either may be null, not both.  get_action_mask_slots: uint8 [A][S][n_action], get_action_mask's row for the
    // row in each slot, zero in vacant slots.  -1 and the last error when refused.
    int set_action_slots(int group, const int *act);
    int get_reward_slots(int group, float *reward, unsigned char *status);
    int get_action_mask_slots(int group, unsigned char *mask);
    // the mean action and the neighbours in slot order (S = slot_space(group), neither waits for the counts):
    // get_mean_action's and get_neighbours's rows for the row in each slot, [A][S][...], with every used idx entry the
    // neighbour's a * slot_space(of) + slot instead of its row; zero / -1 rows and count 0 in vacant slots.  -1 and the
    // last error when refused.
    int get_mean_action_slots(int group, int of, float *mean, int *count);
    int get_neighbours_slots(int group, int of, int k, int *idx, int *rel, int *count);
    // the built-in scripted opponent (rule_phases.h) of one group against group `target`: set as the group's actions
    // (rule_actions), int [n] in row order (get_rule_actions) or int [A][S] in slot order (get_rule_actions_slots).  -1
    // and the last error when refused.
    int rule_actions(int group, int target, int policy, unsigned long long seed);
    int get_rule_actions(int group, int target, int policy, unsigned long long seed, int *act);
    int get_rule_actions_slots(int group, int target, int policy, unsigned long long seed, int *act);
    // replay recorder (replay_phases.h): record frames of chosen arenas on the device, write them as env_render would.
    // -1 and the last error when refused.
    int replay_new(const int *arenas, int n_arenas, int max_frames);
    int replay_record(int id);
    int replay_write(int id, const char *dir, long long *dropped);
    int replay_free(int id);
    int get_counters(long long *out, int cap);
    void sync();
    void get_io_stats(long long *out, int cap);      // bytes so far: device->host over PCIe, host->device, written by host threads
    // CUDA graphs for launch-bound workloads: the device-pointer calls between begin and end become one graph
    void graph_begin();
    int graph_end();
    void graph_launch(int id, int times);
    void *stream();                      // cudaStream_t of this engine's kernels (nullptr before the first device call)
    void set_profiling(bool on);
    void get_profile(double *ms, long long *n);

private:
    // configuration
    int W_ = 0, H_ = 0;
    bool food_mode_ = false, turn_mode_ = false, minimap_mode_ = false, goal_mode_ = false;
    int embedding_size_ = 0;
    int A_ = 1;
    int device_id_ = -1;
    be::Ctx *bx_ = nullptr;             // this engine's device context (device, streams, scratch): backend.h
    std::map<std::string, AgentTypeDef> types_;
    std::vector<const AgentTypeDef *> group_type_;
    std::vector<SymbolDef> symbols_;
    std::vector<NodeDef> nodes_;
    std::vector<RuleDef> rules_;
    std::vector<RuleDev> compiled_rules_;
    int n_allq_ = 0;
    bool may_have_dead_ = true;         // some arena reported dead agents since the last clear_dead (bit 1 of EngineDev::done)
    bool rules_compiled_ = false;
    bool was_reset_ = false;
    int nsep_ = 1;
    bool large_map_ = false;
    int sel_arena_ = -1;

    // replay dump (reference RenderGenerator, src/gridworld/RenderGenerator.cc)
    std::string render_dir_;
    int file_ct_ = 0, frame_ct_ = 0, frame_per_file_ = 10000;
    bool first_render_ = true;
    struct AttackEvent { int id, x, y; };
    std::vector<AttackEvent> attack_events_;
    void collect_attack_events();
    // the one formatter of env_render and replay_write: config.json, and one frame (walls: the wall cells when the frame
    // opens a file, else null; agents: every row of each group, in row order)
    void write_render_config(std::ostream &os) const;
    void write_render_frame(std::ostream &os, const std::vector<int> *walls,
                            const std::vector<std::vector<RepAgent>> &agents,
                            const std::vector<AttackEvent> &events) const;
    // replay recorders: the per-arena episode counters and event-list counts ([A], outside EngineDev and ArenaHdr, kept
    // across re-allocations), the event list ([A][ev_stride_] RepEvent, sized for cap_total at the last replay_new), the
    // arenas whose events the step collects ([A], the union of the live recorders', n_ev_arenas_ of them), and whether
    // this game has ever captured a CUDA graph (steps captured without a live recorder cannot record events)
    std::vector<ReplayRec> replays_;
    RepArena *d_rep_ = nullptr;
    RepEvent *d_ev_ = nullptr;
    int ev_stride_ = 0;
    int *d_ev_arenas_ = nullptr;
    int n_ev_arenas_ = 0;
    bool graph_captured_ = false;
    int live_replays() const;
    void update_ev_arenas();

    // host image
    std::vector<HostArena> arenas_;
    enum Where { HOST, DEVICE } where_ = HOST;
    std::vector<int> h_off_;            // [G][A+1] prefix counts (valid in both states)

    // device image
    EngineDev hE_;                      // host copy of the device block (device pointers inside)
    EngineDev *dE_ = nullptr;
    std::vector<void *> dev_allocs_;
    std::vector<int> cap_;              // per group capacity on the device
    unsigned curmask_ = 0;
    std::vector<int> order_;            // groups with set_action this step, in call order
    void *d_view_stage_ = nullptr, *d_feat_stage_ = nullptr;
    float *d_mm_val_ = nullptr;
    // the view LUTs of get_neighbours in key order, every group's and heading's runs in one device buffer (outside
    // EngineDev, which seven kernels copy into shared memory): group g's start at nbr_lut_base_[g]; nbr_lut_ is the host
    // copy last uploaded; nbr_key_fits_[g] == 0 when g's keys would not fit an int (the call is then refused)
    NbrCell *d_nbr_lut_ = nullptr;
    std::vector<NbrCell> nbr_lut_;
    std::vector<size_t> nbr_lut_base_;
    std::vector<unsigned char> nbr_key_fits_;
    void upload_nbr_luts(bool force);
    bool rule_refused(int group, int target, int policy, bool slots, const char *what);
    // stable slots: the live table ([A][SLOT_HDR + slot_id_cap_], grow-only, outside dev_allocs_ so that a re-allocation
    // of the device image does not drop it), the SlotDev block naming it (allocated once, so captured graphs stay valid
    // when the table grows), and slot_space_[g] = S(g) as the last reset, add_agents, snapshot_arenas or free_snapshot
    // left it
    int *d_slot_tab_ = nullptr;
    int slot_id_cap_ = 0;
    SlotDev *d_slot_dev_ = nullptr;
    std::vector<int> slot_space_;
    void upload_slots();
    void update_slot_space();
    int slot_space(int group) const { return group < (int)slot_space_.size() ? slot_space_[group] : 0; }
    size_t view_stage_bytes_ = 0, feat_stage_bytes_ = 0;
    void *d_io_stage_ = nullptr; size_t io_stage_bytes_ = 0;
    void *h_feat_stage_ = nullptr; size_t h_feat_stage_bytes_ = 0;      // page-locked staging of the feature rows (host path)
    enum { IO_D2H = 0, IO_H2D = 1, IO_HOST_WRITTEN = 2, IO_US_WIRE = 3, IO_US_EXPAND = 4, IO_US_FEATURE = 5, IO_N = 6 };
    long long io_[IO_N] = {0, 0, 0, 0, 0, 0};       // step-loop traffic (hot calls only) and host-path phase times
    bool done_stale_ = false;           // arenas_[a].done not refreshed by the last step (device-pointer done)
    int host_path_ = -1;                // env_get_observation into host memory: 1 wire records + host expansion, 0 dense DMA
    int obs_grid_ = 0, obs_chunk_ = 0, obs_tile_ = 0;   // forced render launch shape (ObsArgs; 0: automatic)
    unsigned long long rand_calls_ = 0;
    // get_observation pre-pass products (hp_norm plane, minimap) stay valid until the state changes
    unsigned long long state_version_ = 1, prep_version_ = 0;
    int prep_vw_ = 0, prep_vh_ = 0;
    bool prep_skip_absorbed_ = false;

    int G() const { return (int)group_type_.size(); }
    int group2channel(int g) const;
    int n_channel() const { return group2channel(G()); }
    int state_channels() const { return 1 + (food_mode_ ? 1 : 0) + 2 * G(); }     // = mg::state_channels(hE_)
    int feature_size(int g) const;
    int total(int g) const { return h_off_[(size_t)g * (A_ + 1) + A_]; }
    int count(int g, int a) const { return h_off_[(size_t)g * (A_ + 1) + a + 1] - h_off_[(size_t)g * (A_ + 1) + a]; }
    void refresh_host_counts();
    bool counts_unknown_ = false;       // steps ran inside replayed graphs: the device's offset table is ahead of h_off_
    unsigned capture_mask_ = 0; int capture_culls_ = 0;
    bool counts_pending_ = false;       // clear_dead queued a fetch of the new counts; h_off_ still holds the old (upper-bound) ones
    void settle_counts();
    void check_group(int g, const char *where) const;
    // snapshots (reset pool)
    std::vector<ArenaSnapshot> snaps_;
    bool snap_matches(const ArenaSnapshot &s, int kpad) const;
    int view_pad() const;               // kpad of the padded observation planes for the current agent types
    std::vector<int> restore_floor() const;          // [G] largest count any usable snapshot can restore an arena to
    void set_counts(const std::vector<int> &c);           // h_off_ from per-arena counts c[G][A]
    void raise_counts(const std::vector<int> &floor);     // h_off_ counts to at least floor[g] in every arena
    int num_bound(int g) const;         // the "num_bound" info key: rows a device-pointer call may write before the counts settle
    bool capture_floor_ = false;        // the capture in progress sizes its launches for restores (graph_begin)

    void ensure_backend();
    void compile_rules();
    void to_device();
    void to_host(bool keep_device_authoritative);
    void free_device();
    void *dalloc(size_t bytes);
    void *io_stage(size_t bytes);
    // the per-agent read-backs (engine.cc read_back): one caller buffer (nullptr: not wanted) and its size in bytes
    struct OutPart { void *buf; size_t bytes; };
    template <size_t N, class F> void read_back(bool dev, const OutPart (&parts)[N], F &&launch);
    void stage_reserve(void *&p, size_t &have, size_t need);
    void prepare_obs(int group);        // the observation pre-pass for group's observers, unless still valid
    void get_observation_wire(int group, void **bufs);
    int max_agents_per_arena() const;

    // host-side placement (reference Map.cc:49-115, GridWorld.cc:180-290)
    bool host_is_blank(const HostArena &ar, int x, int y, int w, int h) const;
    int host_add_agent(HostArena &ar, int g, int x, int y, int dir);
    int host_add_wall(HostArena &ar, int x, int y);
    void host_random_blank(HostArena &ar, int w, int h, int &x, int &y);
};

}  // namespace mg
