// dev_types.h -- plain-old-data layout of the engine state in HBM, shared by host and device.
//
// Layout summary (DESIGN.md §3):
//   * `occ`   int32 [A][H*W]   one cell code per grid cell: OCC_EMPTY, OCC_WALL or an agent code
//             (group << 24 | index-in-group).  A w x l body writes its code into every cell it covers.
//             Replaces reference MapSlot{slot_type,occ_type,occupier*} + channel_ids
//             (src/gridworld/Map.h:23-29,72-73): channel and hp are derived from the code.
//   * per group, arena-major SoA arrays [A][cap] in *group vector order* (the reference keeps
//             std::vector<Agent*> per group, GridWorld.h:256-313; index == position in that vector),
//             ping-pong double buffered so `clear_dead` is a stable parallel compaction.
//   * per-agent step scratch [A][cap_total] addressed by flat = foff[group] + index.
//   * per-arena header (rng state, done flag, relaxation flags) and [G][A] count arrays.
#pragma once
#include <stdint.h>
#include "hd.h"

namespace mg {

enum { MG_MAX_GROUPS = 8, MG_MAX_RULES = 64, MG_MAX_PROG = 16, MG_MAX_RECV = 4, MG_MAX_IN = 4, MG_MAX_ALLQ = 16 };
enum { MG_N_COUNTERS = 8 };
enum Counter { CNT_AGENT_STEPS = 0, CNT_ATTACKS, CNT_HITS, CNT_KILLS, CNT_STARVED,
               CNT_MOVES_OK, CNT_MOVES_BLOCKED, CNT_STEPS };

enum : int { OCC_EMPTY = -1, OCC_WALL = -2, OCC_FOOD = -3 };   // OCC_FOOD: food_mode only (amount in EngineDev::food)
enum : int { TGT_NONE = -1, TGT_FOOD = -3 };                  // EngineDev::tgt of an attacker: none / an agent code (>= 0) / a food cell
enum : int { KIND_EMPTY = 0, KIND_WALL = 1, KIND_GROUP0 = 2, KIND_FOOD = 255 };   // EngineDev::kind
// An agent's kind byte is (KIND_GROUP0 + group) | KIND_FULL when its hp is exactly max_hp: its hp / max_hp is 1.0f by
// arithmetic, so neither the step has to write nor the render to read the hp_norm plane for it (most agents of a sparse
// battle).  KIND_FOOD has the bit set too: test for food first.
enum : int { KIND_FULL = 0x40, KIND_GROUP_MASK = 0x3f };
MG_HD unsigned char kind_agent(int g, bool full_hp) { return (unsigned char)((KIND_GROUP0 + g) | (full_hp ? KIND_FULL : 0)); }
MG_HD bool kind_is_agent(int t) { return t >= KIND_GROUP0 && t != KIND_FOOD; }
MG_HD int kind_group(int t) { return (t & KIND_GROUP_MASK) - KIND_GROUP0; }
enum : int { RANK_NONE = -1, DEATH_NEVER = 0x7fffffff, DEATH_BEFORE = -1 };
enum : unsigned { MVKEY_NONE = 0xffffffffu };

// agent flags
enum : unsigned char { FLAG_DEAD = 1, FLAG_ABSORBED = 2 };
// mover states
enum : unsigned char { MV_NONE = 0, MV_OOB = 1, MV_STATIC_FAIL = 2, MV_PENDING_FAIL = 3, MV_OK = 4, MV_ABSORBED = 5, MV_SKIPPED = 6 };

// EventOp numbering of the reference (src/gridworld/grid_def.h:17-23)
enum EventOp : unsigned char { OP_AND = 0, OP_OR, OP_NOT, OP_KILL, OP_AT, OP_IN, OP_COLLIDE, OP_ATTACK,
                               OP_DIE, OP_IN_A_LINE, OP_ALIGN, OP_NULL };

MG_HD int code_make(int g, int i) { return (g << 24) | i; }
MG_HD int code_group(int c) { return c >> 24; }
MG_HD int code_index(int c) { return c & 0xffffff; }

enum { DIR_EAST = 0, DIR_SOUTH = 1, DIR_WEST = 2, DIR_NORTH = 3 };     // reference Direction (grid_def.h:15)

struct AgentSoA {           // arena-major [A][cap]
    int *x, *y;             // top-left cell of the body (reference Agent::pos)
    float *hp;
    int *act;               // last_action (reference Agent::last_action)
    int *id;
    float *next_reward, *last_reward;
    int *op_obj;            // agent code of the object of last_op, or -1
    unsigned char *last_op; // EventOp
    unsigned char *flags;   // FLAG_DEAD | FLAG_ABSORBED
    unsigned char *dir;     // Direction; always NORTH(3) while turn_mode is unsupported
};

struct GroupDev {
    // ---- type constants (reference AgentType, src/gridworld/AgentType.h:17-48)
    int body_w, body_l;
    float max_hp, damage, step_recover, kill_supply;
    float eat_ability, food_supply;           // food_mode (Map.cc:276-303)
    float step_reward, kill_reward, dead_penalty, attack_penalty;
    int attack_in_group;
    int can_absorb;                           // AgentType::can_absorb (Map.cc:341-349)
    int view_w, view_h, view_x1, view_y1;     // view rectangle and its left-top offset from the eye
    int view_count;                           // in-range cells of the view mask
    int view_xoff, view_yoff;                 // eye offset from pos  (= width/2, length/2)
    int att_xoff, att_yoff;
    int n_move, attack_base, n_action, n_attack;
    int channel;                              // group2channel(g)  (GridWorld.cc:915-924)
    int feature_size;
    const int *move_dx, *move_dy;             // [n_move]    (Range::num2delta)
    const int *att_dx, *att_dy;               // [n_attack]
    const unsigned char *view_mask;           // [view_h*view_w] is_in_range
    // ---- state
    int cap;                                  // per-arena capacity of the SoA arrays
    int foff;                                 // flat scratch offset of this group inside an arena
    AgentSoA soa[2];                          // ping-pong; bit g of `curmask` selects the live one
    int *ev_rank;                             // [A][cap] execution rank of the agent's attack this step, -1 if none (render only)
};

struct ArenaHdr {
    uint32_t rng;            // minstd_rand0 state (reference GridWorld::random_engine)
    uint32_t rng_next;
    int done;
    int n_attack;
    int any_dead;            // some agent of this arena carries FLAG_DEAD (set where it dies, cleared by the cull)
    int changed[3];          // rotating "something changed" flags of the relaxation loops
    unsigned char rule_trig[MG_MAX_RULES];   // rule r triggered this step (RewardRule::trigger)
    float grp_reward[MG_MAX_GROUPS];
    // Agent::index of the reference is written by clear_dead only (GridWorld.cc:655) and is 0 from the
    // constructor (GridWorld.h:136): agents at positions >= n_cull[g] (added since the last clear_dead) have index 0
    int n_cull[MG_MAX_GROUPS];
    // group-quantified ('all' subject) event nodes, reduced once per step (phase_rule_allq): number of agents
    // violating the predicate, and min / max of the varying coordinate for in_a_line
    int allq_viol[MG_MAX_ALLQ], allq_min[MG_MAX_ALLQ], allq_max[MG_MAX_ALLQ];
    // next agent id of the arena (HostArena::id_counter): carried here so that a restored arena's add_agents continues
    // from the snapshot's counter.  Uploaded by to_device, read back by to_host; the step kernels never touch it.
    int id_counter;
};

// Entity roles inside a rule.  The reference binds the rule's input symbols depth-first in order
// (RewardEngine.cc:373-443); input k writes its subject symbol (role 2k) and then the symbol inferred from the
// subject's op_obj (role 2k+1).  A symbol's entity at the leaf is the LAST write to it, resolved at compile time.
enum { ROLE_GROUP = 254, ROLE_ALL = 255 };      // a whole group as receiver / an 'all' subject of an event node
enum { IN_ANY = 0, IN_ALL = 1, IN_FIXED = 2 };
enum { RULE_GENERAL = 0, RULE_ONE_ANY = 1, RULE_DEAD = 2 };
enum { MG_HOT_RULES = 16, MG_HOT_PROG = 4, MG_HOT_RECV = 2 };   // rules whose program also fits the per-CTA copy   // EngineDev::rule_shape  // AgentSymbol::index -1 / -2 / >= 0

struct RuleInstr {           // postfix program over the bound entities
    unsigned char op;        // EventOp
    unsigned char role_a;    // entity role of the first symbol (ROLE_ALL: quantified over `all_group`)
    unsigned char role_b;
    unsigned char allq;      // ROLE_ALL: slot of the per-step reduction in ArenaHdr::allq_*
    int i0, i1, i2, i3;      // OP_AT: x,y ; OP_IN: x1,y1,x2,y2
    int all_group;
};

struct RuleRecv { int role; int group; float value; };

struct RuleInput {           // one level of the reference's DFS (input_symbols[k], infer_obj[k])
    int kind;                // IN_ANY: loop over the group; IN_ALL: binds nothing itself; IN_FIXED: agent `index`
    int group, index;
    int has_obj, obj_group, obj_index;      // symbol bound from the subject's op_obj; obj_index -1 = any
};

struct RuleDev {
    int n_in; RuleInput in[MG_MAX_IN];
    int n_any; int any_in[MG_MAX_IN];       // the IN_ANY levels, outermost first
    int dead;                               // can never fire (fixed-index subject without an inferred object,
                                            // RewardEngine.cc:426-441 has no else branch)
    int n_prog; RuleInstr prog[MG_MAX_PROG];
    int n_recv; RuleRecv recv[MG_MAX_RECV];
    int is_terminal;
};

// the part of a rule every thread reads every step, kept in the per-CTA copy of EngineDev (shared memory)
struct RuleHot {
    unsigned char shape;     // RULE_*
    unsigned char terminal;
    unsigned char group;     // RULE_ONE_ANY: the subject's group ...
    unsigned char has_obj;   // ... and the symbol bound from its op_obj
    int obj_group, obj_index;
    int simple_op;           // RULE_ONE_ANY whose trigger is the single node op(subject, inferred object): the verdict is
                             // last_op == simple_op (op_obj equals the bound object by construction); 0 = evaluate the program
};
// trigger program and receivers of the first MG_HOT_RULES rules when they are small enough (every shipped game's are):
// a candidate that passes the bind evaluates and pays from shared memory instead of walking the HBM table
struct RuleSmall {
    int n_prog, n_recv;      // n_prog < 0: does not fit, use EngineDev::rules[r]
    RuleInstr prog[MG_HOT_PROG];
    RuleRecv recv[MG_HOT_RECV];
};

struct EngineDev {
    int A, W, H, G;
    int nsep, bandwidth, large_map;           // GridWorld.cc:75-85, :407
    int minimap_mode, embedding_size, n_channel, channel_base;
    int food_mode;                            // kills leave food on the attacked cell (Map.cc:276-283)
    float *food;                              // [A][H*W] amount of food on OCC_FOOD cells (food_mode only)
    int turn_mode;                            // agents carry a direction; [moves][turn L, R][attacks] (AgentType.cc:113-117)
    int cap_total, max_body;
    int any_absorb;                           // some group's type has can_absorb
    int scratch_stride;                       // per-arena stride of the step scratch: cap_total in HBM, 0 when it lives in the CTA's shared memory
    uint32_t pow2[32];                        // 16807^(2^b) mod (2^31-1)
    GroupDev grp[MG_MAX_GROUPS];
    ArenaHdr *hdr;                            // [A]
    int *n, *dead_ct;                         // [G][A]
    int *off;                                 // [G][A+1] prefix of n over arenas (ABI concatenation)
    int *done;                                // [A] done flag of the last step
    int *occ, *claim_head;                    // [A][H*W]
    // observation planes, padded by kpad cells on every side so that a view window never needs a bounds check:
    // cell (x, y) of arena a lives at a * kplane + (y + kpad) * kw + x + kpad
    unsigned char *kind;                      // [A][kplane] 0 empty / 1 wall / 2 + group; kept in step with occ; then a
                                              // window of (2 kpad + 1) * kw zero bytes: the blank arena A of vacant slots
                                              // (backend_cuda.cu launch_obs_slots), whose observer stands at (0, 0)
    float *hpn;                               // [A][kplane] hp / max_hp of the occupant where kind lacks KIND_FULL; kept in step with hp
    int kpad, kw;
    long kplane;
    // per-agent step scratch [A][cap_total]
    int *att_rank, *tgt, *in_head, *in_next, *death, *mv_nx, *mv_ny;
    unsigned *mv_key;
    float *hp_fin;
    unsigned char *mv_state;
    // shuffle scratch [A][cap_total]
    int *jv, *sh_head, *sh_next, *sh_first, *att_agent;
    int *cl_next;                             // [A][cap_total*max_body] claimant list links
    int n_rules; const RuleDev *rules;        // [n_rules] in HBM (read through L2; not part of the per-CTA smem copy)
    RuleSmall rule_small[MG_HOT_RULES];
    RuleHot rule_hot[MG_MAX_RULES];           // what phase_reward_rule / phase_done need without touching the table
    int n_allq;                               // group-quantified event nodes over all rules (ArenaHdr::allq_*)
    long long *counters;                      // [MG_N_COUNTERS]
    int *team_scratch;                        // [2 * max CTAs] partial sums of team scans
    int *mm_count;                            // [A][G][max_view_cells] minimap histogram scratch
    int *mm_total;                            // [A][G] agents counted into the minimap
};

// A device-resident copy of every arena's state (Engine::snapshot_arenas, DESIGN.md §3): the live arena-major layout of
// occ, kind, hp_norm and food, the headers and counts, and the live ping-pong SoA buffer of every group with the
// snapshot's own per-group capacity `cap`.  launch_restore copies arenas of it back over live arenas.
struct SnapDev {
    int *occ;                                 // [A][H*W]
    unsigned char *kind;                      // [A][kplane]
    float *hpn;                               // [A][kplane]
    float *food;                              // [A][H*W] (food_mode only, else nullptr)
    ArenaHdr *hdr;                            // [A]
    int *n, *dead_ct;                         // [G][A]
    int *done;                                // [A]
    int cap[MG_MAX_GROUPS];
    AgentSoA soa[MG_MAX_GROUPS];
};

struct StepArgs {
    unsigned curmask;
    int record_events;                        // fill GroupDev::ev_rank (attack events for env_render)
    int n_order;
    int order[MG_MAX_GROUPS];                 // groups that received set_action, in call order
};

struct ObsArgs {
    unsigned curmask;
    int group;
    void *view;                               // [sum_a n][view_h][view_w][n_channel]
    void *feature;                            // [sum_a n][feature_size]
    int half;                                 // 0: float32 (reference ABI), 1: IEEE half (compact hand-off)
    // render launch shape forced by the engine's "obs_grid" / "obs_chunk" / "obs_tile" keys (0: automatic); the backend
    // clamps grid to [1, tiles] and chunk to [1, ceil(tiles / grid)]; tile 1 = narrow, 2 = wide (narrow when it does not fit)
    int grid = 0, chunk = 0, tile = 0;
};

// One entry of a group's view LUT in the key order of magent_b200_get_neighbours (nbr_phases.h nbr_cell_key).
// Engine::to_device builds it on the host, one run of view_count entries per heading in turn_mode, and keeps it outside
// EngineDev: {offset of the map cell in the padded planes from the observer's own cell, dx | dy << 16, key, vx | vy << 16}.
struct alignas(16) NbrCell {
    int off, delta, key, cell;
};

// Stable agent slots (magent_b200_get_slots, slot_phases.h).  The table has one row of SLOT_HDR + id_cap ints per arena:
// words [0, MG_MAX_GROUPS) are the arena's slot counters (agents of each group placed since its last reset), word
// SLOT_HDR + id the slot of the agent with that id.  Ids are unique per arena and restart at 0 with env_reset, so a
// restore copies a row prefix and nothing else changes it between host-side placements.  It lives outside EngineDev and
// outside ArenaHdr, so no step, cull or render kernel sees it; this block is allocated once per engine and names the
// current table, which grows with the largest id counter while a captured graph keeps pointing at the block.
enum { SLOT_HDR = MG_MAX_GROUPS };
struct SlotDev {
    int *tab;                                 // [A][SLOT_HDR + id_cap]
    int id_cap;
};

// The replay recorder (magent_b200_replay_*, replay_phases.h).
// per-arena replay state, [A] in device memory outside EngineDev and ArenaHdr (a restore copies the header from the
// snapshot): the episode counter (env_reset and every restore that replaces the arena bump it) and, per group, the rows
// of the event list the arena's last step wrote (a restore empties it)
struct RepArena {
    int episode;
    int ev_n[MG_MAX_GROUPS];
};

// one attack row of the event list: rank < 0 where the row's agent executed no attack
struct RepEvent { int rank, id, x, y; };
// one agent row of a frame; dir_flags = dir | FLAG_ABSORBED << 8 when absorbed (dir is DIR_NORTH without turn_mode)
struct RepAgent { int id, x, y; float hp; int dir_flags; };

enum { REP_H_EPISODE = 0, REP_H_WALLS = 1, REP_H_N = 2, REP_H_EV_N = 2 + MG_MAX_GROUPS, REP_HDR_INTS = 32 };

// ints of one frame block: header, cap_total agents, cap_total events, wall bitmap
struct RepLayout {
    int cap_total;
    int wall_words;                          // ceil(W * H / 128) * 4: every frame block stays 16-byte aligned
    MG_HD long agent_base() const { return REP_HDR_INTS; }
    MG_HD long event_base() const { return agent_base() + (long)cap_total * (sizeof(RepAgent) / 4); }
    MG_HD long wall_base() const { return event_base() + (long)cap_total * (sizeof(RepEvent) / 4); }
    MG_HD long frame_ints() const { return wall_base() + wall_words; }
};

// the recorder's device control block: frames buffered, frames dropped for want of room, and the CTA ticket of the
// record kernel (the last CTA to finish advances the counters)
struct RepCtl {
    unsigned long long dropped;
    int n_frames;
    unsigned ticket;
};

enum InfoKind { INFO_ID = 0, INFO_POS, INFO_ALIVE, INFO_REWARD, INFO_ACTION_SCATTER, INFO_HP };

}  // namespace mg
