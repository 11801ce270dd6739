// engine.cc -- host side of the B200 grid-world engine.  See engine.h.
#include "engine.h"
#include "step_phases.h"
#include "nbr_phases.h"
#include "rule_phases.h"
#include "slot_phases.h"
#include "replay_phases.h"

#include <errno.h>
#include <math.h>
#include <sys/stat.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <fstream>
#include <initializer_list>
#include <set>
#include <sstream>

#include "backend.h"
#include "host_expand.h"

namespace mg {

static std::string g_last_error;
const char *last_error() { return g_last_error.c_str(); }
void set_last_error(const std::string &s) { g_last_error = s; }

// The reference signals fatal conditions with LOG(FATAL), which throws from a destructor and ends in
// std::terminate (src/utility/utility.h:77-80,103).  Same observable behaviour: message, then abort.
void fatal(const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    fprintf(stderr, "[magent_b200 FATAL] %s\n", buf);
    fflush(stderr);
    abort();
}

static bool strequ(const char *a, const char *b) { return strcmp(a, b) == 0; }

// a refused extension call: the message goes to magent_b200_last_error, the call returns -1 and changes nothing
static int refuse(const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return -1;
}

// whether the kernel of a mask or mean-action call fits the device's shared memory (be::smem_fits); the refusal names
// the call, the group's view or action space and the bytes.  Asked after to_device, before anything is staged or written.
static bool smem_refused(be::Ctx *bx, const EngineDev &hE, int which, int group, int of, const char *call) {
    std::string why;
    if (!be::smem_fits || be::smem_fits(bx, hE, which, group, of, &why)) return false;
    if (which == be::SMEM_ACTION_MASK || which == be::SMEM_ACTION_MASK_SLOTS)
        refuse("%s: the %d actions of group %d need %s", call, hE.grp[group].n_action, group, why.c_str());
    else
        refuse("%s: a view of %d cells of group %d and the %d actions of group %d need %s", call, hE.grp[group].view_count,
               group, hE.grp[of].n_action, of, why.c_str());
    return true;
}

// ---------------------------------------------------------------------------------------------
// ranges  (reference src/gridworld/Range.h:149-190; same double-precision arithmetic)
RangeTab make_circle_range(float radius, float inner_radius, int parity) {
    const double eps = 1e-8;
    RangeTab r;
    r.width = 2 * int(radius + eps) + parity;
    int center = (int)(radius);
    if (r.width % 2 != parity) r.width++;
    r.height = r.width;
    r.mask.assign((size_t)r.width * r.width, 0);
    double delta = (parity == 0 ? 0.5 : 0);
    for (int i = 0; i < r.width; i++) {
        for (int j = 0; j < r.width; j++) {
            double dis_x = fabs(j - center + delta);
            double dis_y = fabs(i - center + delta);
            double dis = sqrt(dis_x * dis_x + dis_y * dis_y);
            if (dis < radius + eps && dis > inner_radius - eps) {
                r.mask[(size_t)i * r.width + j] = 1;
                r.dx.push_back(j - center);
                r.dy.push_back(i - center);
                r.count++;
            }
        }
    }
    r.x1 = r.y1 = -center;
    r.x2 = r.y2 = r.width - center - 1;
    return r;
}

// Sector of `angle` degrees opening towards -y (NORTH), stored as a height x width rectangle above the anchor
// (reference src/gridworld/Range.h:104-144; used when view_angle / attack_angle < 180)
RangeTab make_sector_range(float angle, float radius, int parity) {
    static const double kPi = 3.1415926536;           // the reference's constant, not M_PI (Range.h:16)
    const double eps = 0.00001;
    RangeTab r;
    r.height = (int)(radius + 0.5);
    r.width = (int)(2 * radius * sin(angle / 2 * (kPi / 180)) + 0.5);
    if (r.width % 2 != parity) r.width--;             // "fit to parity"
    if (r.width < 0) r.width = 0;
    r.mask.assign((size_t)r.width * r.height, 0);
    const double lim = tan(angle / 2 * kPi / 180) + eps;
    for (int i = 0; i < r.height; i++)
        for (int j = 0; j < r.width; j++) {
            const double dis_x = fabs(j - (r.width - 1) / 2.0), dis_y = fabs((double)(r.height - i));
            const double dis = sqrt(dis_x * dis_x + dis_y * dis_y);
            if (dis < radius + 0.2 + eps && dis_x / dis_y < lim) {
                r.mask[(size_t)i * r.width + j] = 1;
                r.dx.push_back(j - r.width / 2);
                r.dy.push_back(i - r.height);
                r.count++;
            }
        }
    r.x1 = -(r.width / 2); r.y1 = -r.height;
    r.x2 = (r.width - 1) / 2; r.y2 = -1;
    return r;
}

// Group::clear (GridWorld.h:277-280) empties the agent list and dead_ct but leaves the group's next_reward alone: a
// group reward that was not collected by clear_dead survives a reset (found by the chaotic-caller fuzz).
void HostGroup::clear() { resize(0); dead_ct = 0; n_cull = 0; }
void HostGroup::resize(int n) {
    x.resize(n); y.resize(n); id.resize(n); act.resize(n); op_obj.resize(n);
    hp.resize(n); next_reward.resize(n); last_reward.resize(n);
    last_op.resize(n); flags.resize(n); dir.resize(n);
}

// ---------------------------------------------------------------------------------------------
Engine::Engine() {
    memset(&hE_, 0, sizeof hE_);
    arenas_.resize(1);
    arenas_[0].rng = minstd_seed(0);                  // GridWorld.cc:29
}

Engine::~Engine() {
    for (ArenaSnapshot &sn : snaps_)
        for (void *p : sn.allocs) be::dfree(bx_, p);
    free_device();
    if (d_slot_tab_) be::dfree(bx_, d_slot_tab_);
    if (d_slot_dev_) be::dfree(bx_, d_slot_dev_);
    for (int id = 0; id < (int)replays_.size(); ++id)
        if (replays_[id].live) { replays_[id].in_graph = false; replay_free(id); }
    for (void *p : {(void *)d_rep_, (void *)d_ev_, (void *)d_ev_arenas_}) if (p) be::dfree(bx_, p);
    if (h_feat_stage_) be::host_free(h_feat_stage_);
    if (bx_) be::destroy(bx_);
}

void Engine::check_group(int g, const char *where) const {
    if (g < 0 || g >= G()) fatal("invalid group handle %d in %s", g, where);
}

int Engine::group2channel(int g) const {             // GridWorld.cc:915-924
    int base = 1, scale = 2;
    if (food_mode_) base++;
    if (minimap_mode_) scale++;
    return base + g * scale;
}

int Engine::feature_size(int g) const {              // GridWorld.cc:926-934
    int f = embedding_size_ + group_type_[g]->n_action + 1;
    if (goal_mode_) f += 2;
    if (minimap_mode_) f += 2;
    return f;
}

int Engine::set_config(const char *key, void *p_value) {      // GridWorld.cc:120-149
    int ivalue = *(int *)p_value;
    bool bvalue = *(bool *)p_value;
    if (strequ(key, "map_width")) W_ = ivalue;
    else if (strequ(key, "map_height")) H_ = ivalue;
    else if (strequ(key, "food_mode")) {
        food_mode_ = bvalue;
    } else if (strequ(key, "turn_mode")) {
        turn_mode_ = bvalue;
    } else if (strequ(key, "minimap_mode")) minimap_mode_ = bvalue;
    else if (strequ(key, "goal_mode")) goal_mode_ = bvalue;
    else if (strequ(key, "embedding_size")) embedding_size_ = ivalue;
    else if (strequ(key, "render_dir")) render_dir_ = (const char *)p_value;      // RenderGenerator::set_render("save_dir")
    else if (strequ(key, "seed")) {
        if (where_ == DEVICE) to_host(false);
        for (int a = 0; a < A_; ++a)
            if (sel_arena_ < 0 || sel_arena_ == a)
                arenas_[a].rng = minstd_seed((long long)ivalue + (sel_arena_ < 0 ? a : 0));
    }
    // ---- extension keys (unknown keys are FATAL in the reference, so these cannot collide)
    else if (strequ(key, "num_arenas")) {
        if (was_reset_) fatal("num_arenas must be configured before the first reset");
        if (ivalue < 1) fatal("num_arenas must be >= 1");
        A_ = ivalue;
        uint32_t seed0 = arenas_[0].rng;
        arenas_.assign(A_, HostArena());
        for (int a = 0; a < A_; ++a) arenas_[a].rng = a == 0 ? seed0 : minstd_seed(a);
    } else if (strequ(key, "device_id")) device_id_ = ivalue;
    else if (strequ(key, "host_path")) host_path_ = ivalue;               // 1 wire records + host expansion (default for large
                                                                           // observations), 0 dense DMA, 2 wire whatever the size
    // render launch shape of this engine's observations (0: automatic): CTAs, consecutive tiles per CTA visit, tile
    // width 1 narrow / 2 wide.  Tests use them to make every CTA render many tiles at small sizes.
    else if (strequ(key, "obs_grid") || strequ(key, "obs_chunk") || strequ(key, "obs_tile")) {
        const bool tile = strequ(key, "obs_tile");
        if (ivalue < 0 || (tile && ivalue > 2)) return refuse("%s = %d: must be %s", key, ivalue, tile ? "0, 1 or 2" : ">= 0");
        (strequ(key, "obs_grid") ? obs_grid_ : tile ? obs_tile_ : obs_chunk_) = ivalue;
    }
    else fatal("invalid argument in GridWorld::set_config : %s", key);
    return 0;
}

void Engine::register_agent_type(const char *name, int n, const char **keys, float *values) {
    std::string str(name);
    if (types_.count(str)) fatal("duplicated name of agent type in GridWorld::register_agent_type : %s", name);
    AgentTypeDef t;
    t.name = str;
    for (int i = 0; i < n; i++) {                     // AgentType.cc:52-83
        const char *k = keys[i];
        float v = values[i];
#define MG_SET_INT(f) if (strequ(k, #f)) { t.f = (int)(v + 0.5); continue; }
#define MG_SET_FLT(f) if (strequ(k, #f)) { t.f = v; continue; }
#define MG_SET_BOOL(f) if (strequ(k, #f)) { t.f = bool(int(v + 0.5)); continue; }
        MG_SET_INT(width) MG_SET_INT(length)
        MG_SET_FLT(speed) MG_SET_FLT(hp)
        MG_SET_FLT(view_radius) MG_SET_FLT(view_angle) MG_SET_FLT(attack_radius) MG_SET_FLT(attack_angle)
        MG_SET_FLT(hear_radius) MG_SET_FLT(speak_radius) MG_SET_INT(speak_ability)
        MG_SET_FLT(damage) MG_SET_FLT(trace) MG_SET_FLT(eat_ability)
        MG_SET_FLT(step_recover) MG_SET_FLT(kill_supply) MG_SET_FLT(food_supply)
        MG_SET_BOOL(attack_in_group) MG_SET_BOOL(can_absorb)
        MG_SET_FLT(step_reward) MG_SET_FLT(kill_reward) MG_SET_FLT(dead_penalty) MG_SET_FLT(attack_penalty)
#undef MG_SET_INT
#undef MG_SET_FLT
#undef MG_SET_BOOL
        // accepted but overwritten by the reference too (AgentType.cc:106-108)
        if (strequ(k, "view_x_offset") || strequ(k, "view_y_offset") || strequ(k, "att_x_offset") ||
            strequ(k, "att_y_offset") || strequ(k, "turn_x_offset") || strequ(k, "turn_y_offset")) continue;
        fatal("invalid agent config in AgentType::AgentType : %s", k);
    }
    if (t.width < 1 || t.length < 1 || t.width * t.length > 16) fatal("unsupported body size %dx%d", t.width, t.length);

    int parity = t.width % 2;                         // AgentType.cc:86-105
    if (t.view_angle >= 180) {
        if (fabs(t.view_angle - 360) > 1e-5) fatal("only supports ranges with angle = 360, when angle > 180.");
        t.view = make_circle_range(t.view_radius, 0, parity);
    } else {
        t.view = make_sector_range(t.view_angle, t.view_radius, parity);
        if (t.view.width < 1 || t.view.height < 1) fatal("empty view range (view_radius %g, view_angle %g)", t.view_radius, t.view_angle);
    }
    if (t.attack_angle >= 180) {
        if (fabs(t.attack_angle - 360) > 1e-5) fatal("only supports ranges with angle = 360, when angle > 180.");
        t.attack = make_circle_range(t.attack_radius, t.width / 2.0f, parity);
    } else {
        // the reference default (attack_angle = 0, radius 0) builds an empty SectorRange: no attack actions
        t.attack = make_sector_range(t.attack_angle, t.attack_radius, parity);
    }
    t.move = make_circle_range(t.speed, 0, 1);
    t.view_x_offset = t.width / 2; t.view_y_offset = t.length / 2;       // AgentType.cc:106-108
    t.att_x_offset = t.width / 2;  t.att_y_offset = t.length / 2;
    t.move_base = 0;
    t.turn_base = t.move.count;
    t.attack_base = t.turn_base + (turn_mode_ ? 2 : 0);        // AgentType.cc:113-117: [moves][turn L, R][attacks]
    t.n_action = t.attack_base + t.attack.count;
    types_.insert(std::make_pair(str, t));
}

void Engine::new_group(const char *type_name, int *handle) {            // GridWorld.cc:160-169
    auto it = types_.find(std::string(type_name));
    if (it == types_.end()) fatal("invalid name of agent type in new_group : %s", type_name);
    if (G() >= MG_MAX_GROUPS) fatal("too many groups (max %d)", (int)MG_MAX_GROUPS);
    if (where_ == DEVICE) to_host(false);
    *handle = G();
    group_type_.push_back(&it->second);
    for (auto &ar : arenas_) ar.groups.resize(G());
    refresh_host_counts();
}

void Engine::define_agent_symbol(int no, int group, int index) {        // RewardEngine.cc:28-35
    if (no >= (int)symbols_.size()) symbols_.resize(no + 1);
    symbols_[no].group = group;
    symbols_[no].index = index;
}

void Engine::define_event_node(int no, int op, int *inputs, int n_inputs) {   // RewardEngine.cc:37-49
    if (no >= (int)nodes_.size()) nodes_.resize(no + 1);
    nodes_[no].op = op;
    for (int i = 0; i < n_inputs; i++) nodes_[no].raw.push_back(inputs[i]);
}

void Engine::add_reward_rule(int on, int *receivers, float *values, int n_receiver,
                             bool is_terminal, bool auto_value) {       // RewardEngine.cc:51-69
    RuleDef r;
    r.on = on;
    for (int i = 0; i < n_receiver; i++) { r.recv.push_back(receivers[i]); r.values.push_back(values[i]); }
    r.is_terminal = is_terminal;
    r.auto_value = auto_value;
    rules_.push_back(r);
}

// ---------------------------------------------------------------------------------------------
// Reward-rule compiler.  Re-derives the reference's binding plan (related symbols, inference map,
// input_symbols / infer_obj; RewardEngine.cc:71-189) and lowers the shapes the device evaluator
// into a flat binding plan (RuleDev): 'any' levels become loops, 'all' / fixed-index levels bind once.
namespace {
struct NodeInfo { std::set<int> related; std::map<int, int> infer; };

void collect(const std::vector<NodeDef> &nodes, int no, std::vector<NodeInfo> &info, std::vector<char> &seen) {
    if (seen[no]) return;
    seen[no] = 1;
    const NodeDef &n = nodes[no];
    NodeInfo &me = info[no];
    switch (n.op) {
        case OP_AND: case OP_OR:
            for (int q = 0; q < 2; ++q) {
                collect(nodes, n.raw[q], info, seen);
                me.related.insert(info[n.raw[q]].related.begin(), info[n.raw[q]].related.end());
                me.infer.insert(info[n.raw[q]].infer.begin(), info[n.raw[q]].infer.end());
            }
            break;
        case OP_NOT:
            collect(nodes, n.raw[0], info, seen);
            me.related = info[n.raw[0]].related;
            me.infer = info[n.raw[0]].infer;
            break;
        case OP_KILL: case OP_COLLIDE: case OP_ATTACK:
            me.related.insert(n.raw[0]); me.related.insert(n.raw[1]);
            me.infer.insert(std::make_pair(n.raw[0], n.raw[1]));
            break;
        case OP_AT: case OP_IN: case OP_DIE: case OP_IN_A_LINE: case OP_ALIGN:
            me.related.insert(n.raw[0]);
            break;
        default:
            fatal("invalid event op in GridWorld::collect_related_symbol");
    }
}
}  // namespace

void Engine::compile_rules() {
    compiled_rules_.clear();
    n_allq_ = 0;
    if (rules_.size() > MG_MAX_RULES) fatal("too many reward rules (max %d)", (int)MG_MAX_RULES);
    std::vector<NodeInfo> info(nodes_.size());
    std::vector<char> seen(nodes_.size(), 0);
    for (size_t i = 0; i < nodes_.size(); ++i) collect(nodes_, (int)i, info, seen);

    for (size_t ri = 0; ri < rules_.size(); ++ri) {
        const RuleDef &rd = rules_[ri];
        const NodeInfo &on = info[rd.on];
        std::vector<int> input, infer;
        std::set<int> added;
        for (int s : on.related) {                    // first pass: symbols whose object can be inferred
            if (added.count(s)) continue;
            auto it = on.infer.find(s);
            if (it != on.infer.end()) {
                input.push_back(s); infer.push_back(it->second);
                added.insert(s); added.insert(it->second);
            }
        }
        for (int s : on.related)                      // second pass: the rest
            if (!added.count(s)) { input.push_back(s); infer.push_back(-1); }

        if (input.empty()) fatal("reward rule %d: the trigger event binds no agent symbol", (int)ri);
        if (input.size() > MG_MAX_IN)
            fatal("reward rule %d: %d input symbols (max %d)", (int)ri, (int)input.size(), (int)MG_MAX_IN);
        RuleDev R;
        memset(&R, 0, sizeof R);
        R.n_in = (int)input.size();
        // writes[sym] = role of the LAST binding of the symbol along the reference's depth-first order: level k
        // sets its subject (any / fixed index; an 'all' symbol has no entity) and then the symbol inferred from
        // the subject's op_obj (RewardEngine.cc:396-441).  Two levels inferring the same object symbol, or a level
        // inferring an earlier level's subject, overwrite -- the leaf sees the last one.
        std::map<int, int> writes;
        for (int k = 0; k < R.n_in; ++k) {
            const SymbolDef &sd = symbols_[input[k]];
            RuleInput &in = R.in[k];
            check_group(sd.group, "reward rule subject");
            in.group = sd.group; in.index = sd.index;
            in.kind = sd.index == -1 ? IN_ANY : sd.index == -2 ? IN_ALL : IN_FIXED;
            if (sd.index < -2) fatal("reward rule %d: invalid agent symbol index %d", (int)ri, sd.index);
            if (in.kind == IN_ANY) R.any_in[R.n_any++] = k;
            if (in.kind != IN_ALL) writes[input[k]] = 2 * k;
            in.has_obj = infer[k] >= 0;
            if (in.has_obj) {
                const SymbolDef &od = symbols_[infer[k]];
                check_group(od.group, "reward rule object");
                if (od.index == -2) fatal("reward rule %d: the object of attack/kill/collide cannot be a group", (int)ri);
                in.obj_group = od.group; in.obj_index = od.index;
                writes[infer[k]] = 2 * k + 1;
            } else if (in.kind == IN_FIXED) {
                R.dead = 1;                            // calc_rule never recurses past it (RewardEngine.cc:426-441)
            }
        }
        auto role_of = [&](int sym) -> int {
            auto it = writes.find(sym);
            if (it == writes.end()) fatal("reward rule %d: symbol %d is not bound by the trigger event", (int)ri, sym);
            return it->second;
        };
        // postfix lowering of the trigger tree
        struct Lower {
            const std::vector<NodeDef> &nodes; const std::vector<SymbolDef> &syms; RuleDev &R;
            decltype(role_of) &role; int &n_allq; int ri;
            void subject(RuleInstr &I, int sym) {
                if (syms[sym].index == -2) {           // quantified over the group (calc_event_node's is_all() branches)
                    if (n_allq >= MG_MAX_ALLQ) fatal("too many group-quantified ('all') events in the reward rules");
                    I.role_a = ROLE_ALL; I.all_group = syms[sym].group; I.allq = (unsigned char)n_allq++;
                } else {
                    I.role_a = (unsigned char)role(sym);
                }
            }
            void go(int no) {
                const NodeDef &n = nodes[no];
                RuleInstr I; memset(&I, 0, sizeof I);
                I.op = (unsigned char)n.op;
                switch (n.op) {
                    case OP_AND: case OP_OR: go(n.raw[0]); go(n.raw[1]); break;
                    case OP_NOT: go(n.raw[0]); break;
                    case OP_KILL: case OP_COLLIDE: case OP_ATTACK:
                        if (syms[n.raw[1]].index == -2)
                            fatal("reward rule %d: the object of attack/kill/collide cannot be a group", ri);
                        subject(I, n.raw[0]); I.role_b = (unsigned char)role(n.raw[1]); break;
                    case OP_AT: subject(I, n.raw[0]); I.i0 = n.raw[1]; I.i1 = n.raw[2]; break;
                    case OP_IN: subject(I, n.raw[0]);
                        I.i0 = n.raw[1]; I.i1 = n.raw[2]; I.i2 = n.raw[3]; I.i3 = n.raw[4]; break;
                    case OP_DIE: subject(I, n.raw[0]); break;
                    case OP_IN_A_LINE:                 // the reference asserts is_all() (RewardEngine.cc:263)
                        if (syms[n.raw[0]].index != -2) fatal("reward rule %d: 'in_a_line' needs an 'all' subject", ri);
                        subject(I, n.raw[0]); break;
                    case OP_ALIGN:
                        fatal("reward rule %d: 'align' reads GridWorld::counter_x/counter_y, which the reference never "
                              "allocates (GridWorld.cc:31, RewardEngine.cc:241-260: null dereference); not supported", ri);
                    default: fatal("invalid op of EventNode (%d)", n.op);
                }
                if (R.n_prog >= MG_MAX_PROG) fatal("reward rule trigger too large");
                R.prog[R.n_prog++] = I;
            }
        } lower{nodes_, symbols_, R, role_of, n_allq_, (int)ri};
        lower.go(rd.on);
        if (rd.recv.size() > MG_MAX_RECV) fatal("too many receivers in a reward rule");
        for (size_t q = 0; q < rd.recv.size(); ++q) {
            RuleRecv rc;
            const SymbolDef &sd = symbols_[rd.recv[q]];
            check_group(sd.group, "reward rule receiver");
            if (sd.index == -2) { rc.role = ROLE_GROUP; rc.group = sd.group; }
            else { rc.role = R.dead ? 0 : role_of(rd.recv[q]); rc.group = sd.group; }
            rc.value = rd.values[q];
            R.recv[R.n_recv++] = rc;
        }
        R.is_terminal = rd.is_terminal;
        compiled_rules_.push_back(R);
    }
    rules_compiled_ = true;
}

// ---------------------------------------------------------------------------------------------
// host image of the arenas: episode setup
void Engine::refresh_host_counts() {
    h_off_.assign((size_t)G() * (A_ + 1), 0);
    for (int g = 0; g < G(); ++g)
        for (int a = 0; a < A_; ++a)
            h_off_[(size_t)g * (A_ + 1) + a + 1] = h_off_[(size_t)g * (A_ + 1) + a] +
                (g < (int)arenas_[a].groups.size() ? arenas_[a].groups[g].size() : 0);
}

void Engine::reset() {                                // GridWorld.cc:72-118, Map.cc:23-47
    if (W_ <= 2 || H_ <= 2) fatal("map size not configured");
    settle_counts();
    if (where_ == DEVICE) {                           // keep the RNG streams: they persist across reset
        std::vector<ArenaHdr> hdr(A_);
        be::d2h(bx_, hdr.data(), hE_.hdr, sizeof(ArenaHdr) * A_);
        for (int a = 0; a < A_; ++a) {
            arenas_[a].rng = hdr[a].rng;
            for (int g = 0; g < (int)arenas_[a].groups.size(); ++g) arenas_[a].groups[g].grp_reward = hdr[a].grp_reward[g];
        }
        where_ = HOST;
    }
    file_ct_++; frame_ct_ = 0;                        // RenderGenerator::next_file (GridWorld.cc:97)
    if (d_rep_) {                                     // a new episode in every arena for the replay recorders
        std::vector<RepArena> rep(A_);
        be::d2h(bx_, rep.data(), d_rep_, sizeof(RepArena) * A_);
        for (RepArena &r : rep) r.episode++;
        be::h2d(bx_, d_rep_, rep.data(), sizeof(RepArena) * A_);
    }
    large_map_ = (long)W_ * H_ > 99 * 99;
    nsep_ = large_map_ ? ((long)W_ * H_ > 1000 * 1000 ? 16 : 8) : 1;
    for (auto &ar : arenas_) {
        ar.id_counter = 0;
        ar.slot_of_id.clear();
        for (int &c : ar.slot_ct) c = 0;
        ar.done = 0;
        ar.occ.assign((size_t)W_ * H_, OCC_EMPTY);
        ar.food.assign(food_mode_ ? (size_t)W_ * H_ : 0, 0.0f);
        for (int i = 0; i < W_; i++) { ar.occ[i] = OCC_WALL; ar.occ[(size_t)(H_ - 1) * W_ + i] = OCC_WALL; }
        for (int i = 0; i < H_; i++) { ar.occ[(size_t)i * W_] = OCC_WALL; ar.occ[(size_t)i * W_ + W_ - 1] = OCC_WALL; }
        ar.groups.resize(G());
        for (auto &g : ar.groups) g.clear();
    }
    if (!rules_compiled_) compile_rules();
    was_reset_ = true;
    order_.clear();
    refresh_host_counts();
    update_slot_space();
}

bool Engine::host_is_blank(const HostArena &ar, int x, int y, int w, int h) const {   // Map.cc:454-470
    if (x < 0 || y < 0 || x + w >= W_ || y + h >= H_) return false;
    for (int i = 0; i < w; i++)
        for (int j = 0; j < h; j++)
            if (ar.occ[(size_t)(y + j) * W_ + x + i] != OCC_EMPTY) return false;
    return true;
}

static inline uint32_t rng_next(uint32_t &state) { state = mulmod31(state, MINSTD_A); return state; }

void Engine::host_random_blank(HostArena &ar, int w, int h, int &x, int &y) {         // Map.cc:49-63
    int tries = 0;
    for (;;) {
        x = (int)rng_next(ar.rng) % (W_ - w);
        y = (int)rng_next(ar.rng) % (H_ - h);
        if (host_is_blank(ar, x, y, w, h)) return;
        if (tries++ > W_ * H_) fatal("cannot find a blank position in a filled map");
    }
}

int Engine::host_add_wall(HostArena &ar, int x, int y) {                              // Map.cc:108-115
    if (x < 0 || y < 0 || x >= W_ || y >= H_) return 1;
    int &c = ar.occ[(size_t)y * W_ + x];
    if (c >= 0 || c == OCC_FOOD) return 1;            // a BLANK slot with an occupier is refused (Map.cc:108-112)
    c = OCC_WALL;
    return 0;
}

int Engine::host_add_agent(HostArena &ar, int g, int x, int y, int dir) {             // Map.cc:75-97 + Agent ctor
    const AgentTypeDef &t = *group_type_[g];
    const bool upright = dir == DIR_NORTH || dir == DIR_SOUTH;                        // get_size_for_dir, Map.cc:597-607
    const int bw = upright ? t.width : t.length, bh = upright ? t.length : t.width;
    if (!host_is_blank(ar, x, y, bw, bh)) return 1;
    HostGroup &hg = ar.groups[g];
    int i = hg.size();
    if (i >= (1 << 23)) fatal("too many agents in one group of one arena (max %d)", 1 << 23);
    hg.resize(i + 1);
    hg.x[i] = x; hg.y[i] = y; hg.id[i] = ar.id_counter++;
    ar.slot_of_id.push_back(ar.slot_ct[g]++);           // the id's slot (slot_phases.h); ids are handed out in order
    hg.act[i] = t.n_action;                           // "dangerous here !" (GridWorld.h:140)
    hg.op_obj[i] = -1;
    hg.hp[i] = t.hp;
    hg.next_reward[i] = t.step_reward; hg.last_reward[i] = 0.0f;
    hg.last_op[i] = OP_NULL; hg.flags[i] = 0; hg.dir[i] = (unsigned char)dir;
    int code = code_make(g, i);
    for (int bx = 0; bx < bw; bx++)
        for (int by = 0; by < bh; by++)
            ar.occ[(size_t)(y + by) * W_ + x + bx] = code;
    return 0;
}

void Engine::add_agents(int group, int n, const char *method,
                        const int *pos_x, const int *pos_y, const int *pos_dir) {    // GridWorld.cc:180-290
    if (!was_reset_) fatal("add_agents before reset");
    if (where_ == DEVICE) to_host(false);
    const bool is_random = strequ(method, "random"), is_custom = strequ(method, "custom"),
               is_fill = strequ(method, "fill");
    if (!is_random && !is_custom && !is_fill) fatal("unsupported method in GridWorld::add_agents : %s", method);
    if (group != -1) check_group(group, "GridWorld::add_agents");
    for (int a = 0; a < A_; ++a) {
        if (sel_arena_ >= 0 && sel_arena_ != a) continue;
        HostArena &ar = arenas_[a];
        if (group == -1) {
            if (is_random) {
                for (int i = 0; i < n; i++) { int x, y; host_random_blank(ar, 1, 1, x, y); host_add_wall(ar, x, y); }
            } else if (is_custom) {
                for (int i = 0; i < n; i++) host_add_wall(ar, pos_x[i], pos_y[i]);
            } else {
                int x0 = pos_x[0], y0 = pos_x[1], x1 = x0 + pos_x[2], y1 = y0 + pos_x[3];
                for (int x = x0; x < x1; x++) for (int y = y0; y < y1; y++) host_add_wall(ar, x, y);
            }
        } else {
            const AgentTypeDef &t = *group_type_[group];
            if (is_random) {
                for (int i = 0; i < n; i++) {
                    // GridWorld.cc:228-243: with turn_mode the direction is drawn first, then the position of the
                    // (possibly rotated) footprint
                    const int dir = turn_mode_ ? (int)(rng_next(ar.rng) % 4u) : DIR_NORTH;
                    const bool upright = dir == DIR_NORTH || dir == DIR_SOUTH;
                    int x, y;
                    host_random_blank(ar, upright ? t.width : t.length, upright ? t.length : t.width, x, y);
                    host_add_agent(ar, group, x, y, dir);
                }
            } else if (is_custom) {
                for (int i = 0; i < n; i++) {
                    if (pos_dir && pos_dir[i] >= 4) fatal("invalid direction in GridWorld::add_agent");
                    host_add_agent(ar, group, pos_x[i], pos_y[i], turn_mode_ && pos_dir ? pos_dir[i] : DIR_NORTH);
                }
            } else {
                int x0 = pos_x[0], y0 = pos_x[1], x1 = x0 + pos_x[2], y1 = y0 + pos_x[3];
                const int dir = turn_mode_ ? pos_x[4] : DIR_NORTH;                    // GridWorld.cc:264-287
                if (dir < 0 || dir >= 4) fatal("invalid direction in GridWorld::add_agent");
                const bool upright = dir == DIR_NORTH || dir == DIR_SOUTH;
                const int mw = upright ? t.width : t.length, mh = upright ? t.length : t.width;
                for (int x = x0; x < x1; x += mw)
                    for (int y = y0; y < y1; y += mh) host_add_agent(ar, group, x, y, dir);
            }
        }
    }
    refresh_host_counts();
    update_slot_space();
}

// ---------------------------------------------------------------------------------------------
// device image
void Engine::ensure_backend() {
    if (bx_) {
        // one context per engine for its whole life: the device cannot change under allocations that live on it
        if (device_id_ >= 0 && device_id_ != be::device_of(bx_)) fatal("device_id changed after the engine had started on device %d", be::device_of(bx_));
        return;
    }
    std::string err;
    bx_ = be::create(device_id_, &err);
    if (!bx_) fatal("no usable CUDA device for the B200 engine: %s (there is no CPU fallback)", err.c_str());
}

void *Engine::dalloc(size_t bytes) {
    void *p = be::dmalloc(bx_, bytes ? bytes : 16);
    dev_allocs_.push_back(p);
    return p;
}

void Engine::free_device() {
    for (void *p : dev_allocs_) be::dfree(bx_, p);
    dev_allocs_.clear();
    if (d_view_stage_) be::dfree(bx_, d_view_stage_);
    if (d_feat_stage_) be::dfree(bx_, d_feat_stage_);
    if (d_io_stage_) be::dfree(bx_, d_io_stage_);
    d_view_stage_ = d_feat_stage_ = nullptr; d_io_stage_ = nullptr;
    view_stage_bytes_ = feat_stage_bytes_ = io_stage_bytes_ = 0;
    d_nbr_lut_ = nullptr;
    nbr_lut_.clear();
    dE_ = nullptr;
    cap_.clear();
}

void *Engine::io_stage(size_t bytes) {
    if (bytes > io_stage_bytes_) {
        if (d_io_stage_) be::dfree(bx_, d_io_stage_);
        io_stage_bytes_ = bytes + bytes / 4 + 256;
        d_io_stage_ = be::dmalloc(bx_, io_stage_bytes_);
    }
    return d_io_stage_;
}

// The per-agent read-backs (get_reward, get_info's id/pos/alive/hp, get_action_mask, get_mean_action, get_neighbours,
// get_slots) write into caller buffers that are all host memory or all CUDA device memory, the null ones aside.
// out_memory says which: 1 device, 0 host, -1 refused.
static int out_memory(const char *what, std::initializer_list<const void *> bufs) {
    int dev = 0, host = 0;
    for (const void *p : bufs) if (p) ++(be::is_device_ptr(p) ? dev : host);
    const char *q = bufs.size() == 2 ? "both" : "all";
    if (dev && host) return refuse("%s must %s be host memory or %s CUDA device memory", what, q, q);
    return dev ? 1 : 0;
}

// launch(void **to) writes each wanted part to to[i] (nullptr: not wanted).  Device buffers: to[] are the caller's, the
// launch is sized by the host's upper-bound counts and clamped by the device's, and nothing is staged, allocated or
// waited for, so the call can be recorded into a CUDA graph.  Host buffers (the caller settled the counts): the wanted
// parts are packed back to back in one i/o staging block, then each is copied back and counted in IO_D2H.  Nothing runs
// when the wanted parts total 0 bytes.
template <size_t N, class F> void Engine::read_back(bool dev, const OutPart (&parts)[N], F &&launch) {
    void *to[N];
    size_t bytes = 0;
    for (size_t i = 0; i < N; ++i) { to[i] = parts[i].buf; bytes += parts[i].buf ? parts[i].bytes : 0; }
    if (bytes == 0) return;
    if (dev) { launch(to); return; }
    char *st = (char *)io_stage(bytes);
    for (size_t i = 0, off = 0; i < N; ++i)
        if (parts[i].buf) { to[i] = st + off; off += parts[i].bytes; }
    launch(to);
    for (size_t i = 0; i < N; ++i)
        if (parts[i].buf) { be::d2h(bx_, parts[i].buf, to[i], parts[i].bytes); io_[IO_D2H] += (long long)parts[i].bytes; }
}

// the padded observation planes cover the widest view window of any group, in any heading when agents can turn
int Engine::view_pad() const {
    int pad = 0;
    for (int g = 0; g < G(); ++g) {
        const AgentTypeDef &t = *group_type_[g];
        const int ox = t.view_x_offset + t.view.x1, oy = t.view_y_offset + t.view.y1;
        const int ext[4] = {-ox, ox + t.view.width - 1, -oy, oy + t.view.height - 1};
        for (int e : ext) pad = std::max(pad, e + (turn_mode_ ? std::max(t.width, t.length) : 0));
    }
    return pad;
}

int Engine::max_agents_per_arena() const {
    int m = 0;
    for (int a = 0; a < A_; ++a) {
        int s = 0;
        for (int g = 0; g < G(); ++g) s += count(g, a);
        m = std::max(m, s);
    }
    return m;
}

template <class T>
static T *upload_vec(be::Ctx *bx_, std::vector<void *> &allocs, const std::vector<T> &v) {
    T *p = (T *)be::dmalloc(bx_, std::max<size_t>(v.size(), 1) * sizeof(T));
    allocs.push_back(p);
    if (!v.empty()) be::h2d(bx_, p, v.data(), v.size() * sizeof(T));
    return p;
}

// The view LUTs of get_neighbours: per group and heading (one run of view_count cells, four in turn_mode) the in-range
// cells of the window in key order, built from the group's geometry alone with the functions the kernel and the test
// emulation use (nbr_phases.h).  Uploaded when the device image is new or the LUTs changed (turn_mode or the padded plane
// width), so the call itself never allocates or copies.
void Engine::upload_nbr_luts(bool force) {
    const int Gn = G();
    std::vector<NbrCell> lut;
    nbr_lut_base_.assign(Gn, 0);
    nbr_key_fits_.assign(Gn, 0);
    for (int g = 0; g < Gn; ++g) {
        const AgentTypeDef &t = *group_type_[g];
        const GroupDev &D = hE_.grp[g];
        nbr_lut_base_[g] = lut.size();
        // no in-range cell lies farther than kpad cells from the body on either axis: d2 <= 2 kpad^2
        const long long cells = (long long)t.view.width * t.view.height;
        if ((2LL * hE_.kpad * hE_.kpad + 1) * cells > 0x7fffffffLL) continue;
        nbr_key_fits_[g] = 1;
        for (int d = 0; d < (turn_mode_ ? 4 : 1); ++d) {
            const int dir = turn_mode_ ? d : DIR_NORTH;
            const size_t first = lut.size();
            for (int vy = 0; vy < t.view.height; ++vy)
                for (int vx = 0; vx < t.view.width; ++vx) {
                    if (!t.view.mask[(size_t)vy * t.view.width + vx]) continue;
                    int dx, dy;
                    nbr_view_delta(hE_, D, dir, vx, vy, dx, dy);
                    NbrCell c;
                    c.off = dy * hE_.kw + dx;
                    c.delta = (dx & 0xffff) | (int)((unsigned)dy << 16);
                    c.key = nbr_cell_key(D, dir, dx, dy, vx, vy);
                    c.cell = vx | vy << 16;
                    lut.push_back(c);
                }
            std::sort(lut.begin() + first, lut.end(), [](const NbrCell &p, const NbrCell &q) { return p.key < q.key; });
        }
    }
    const bool same = lut.size() == nbr_lut_.size() && (lut.empty() || !memcmp(lut.data(), nbr_lut_.data(), lut.size() * sizeof(NbrCell)));
    if (!force && same) return;
    if (!lut.empty()) be::h2d(bx_, d_nbr_lut_, lut.data(), lut.size() * sizeof(NbrCell));
    nbr_lut_.swap(lut);
}

// The slot table of the host image.  Its width covers every id an arena or a live snapshot's arena has handed out, so a
// restore never needs more; it only grows (by half at least, so that mid-episode placements rarely re-allocate), and the
// SlotDev block that names it keeps its address.
void Engine::upload_slots() {
    int need = 0;
    for (const HostArena &ar : arenas_) need = std::max(need, ar.id_counter);
    for (const ArenaSnapshot &sn : snaps_)
        if (sn.live) need = std::max(need, sn.max_ids);
    if (!d_slot_dev_) d_slot_dev_ = (SlotDev *)be::dmalloc(bx_, sizeof(SlotDev));
    if (!d_slot_tab_ || need > slot_id_cap_) {
        if (d_slot_tab_) be::dfree(bx_, d_slot_tab_);
        const int want = std::max(need, slot_id_cap_ + slot_id_cap_ / 2);
        slot_id_cap_ = std::max(64, (want + 63) / 64 * 64);
        d_slot_tab_ = (int *)be::dmalloc(bx_, (size_t)A_ * slot_row_stride(slot_id_cap_) * 4);
        const SlotDev T = {d_slot_tab_, slot_id_cap_};
        be::h2d(bx_, d_slot_dev_, &T, sizeof T);
    }
    const long ld = slot_row_stride(slot_id_cap_);
    std::vector<int> tab((size_t)A_ * ld, -1);
    for (int a = 0; a < A_; ++a) {
        int *row = tab.data() + a * ld;
        std::copy(arenas_[a].slot_ct, arenas_[a].slot_ct + SLOT_HDR, row);
        std::copy(arenas_[a].slot_of_id.begin(), arenas_[a].slot_of_id.end(), row + SLOT_HDR);
    }
    be::h2d(bx_, d_slot_tab_, tab.data(), tab.size() * 4);
}

// S(g): the largest slot count of group g over the arenas as they are now and over the arenas of every snapshot a restore
// may copy in.  Device restores cannot exceed it, so only the host-side calls that can change it recompute it.
void Engine::update_slot_space() {
    const int Gn = G();
    slot_space_.assign(Gn, 0);
    std::vector<int> tab;
    const long ld = slot_row_stride(slot_id_cap_);
    if (where_ == DEVICE) {
        tab.resize((size_t)A_ * ld);
        be::d2h(bx_, tab.data(), d_slot_tab_, tab.size() * 4);
    }
    for (int a = 0; a < A_; ++a)
        for (int g = 0; g < Gn; ++g)
            slot_space_[g] = std::max(slot_space_[g], where_ == DEVICE ? tab[a * ld + g] : arenas_[a].slot_ct[g]);
    const int pad = view_pad();
    for (const ArenaSnapshot &sn : snaps_)
        if (sn.live && snap_matches(sn, pad))
            for (int g = 0; g < Gn; ++g) slot_space_[g] = std::max(slot_space_[g], sn.slot_max[g]);
}

void Engine::to_device() {
    if (where_ == DEVICE) return;
    if (!was_reset_) fatal("environment used before reset");
    ensure_backend();
    const int Gn = G();
    const int pad = view_pad();
    // capacities: grow-only while the geometry is unchanged; they also hold every arena of every snapshot a restore
    // may copy in
    std::vector<int> need(Gn, 0);
    for (int g = 0; g < Gn; ++g) {
        for (int a = 0; a < A_; ++a) need[g] = std::max(need[g], count(g, a));
        for (const ArenaSnapshot &sn : snaps_)
            if (sn.live && snap_matches(sn, pad)) need[g] = std::max(need[g], sn.max_n[g]);
        need[g] = std::max(64, (need[g] + 63) / 64 * 64);
    }
    // env_config_game may change the modes between episodes (as in the reference): everything an allocation's size or
    // presence depends on is part of the predicate
    bool realloc = dE_ == nullptr || hE_.A != A_ || hE_.W != W_ || hE_.H != H_ || hE_.G != Gn || hE_.kpad != pad ||
                   (hE_.food != nullptr) != food_mode_;
    if (!realloc) for (int g = 0; g < Gn; ++g) if (need[g] > cap_[g]) realloc = true;
    if (realloc) {
        // the event counters are "since construction": they survive a re-allocation (a late add_agents beyond capacity)
        std::vector<long long> saved_counters;
        if (dE_ != nullptr) { saved_counters.resize(MG_N_COUNTERS); be::d2h(bx_, saved_counters.data(), hE_.counters, sizeof(long long) * MG_N_COUNTERS); }
        free_device();
        memset(&hE_, 0, sizeof hE_);
        cap_ = need;
        hE_.A = A_; hE_.W = W_; hE_.H = H_; hE_.G = Gn;
        int foff = 0, max_body = 1, max_cells = 1;
        for (int g = 0; g < Gn; ++g) {
            const AgentTypeDef &t = *group_type_[g];
            GroupDev &D = hE_.grp[g];
            D.body_w = t.width; D.body_l = t.length;
            D.max_hp = t.hp; D.damage = t.damage; D.step_recover = t.step_recover; D.kill_supply = t.kill_supply;
            D.eat_ability = t.eat_ability; D.food_supply = t.food_supply;
            D.step_reward = t.step_reward; D.kill_reward = t.kill_reward;
            D.dead_penalty = t.dead_penalty; D.attack_penalty = t.attack_penalty;
            D.attack_in_group = t.attack_in_group;
            D.can_absorb = t.can_absorb;
            if (t.can_absorb) hE_.any_absorb = 1;
            D.view_w = t.view.width; D.view_h = t.view.height; D.view_x1 = t.view.x1; D.view_y1 = t.view.y1;
            D.view_count = t.view.count;
            D.view_xoff = t.view_x_offset; D.view_yoff = t.view_y_offset;
            D.att_xoff = t.att_x_offset; D.att_yoff = t.att_y_offset;
            D.n_move = t.move.count; D.attack_base = t.attack_base; D.n_action = t.n_action; D.n_attack = t.attack.count;
            D.channel = group2channel(g);
            D.feature_size = feature_size(g);
            D.move_dx = upload_vec(bx_, dev_allocs_, t.move.dx); D.move_dy = upload_vec(bx_, dev_allocs_, t.move.dy);
            D.att_dx = upload_vec(bx_, dev_allocs_, t.attack.dx); D.att_dy = upload_vec(bx_, dev_allocs_, t.attack.dy);
            D.view_mask = upload_vec(bx_, dev_allocs_, t.view.mask);
            D.cap = cap_[g];
            D.foff = foff; foff += cap_[g];
            max_body = std::max(max_body, t.width * t.length);
            max_cells = std::max(max_cells, t.view.width * t.view.height);
            size_t n = (size_t)A_ * cap_[g];
            for (int b = 0; b < 2; ++b) {
                AgentSoA &s = D.soa[b];
                s.x = (int *)dalloc(n * 4); s.y = (int *)dalloc(n * 4); s.hp = (float *)dalloc(n * 4);
                s.act = (int *)dalloc(n * 4); s.id = (int *)dalloc(n * 4);
                s.next_reward = (float *)dalloc(n * 4); s.last_reward = (float *)dalloc(n * 4);
                s.op_obj = (int *)dalloc(n * 4);
                s.last_op = (unsigned char *)dalloc(n); s.flags = (unsigned char *)dalloc(n); s.dir = (unsigned char *)dalloc(n);
            }
            D.ev_rank = (int *)dalloc(n * 4);
        }
        hE_.cap_total = foff; hE_.max_body = max_body; hE_.scratch_stride = foff;
        size_t cells = (size_t)A_ * W_ * H_, sc = (size_t)A_ * foff;
        hE_.hdr = (ArenaHdr *)dalloc(sizeof(ArenaHdr) * A_);
        hE_.n = (int *)dalloc((size_t)Gn * A_ * 4); hE_.dead_ct = (int *)dalloc((size_t)Gn * A_ * 4);
        hE_.off = (int *)dalloc((size_t)Gn * (A_ + 1) * 4);
        hE_.done = (int *)dalloc((size_t)A_ * 4);
        hE_.occ = (int *)dalloc(cells * 4); hE_.claim_head = (int *)dalloc(cells * 4);
        hE_.food = food_mode_ ? (float *)dalloc(cells * 4) : nullptr;
        {   // padded observation planes (dev_types.h)
            hE_.kpad = pad; hE_.kw = W_ + 2 * pad; hE_.kplane = (long)hE_.kw * (H_ + 2 * pad);
            const size_t blank = (size_t)(2 * pad + 1) * hE_.kw;          // the blank arena's window, zero for good
            hE_.kind = (unsigned char *)dalloc((size_t)A_ * hE_.kplane + blank + 16);
            be::dmemset(bx_, hE_.kind + (size_t)A_ * hE_.kplane, 0, blank + 16);
            hE_.hpn = (float *)dalloc(((size_t)A_ * hE_.kplane + 4) * 4);
            be::dmemset(bx_, hE_.hpn, 0, ((size_t)A_ * hE_.kplane + 4) * 4);
        }
        hE_.att_rank = (int *)dalloc(sc * 4); hE_.tgt = (int *)dalloc(sc * 4);
        hE_.in_head = (int *)dalloc(sc * 4); hE_.in_next = (int *)dalloc(sc * 4);
        hE_.death = (int *)dalloc(sc * 4); hE_.mv_nx = (int *)dalloc(sc * 4); hE_.mv_ny = (int *)dalloc(sc * 4);
        hE_.mv_key = (unsigned *)dalloc(sc * 4); hE_.hp_fin = (float *)dalloc(sc * 4);
        hE_.mv_state = (unsigned char *)dalloc(sc);
        hE_.jv = (int *)dalloc(sc * 4); hE_.sh_head = (int *)dalloc(sc * 4); hE_.sh_next = (int *)dalloc(sc * 4);
        hE_.sh_first = (int *)dalloc(sc * 4); hE_.att_agent = (int *)dalloc(sc * 4);
        hE_.cl_next = (int *)dalloc(sc * max_body * 4);
        hE_.counters = (long long *)dalloc(sizeof(long long) * MG_N_COUNTERS);
        if (saved_counters.empty()) be::dmemset(bx_, hE_.counters, 0, sizeof(long long) * MG_N_COUNTERS);
        else be::h2d(bx_, hE_.counters, saved_counters.data(), sizeof(long long) * MG_N_COUNTERS);
        hE_.team_scratch = (int *)dalloc(sizeof(int) * 2 * 4096);
        hE_.mm_count = (int *)dalloc((size_t)A_ * Gn * max_cells * 4);
        hE_.mm_total = (int *)dalloc((size_t)A_ * Gn * 4);
        d_mm_val_ = (float *)dalloc((size_t)A_ * Gn * max_cells * 4);
        hE_.rules = (const RuleDev *)dalloc(sizeof(RuleDev) * (compiled_rules_.size() + 1));
        size_t lut_cells = 0;                         // room for four headings: turn_mode may change without a re-allocation
        for (int g = 0; g < Gn; ++g) lut_cells += 4 * (size_t)hE_.grp[g].view_count;
        d_nbr_lut_ = (NbrCell *)dalloc(sizeof(NbrCell) * lut_cells);
        dE_ = (EngineDev *)dalloc(sizeof(EngineDev));
    }
    // constants that may change between episodes without a re-allocation
    hE_.nsep = nsep_; hE_.large_map = large_map_; hE_.bandwidth = (W_ + nsep_ - 1) / nsep_;
    hE_.minimap_mode = minimap_mode_; hE_.embedding_size = embedding_size_; hE_.turn_mode = turn_mode_ ? 1 : 0;
    hE_.food_mode = food_mode_ ? 1 : 0;
    hE_.n_channel = n_channel(); hE_.channel_base = group2channel(0);
    {
        uint32_t p = MINSTD_A;
        for (int b = 0; b < 32; ++b) { hE_.pow2[b] = p; p = mulmod31(p, p); }
    }
    hE_.n_rules = (int)compiled_rules_.size();
    if (hE_.n_rules) be::h2d(bx_, (void *)hE_.rules, compiled_rules_.data(), sizeof(RuleDev) * compiled_rules_.size());
    hE_.n_allq = n_allq_;
    for (int r = 0; r < hE_.n_rules; ++r) {
        const RuleDev &R = compiled_rules_[r];
        RuleHot &H = hE_.rule_hot[r];
        H.shape = R.dead ? RULE_DEAD : (R.n_in == 1 && R.n_any == 1) ? RULE_ONE_ANY : RULE_GENERAL;
        H.terminal = R.is_terminal ? 1 : 0;
        H.group = (unsigned char)R.in[0].group; H.has_obj = (unsigned char)R.in[0].has_obj;
        H.obj_group = R.in[0].obj_group; H.obj_index = R.in[0].obj_index;
        H.simple_op = 0;
        if (H.shape == RULE_ONE_ANY && R.in[0].has_obj && R.n_prog == 1 && R.prog[0].role_a == 0 && R.prog[0].role_b == 1 &&
            (R.prog[0].op == OP_KILL || R.prog[0].op == OP_ATTACK || R.prog[0].op == OP_COLLIDE))
            H.simple_op = R.prog[0].op;
        if (r < MG_HOT_RULES) {
            RuleSmall &Sm = hE_.rule_small[r];
            memset(&Sm, 0, sizeof Sm);
            Sm.n_prog = -1;
            if (R.n_prog <= MG_HOT_PROG && R.n_recv <= MG_HOT_RECV) {
                Sm.n_prog = R.n_prog; Sm.n_recv = R.n_recv;
                for (int q = 0; q < R.n_prog; ++q) Sm.prog[q] = R.prog[q];
                for (int q = 0; q < R.n_recv; ++q) Sm.recv[q] = R.recv[q];
            }
        }
    }
    for (int g = 0; g < Gn; ++g) hE_.grp[g].feature_size = feature_size(g);
    curmask_ = 0;
    upload_nbr_luts(realloc);

    // ---- pack and upload the state
    std::vector<int> ibuf; std::vector<float> fbuf; std::vector<unsigned char> bbuf;
    for (int g = 0; g < Gn; ++g) {
        const size_t cap = cap_[g], n = (size_t)A_ * cap;
        const AgentSoA &s = hE_.grp[g].soa[0];
        auto up_i = [&](int *dst, std::vector<int> HostGroup::*m) {
            ibuf.assign(n, 0);
            for (int a = 0; a < A_; ++a) { const auto &v = arenas_[a].groups[g].*m; std::copy(v.begin(), v.end(), ibuf.begin() + a * cap); }
            be::h2d(bx_, dst, ibuf.data(), n * 4);
        };
        auto up_f = [&](float *dst, std::vector<float> HostGroup::*m) {
            fbuf.assign(n, 0);
            for (int a = 0; a < A_; ++a) { const auto &v = arenas_[a].groups[g].*m; std::copy(v.begin(), v.end(), fbuf.begin() + a * cap); }
            be::h2d(bx_, dst, fbuf.data(), n * 4);
        };
        auto up_b = [&](unsigned char *dst, std::vector<unsigned char> HostGroup::*m) {
            bbuf.assign(n, 0);
            for (int a = 0; a < A_; ++a) { const auto &v = arenas_[a].groups[g].*m; std::copy(v.begin(), v.end(), bbuf.begin() + a * cap); }
            be::h2d(bx_, dst, bbuf.data(), n);
        };
        up_i(s.x, &HostGroup::x); up_i(s.y, &HostGroup::y); up_i(s.act, &HostGroup::act);
        up_i(s.id, &HostGroup::id); up_i(s.op_obj, &HostGroup::op_obj);
        up_f(s.hp, &HostGroup::hp); up_f(s.next_reward, &HostGroup::next_reward); up_f(s.last_reward, &HostGroup::last_reward);
        up_b(s.last_op, &HostGroup::last_op); up_b(s.flags, &HostGroup::flags); up_b(s.dir, &HostGroup::dir);
    }
    for (int a = 0; a < A_; ++a)
        be::h2d(bx_, hE_.occ + (size_t)a * W_ * H_, arenas_[a].occ.data(), (size_t)W_ * H_ * 4);
    if (food_mode_)
        for (int a = 0; a < A_; ++a) {
            arenas_[a].food.resize((size_t)W_ * H_, 0.0f);
            be::h2d(bx_, hE_.food + (size_t)a * W_ * H_, arenas_[a].food.data(), (size_t)W_ * H_ * 4);
        }
    {   // the kind plane mirrors the occupancy image; from here on the step kernels keep it current
        std::vector<unsigned char> kp((size_t)hE_.kplane);
        for (int a = 0; a < A_; ++a) {
            std::fill(kp.begin(), kp.end(), (unsigned char)0);
            const std::vector<int> &occ = arenas_[a].occ;
            for (int y = 0; y < H_; ++y)
                for (int x = 0; x < W_; ++x) {
                    const int o = occ[(size_t)y * W_ + x];
                    kp[(size_t)(y + hE_.kpad) * hE_.kw + x + hE_.kpad] =
                        o == OCC_WALL ? KIND_WALL : o == OCC_FOOD ? KIND_FOOD : o >= 0 ?
                        kind_agent(code_group(o), arenas_[a].groups[code_group(o)].hp[code_index(o)] == group_type_[code_group(o)]->hp) : KIND_EMPTY;
                }
            be::h2d(bx_, hE_.kind + (size_t)a * hE_.kplane, kp.data(), kp.size());
        }
        // ... and the hp_norm plane: hp / max_hp (Map.cc:197) under every cell a living agent covers
        std::vector<float> hp((size_t)hE_.kplane);
        for (int a = 0; a < A_; ++a) {
            std::fill(hp.begin(), hp.end(), 0.0f);
            for (int g = 0; g < Gn; ++g) {
                const HostGroup &hg = arenas_[a].groups[g];
                const AgentTypeDef &t = *group_type_[g];
                for (int i = 0; i < hg.size(); ++i) {
                    if (hg.flags[i] & FLAG_DEAD) continue;
                    const bool upright = !turn_mode_ || hg.dir[i] == DIR_NORTH || hg.dir[i] == DIR_SOUTH;
                    const int bw = upright ? t.width : t.length, bh = upright ? t.length : t.width;
                    const float v = hg.hp[i] / t.hp;
                    for (int bx = 0; bx < bw; ++bx)
                        for (int by = 0; by < bh; ++by)
                            hp[(size_t)(hg.y[i] + by + hE_.kpad) * hE_.kw + hg.x[i] + bx + hE_.kpad] = v;
                }
            }
            be::h2d(bx_, hE_.hpn + (size_t)a * hE_.kplane, hp.data(), hp.size() * 4);
        }
    }
    be::dmemset(bx_, hE_.claim_head, 0xff, (size_t)A_ * W_ * H_ * 4);
    {
        std::vector<ArenaHdr> hdr(A_);
        std::vector<int> n((size_t)Gn * A_), dc((size_t)Gn * A_), done(A_);
        for (int a = 0; a < A_; ++a) {
            memset(&hdr[a], 0, sizeof(ArenaHdr));
            hdr[a].rng = hdr[a].rng_next = arenas_[a].rng;
            hdr[a].done = done[a] = arenas_[a].done;
            hdr[a].id_counter = arenas_[a].id_counter;
            for (int g = 0; g < Gn; ++g) {
                hdr[a].grp_reward[g] = arenas_[a].groups[g].grp_reward;
                hdr[a].n_cull[g] = arenas_[a].groups[g].n_cull;
                n[(size_t)g * A_ + a] = arenas_[a].groups[g].size();
                dc[(size_t)g * A_ + a] = arenas_[a].groups[g].dead_ct;
            }
        }
        be::h2d(bx_, hE_.hdr, hdr.data(), sizeof(ArenaHdr) * A_);
        be::h2d(bx_, hE_.n, n.data(), n.size() * 4);
        be::h2d(bx_, hE_.dead_ct, dc.data(), dc.size() * 4);
        be::h2d(bx_, hE_.done, done.data(), done.size() * 4);
        be::h2d(bx_, hE_.off, h_off_.data(), h_off_.size() * 4);
    }
    upload_slots();
    be::h2d(bx_, dE_, &hE_, sizeof(EngineDev));
    ++state_version_;
    may_have_dead_ = true;                            // conservative: the first clear_dead after an upload re-reads the counts
    where_ = DEVICE;
}

void Engine::to_host(bool keep_device_authoritative) {
    if (where_ == HOST) return;
    settle_counts();
    const int Gn = G();
    std::vector<int> ibuf; std::vector<float> fbuf; std::vector<unsigned char> bbuf;
    std::vector<int> dc((size_t)Gn * A_);
    be::d2h(bx_, dc.data(), hE_.dead_ct, dc.size() * 4);
    std::vector<ArenaHdr> hdr(A_);
    be::d2h(bx_, hdr.data(), hE_.hdr, sizeof(ArenaHdr) * A_);
    for (int g = 0; g < Gn; ++g) {
        const size_t cap = cap_[g], n = (size_t)A_ * cap;
        const AgentSoA &s = hE_.grp[g].soa[(curmask_ >> g) & 1u];
        for (int a = 0; a < A_; ++a) arenas_[a].groups[g].resize(count(g, a));
        auto dn_i = [&](const int *src, std::vector<int> HostGroup::*m) {
            ibuf.resize(n); be::d2h(bx_, ibuf.data(), src, n * 4);
            for (int a = 0; a < A_; ++a) { auto &v = arenas_[a].groups[g].*m; std::copy(ibuf.begin() + a * cap, ibuf.begin() + a * cap + v.size(), v.begin()); }
        };
        auto dn_f = [&](const float *src, std::vector<float> HostGroup::*m) {
            fbuf.resize(n); be::d2h(bx_, fbuf.data(), src, n * 4);
            for (int a = 0; a < A_; ++a) { auto &v = arenas_[a].groups[g].*m; std::copy(fbuf.begin() + a * cap, fbuf.begin() + a * cap + v.size(), v.begin()); }
        };
        auto dn_b = [&](const unsigned char *src, std::vector<unsigned char> HostGroup::*m) {
            bbuf.resize(n); be::d2h(bx_, bbuf.data(), src, n);
            for (int a = 0; a < A_; ++a) { auto &v = arenas_[a].groups[g].*m; std::copy(bbuf.begin() + a * cap, bbuf.begin() + a * cap + v.size(), v.begin()); }
        };
        dn_i(s.x, &HostGroup::x); dn_i(s.y, &HostGroup::y); dn_i(s.act, &HostGroup::act);
        dn_i(s.id, &HostGroup::id); dn_i(s.op_obj, &HostGroup::op_obj);
        dn_f(s.hp, &HostGroup::hp); dn_f(s.next_reward, &HostGroup::next_reward); dn_f(s.last_reward, &HostGroup::last_reward);
        dn_b(s.last_op, &HostGroup::last_op); dn_b(s.flags, &HostGroup::flags); dn_b(s.dir, &HostGroup::dir);
        for (int a = 0; a < A_; ++a) {
            arenas_[a].groups[g].dead_ct = dc[(size_t)g * A_ + a];
            arenas_[a].groups[g].grp_reward = hdr[a].grp_reward[g];
            arenas_[a].groups[g].n_cull = hdr[a].n_cull[g];
        }
    }
    for (int a = 0; a < A_; ++a) {
        arenas_[a].occ.resize((size_t)W_ * H_);
        be::d2h(bx_, arenas_[a].occ.data(), hE_.occ + (size_t)a * W_ * H_, (size_t)W_ * H_ * 4);
        if (food_mode_) {
            arenas_[a].food.resize((size_t)W_ * H_);
            be::d2h(bx_, arenas_[a].food.data(), hE_.food + (size_t)a * W_ * H_, (size_t)W_ * H_ * 4);
        }
        arenas_[a].rng = hdr[a].rng;
        arenas_[a].done = hdr[a].done;
        arenas_[a].id_counter = hdr[a].id_counter;
    }
    {   // the slot table: restores may have replaced rows
        const long ld = slot_row_stride(slot_id_cap_);
        std::vector<int> tab((size_t)A_ * ld);
        be::d2h(bx_, tab.data(), d_slot_tab_, tab.size() * 4);
        for (int a = 0; a < A_; ++a) {
            const int *row = tab.data() + a * ld;
            std::copy(row, row + SLOT_HDR, arenas_[a].slot_ct);
            arenas_[a].slot_of_id.assign(row + SLOT_HDR, row + SLOT_HDR + arenas_[a].id_counter);
        }
    }
    if (!keep_device_authoritative) where_ = HOST;
}

// ---------------------------------------------------------------------------------------------
// the step loop
void Engine::stage_reserve(void *&p, size_t &have, size_t need) {
    if (need <= have) return;
    if (p) be::dfree(bx_, p);
    have = need + need / 8 + 256;
    p = be::dmalloc(bx_, have);
}

// The observation pre-pass (normalised minimap) for group's observers, unless the last one still holds: its products
// depend on the state, on the observer's view size (minimap grid) and on whether the observer's type skips absorbed
// agents in the minimap (GridWorld.cc:343-347)
void Engine::prepare_obs(int group) {
    const AgentTypeDef &t = *group_type_[group];
    if (prep_version_ != state_version_ || prep_vw_ != t.view.width || prep_vh_ != t.view.height ||
        prep_skip_absorbed_ != t.can_absorb) {
        be::launch_obs_prepare(bx_, dE_, hE_, curmask_, group, minimap_mode_ ? d_mm_val_ : nullptr);
        prep_version_ = state_version_; prep_vw_ = t.view.width; prep_vh_ = t.view.height; prep_skip_absorbed_ = t.can_absorb;
    }
}

void Engine::get_observation(int group, void **bufs, int half) {      // GridWorld.cc:292-401
    check_group(group, "GridWorld::get_observation");
    to_device();
    if (!(be::is_device_ptr(bufs[0]) && be::is_device_ptr(bufs[1]))) settle_counts();    // host copies need exact sizes
    const int n = total(group);
    if (n == 0) return;
    const AgentTypeDef &t = *group_type_[group];
    const size_t esz = half ? 2 : 4;
    const size_t vbytes = (size_t)n * t.view.height * t.view.width * n_channel() * esz;
    const size_t fbytes = (size_t)n * feature_size(group) * esz;
    const bool vdev = be::is_device_ptr(bufs[0]), fdev = be::is_device_ptr(bufs[1]);
    prepare_obs(group);
    if (host_path_ < 0) {                 // MAGENT_B200_HOST_PATH=dense keeps the round-1 path (dense records over PCIe) for A/B runs
        const char *e = getenv("MAGENT_B200_HOST_PATH");                 // dense | wire (whatever the size) | default: by size
        host_path_ = (e && !strcmp(e, "dense")) ? 0 : (e && !strcmp(e, "wire")) ? 2 : 1;
    }
    // small observations (a few MB) are latency-, not bandwidth-bound: one plain copy of the dense records beats the
    // wire protocol's fixed costs (totals read-back, waves, waking the pool).  A view whose LUT the wire kernel cannot
    // hold takes the dense path whatever the setting.
    if (!vdev && !fdev && !half && (host_path_ == 2 || (host_path_ == 1 && vbytes >= ((size_t)16 << 20))) && t.view.height * t.view.width < 0xffff &&
        (long long)t.view.height * t.view.width * n_channel() < (1ll << 30) &&
        (!be::smem_fits || be::smem_fits(bx_, hE_, be::SMEM_OBS_WIRE, group, group, nullptr))) {
        get_observation_wire(group, bufs);
        return;
    }
    ObsArgs O;
    O.curmask = curmask_; O.group = group; O.half = half ? 1 : 0;
    O.grid = obs_grid_; O.chunk = obs_chunk_; O.tile = obs_tile_;
    if (vdev) O.view = bufs[0];
    else { stage_reserve(d_view_stage_, view_stage_bytes_, vbytes); O.view = d_view_stage_; }
    if (fdev) O.feature = bufs[1];
    else { stage_reserve(d_feat_stage_, feat_stage_bytes_, fbytes); O.feature = d_feat_stage_; }
    be::launch_obs(bx_, dE_, hE_, O, minimap_mode_ ? d_mm_val_ : nullptr, n);
    if (!vdev) { be::d2h(bx_, bufs[0], d_view_stage_, vbytes); io_[IO_D2H] += (long long)vbytes; }
    if (!fdev) { be::d2h(bx_, bufs[1], d_feat_stage_, fbytes); io_[IO_D2H] += (long long)fbytes; }
}

// Host buffers (the reference ABI's normal case, python/magent/gridworld.py:221-248): the GPU gathers, PCIe carries the
// compact wire records, host threads write the dense float32 bytes (host_expand.h; DESIGN.md 6b).
void Engine::get_observation_wire(int group, void **bufs) {
    const int n = total(group);
    const AgentTypeDef &t = *group_type_[group];
    const size_t fbytes = (size_t)n * feature_size(group) * 4;
    ObsArgs O;
    O.curmask = curmask_; O.group = group; O.half = 0;
    O.view = nullptr;                                                     // no dense records on the device in this path
    stage_reserve(d_feat_stage_, feat_stage_bytes_, fbytes);
    O.feature = d_feat_stage_;
    const auto t0 = std::chrono::steady_clock::now();
    be::WireDesc W;
    be::obs_wire_begin(bx_, dE_, hE_, O, minimap_mode_ ? d_mm_val_ : nullptr, n, &W);
    const auto t1 = std::chrono::steady_clock::now();
    // feature rows: DMA straight into page-locked caller memory, else through page-locked staging + a threaded copy
    const bool fpinned = be::is_pinned_host_ptr(bufs[1]);
    if (!fpinned && fbytes > h_feat_stage_bytes_) {
        if (h_feat_stage_) be::host_free(h_feat_stage_);
        h_feat_stage_bytes_ = fbytes + fbytes / 8 + 256;
        h_feat_stage_ = be::host_alloc(h_feat_stage_bytes_);
        if (!h_feat_stage_) fatal("cannot allocate %zu bytes of page-locked staging", h_feat_stage_bytes_);
    }
    be::dma_d2h_async(bx_, fpinned ? bufs[1] : h_feat_stage_, d_feat_stage_, fbytes);
    ExpandGeom g;
    memset(&g, 0, sizeof g);
    g.C = n_channel(); g.cells = t.view.height * t.view.width; g.rec = g.cells * g.C; g.G = G();
    g.minimap = minimap_mode_ ? 1 : 0;
    const int stride = 2 + (minimap_mode_ ? 1 : 0);
    for (int j = 0; j < G(); ++j) {
        int rel = j - group; if (rel < 0) rel += G();
        g.mm_ch[j] = group2channel(0) + rel * stride + 2;                 // make_channel_trans, GridWorld.cc:897-913
    }
    be::Ctx *bx = bx_;
    expand_views(g, W, (float *)bufs[0], [bx](int w) { be::obs_wire_wait(bx, w); });
    const auto t2 = std::chrono::steady_clock::now();
    be::dma_wait(bx_, 0);
    if (!fpinned) parallel_copy(bufs[1], h_feat_stage_, fbytes);
    const auto t3 = std::chrono::steady_clock::now();
    // where the host-buffer call spends its time (microseconds): producing the wire records up to the first queued copy,
    // expanding, finishing the feature rows
    io_[IO_US_WIRE] += std::chrono::duration_cast<std::chrono::microseconds>(t1 - t0).count();
    io_[IO_US_EXPAND] += std::chrono::duration_cast<std::chrono::microseconds>(t2 - t1).count();
    io_[IO_US_FEATURE] += std::chrono::duration_cast<std::chrono::microseconds>(t3 - t2).count();
    // what crossed PCIe: headers, marks, chunk table, minimap rows, feature rows; what the host threads wrote: the views
    io_[IO_D2H] += (long long)W.n_total * (long long)sizeof(be::WireHdr) + W.chunk_base[W.n_chunks] * (long long)sizeof(be::WireMark) +
                   (long long)(W.n_chunks + 1) * 8 + (W.mm ? (long long)A_ * W.mm_stride * 4 : 0) + (long long)fbytes;
    io_[IO_HOST_WRITTEN] += (long long)n * g.rec * 4 + (fpinned ? 0 : (long long)fbytes);
}

// The global state has a fixed shape, so it needs no agent counts: a device buffer takes one kernel and no host
// synchronisation (recordable into a graph).  It always covers every arena, whatever select_arena says, and leaves the
// observation pre-pass cache alone.  A host buffer goes through the device staging the dense observations use.
void Engine::get_global_state(void *buf, int half) {
    if (!be::launch_global_state) fatal("the %s backend has no global-state kernel", be::name());
    to_device();
    if (be::is_device_ptr(buf)) { be::launch_global_state(bx_, dE_, hE_, buf, half ? 1 : 0); return; }
    const size_t bytes = (size_t)A_ * H_ * W_ * state_channels() * (half ? 2 : 4);
    stage_reserve(d_view_stage_, view_stage_bytes_, bytes);
    be::launch_global_state(bx_, dE_, hE_, d_view_stage_, half ? 1 : 0);
    be::d2h(bx_, buf, d_view_stage_, bytes);
    io_[IO_D2H] += (long long)bytes;
}

// ---------------------------------------------------------------------------------------------
// reset pool (DESIGN.md §3, §5): snapshots of every arena in HBM, restored into any subset of arenas by one kernel.
// Placement stays on the host; the device only copies arena states.
bool Engine::snap_matches(const ArenaSnapshot &s, int kpad) const {
    return s.W == W_ && s.H == H_ && s.kpad == kpad && s.food_mode == food_mode_ && s.turn_mode == turn_mode_ &&
           s.types == group_type_;
}

std::vector<int> Engine::restore_floor() const {
    std::vector<int> floor(G(), 0);
    const int pad = view_pad();
    for (const ArenaSnapshot &sn : snaps_)
        if (sn.live && snap_matches(sn, pad))
            for (int g = 0; g < G(); ++g) floor[g] = std::max(floor[g], sn.max_n[g]);
    return floor;
}

void Engine::set_counts(const std::vector<int> &c) {
    for (int g = 0; g < G(); ++g)
        for (int a = 0; a < A_; ++a)
            h_off_[(size_t)g * (A_ + 1) + a + 1] = h_off_[(size_t)g * (A_ + 1) + a] + c[(size_t)g * A_ + a];
}

int Engine::num_bound(int g) const {
    const std::vector<int> floor = restore_floor();
    long long n = 0;
    for (int a = 0; a < A_; ++a) n += std::max(count(g, a), floor[g]);
    return (int)n;
}

void Engine::raise_counts(const std::vector<int> &floor) {
    std::vector<int> c((size_t)G() * A_);
    for (int g = 0; g < G(); ++g)
        for (int a = 0; a < A_; ++a) c[(size_t)g * A_ + a] = std::max(count(g, a), floor[g]);
    set_counts(c);
}

template <class T>
static void snap_copy(be::Ctx *bx, std::vector<void *> &allocs, T *&dst, const T *src, size_t n) {
    dst = (T *)be::dmalloc(bx, std::max<size_t>(n, 1) * sizeof(T));
    allocs.push_back(dst);
    be::d2d(bx, dst, src, n * sizeof(T));
}

int Engine::snapshot_arenas() {
    if (!was_reset_) return refuse("snapshot_arenas before reset");
    if (bx_ && be::capturing(bx_)) return refuse("snapshot_arenas allocates device memory: not possible while a CUDA graph is being captured");
    if (!be::launch_restore) return refuse("the %s backend has no restore kernel", be::name());
    to_device();
    settle_counts();
    const int Gn = G();
    ArenaSnapshot sn;
    sn.live = true;
    sn.W = W_; sn.H = H_; sn.kpad = hE_.kpad; sn.food_mode = food_mode_; sn.turn_mode = turn_mode_;
    sn.types = group_type_;
    sn.n.resize((size_t)Gn * A_);
    sn.max_n.assign(Gn, 0);
    for (int g = 0; g < Gn; ++g)
        for (int a = 0; a < A_; ++a) {
            sn.n[(size_t)g * A_ + a] = count(g, a);
            sn.max_n[g] = std::max(sn.max_n[g], count(g, a));
        }
    SnapDev &D = sn.dev;
    memset(&D, 0, sizeof D);
    const size_t cells = (size_t)A_ * W_ * H_, kp = (size_t)A_ * hE_.kplane;
    snap_copy(bx_, sn.allocs, D.occ, hE_.occ, cells);
    snap_copy(bx_, sn.allocs, D.kind, hE_.kind, kp);
    snap_copy(bx_, sn.allocs, D.hpn, hE_.hpn, kp);
    if (food_mode_) snap_copy(bx_, sn.allocs, D.food, hE_.food, cells);
    snap_copy(bx_, sn.allocs, D.hdr, hE_.hdr, (size_t)A_);
    snap_copy(bx_, sn.allocs, D.n, hE_.n, (size_t)Gn * A_);
    snap_copy(bx_, sn.allocs, D.dead_ct, hE_.dead_ct, (size_t)Gn * A_);
    snap_copy(bx_, sn.allocs, D.done, hE_.done, (size_t)A_);
    for (int g = 0; g < Gn; ++g) {                    // the live ping-pong buffer, at the live capacity
        const AgentSoA &L = hE_.grp[g].soa[(curmask_ >> g) & 1u];
        AgentSoA &S = D.soa[g];
        const size_t n = (size_t)A_ * cap_[g];
        D.cap[g] = cap_[g];
        snap_copy(bx_, sn.allocs, S.x, L.x, n); snap_copy(bx_, sn.allocs, S.y, L.y, n);
        snap_copy(bx_, sn.allocs, S.hp, L.hp, n); snap_copy(bx_, sn.allocs, S.act, L.act, n);
        snap_copy(bx_, sn.allocs, S.id, L.id, n);
        snap_copy(bx_, sn.allocs, S.next_reward, L.next_reward, n); snap_copy(bx_, sn.allocs, S.last_reward, L.last_reward, n);
        snap_copy(bx_, sn.allocs, S.op_obj, L.op_obj, n);
        snap_copy(bx_, sn.allocs, S.last_op, L.last_op, n); snap_copy(bx_, sn.allocs, S.flags, L.flags, n);
        snap_copy(bx_, sn.allocs, S.dir, L.dir, n);
    }
    {   // the slot table, and the id and slot counts a restore from it can bring in
        const long ld = slot_row_stride(slot_id_cap_);
        snap_copy(bx_, sn.allocs, sn.slot_tab, (const int *)d_slot_tab_, (size_t)A_ * ld);
        sn.slot_id_cap = slot_id_cap_;
        std::vector<int> tab((size_t)A_ * ld);
        be::d2h(bx_, tab.data(), d_slot_tab_, tab.size() * 4);
        std::vector<ArenaHdr> hdr(A_);
        be::d2h(bx_, hdr.data(), hE_.hdr, sizeof(ArenaHdr) * A_);
        sn.slot_max.assign(Gn, 0);
        for (int a = 0; a < A_; ++a) {
            sn.max_ids = std::max(sn.max_ids, hdr[a].id_counter);
            for (int g = 0; g < Gn; ++g) sn.slot_max[g] = std::max(sn.slot_max[g], tab[a * ld + g]);
        }
    }
    snaps_.push_back(sn);                             // ids are never reused: a freed id stays unknown
    update_slot_space();
    return (int)snaps_.size() - 1;
}

int Engine::free_snapshot(int id) {
    if (id < 0 || id >= (int)snaps_.size() || !snaps_[id].live) return refuse("unknown or freed snapshot id %d", id);
    ArenaSnapshot &sn = snaps_[id];
    if (sn.in_graph) return refuse("snapshot %d is restored from inside a recorded CUDA graph: it lives as long as the game", id);
    if (be::capturing(bx_)) return refuse("free_snapshot is not possible while a CUDA graph is being captured");
    for (void *p : sn.allocs) be::dfree(bx_, p);
    sn = ArenaSnapshot();
    update_slot_space();
    return 0;
}

// Counts: the host's h_off_ must stay an upper bound of the device's counts (every count-sized launch relies on it).
// A host src gives the new counts exactly.  A device src or the done flags are only known on the device: every arena's
// bound is raised to the snapshot's largest count and the exact counts are fetched asynchronously, as clear_dead does;
// inside a capture they are marked unknown.
int Engine::restore_arenas(int id, const int *src, int keep_rng) {
    if (id < 0 || id >= (int)snaps_.size() || !snaps_[id].live) return refuse("unknown or freed snapshot id %d", id);
    ArenaSnapshot &sn = snaps_[id];
    if (!order_.empty()) return refuse("restore_arenas while actions are set for the current step (call env_step first)");
    if (!first_render_) return refuse("restore_arenas while rendering is not supported");
    if (!snap_matches(sn, view_pad()))
        return refuse("snapshot %d was taken under a different geometry (map size, groups, agent types, food_mode or turn_mode)", id);
    if (!be::launch_restore) return refuse("the %s backend has no restore kernel", be::name());
    const bool capturing = bx_ && be::capturing(bx_);
    const bool dev_src = src != nullptr && be::is_device_ptr(src);
    if (src && !dev_src) {
        if (capturing) return refuse("restore_arenas with a host src cannot be recorded into a CUDA graph");
        for (int a = 0; a < A_; ++a)
            if (src[a] < -1 || src[a] >= A_) return refuse("restore_arenas: src[%d] = %d is outside [-1, %d)", a, src[a], A_);
    }
    to_device();
    const int *d_src = src;
    if (src && !dev_src) {
        settle_counts();
        int *st = (int *)io_stage((size_t)A_ * 4);
        be::h2d(bx_, st, src, (size_t)A_ * 4);
        io_[IO_H2D] += (long long)A_ * 4;
        d_src = st;
    }
    // the slot rows and the recorders' episodes first: launch_restore rewrites the done words a null src decides by
    if (live_replays()) be::launch_replay_restore(bx_, hE_, d_rep_, d_src);
    if (be::launch_restore_slots) be::launch_restore_slots(bx_, dE_, hE_, d_slot_dev_, sn.slot_tab, sn.slot_id_cap, d_src);
    be::launch_restore(bx_, dE_, hE_, curmask_, sn.dev, d_src, keep_rng ? 1 : 0);
    ++state_version_;
    may_have_dead_ = true;
    done_stale_ = true;
    if (capturing) sn.in_graph = true;
    if (src && !dev_src) {
        std::vector<int> c((size_t)G() * A_);
        for (int g = 0; g < G(); ++g)
            for (int a = 0; a < A_; ++a) c[(size_t)g * A_ + a] = src[a] >= 0 ? sn.n[(size_t)g * A_ + src[a]] : count(g, a);
        set_counts(c);
        return 0;
    }
    raise_counts(sn.max_n);
    if (capturing) { counts_unknown_ = true; return 0; }
    be::counts_fetch_begin(bx_, hE_.off, h_off_.size());
    counts_pending_ = true;
    counts_unknown_ = false;
    return 0;
}

int Engine::get_arena_done(int *out) {
    if (be::is_device_ptr(out)) {
        if (!be::launch_arena_done) return refuse("the %s backend has no arena-done kernel", be::name());
        to_device();
        be::launch_arena_done(bx_, dE_, hE_, out);
        return 0;
    }
    get_info(-1, "arena_done", out);
    return 0;
}

void Engine::set_action(int group, const int *actions) {              // GridWorld.cc:403-454
    check_group(group, "GridWorld::set_action");
    to_device();
    if (!be::is_device_ptr(actions)) settle_counts();
    const int n = total(group);
    if (std::find(order_.begin(), order_.end(), group) == order_.end()) order_.push_back(group);
    if (n == 0) return;
    const void *src = actions;
    if (!be::is_device_ptr(actions)) {
        void *st = io_stage((size_t)n * 4);
        be::h2d(bx_, st, actions, (size_t)n * 4);
        io_[IO_H2D] += (long long)n * 4;
        src = st;
    }
    be::launch_info(bx_, dE_, hE_, curmask_, INFO_ACTION_SCATTER, group, const_cast<void *>(src), n);
}

void Engine::random_actions(int group, unsigned long long seed) {
    check_group(group, "random_actions");
    to_device();
    if (std::find(order_.begin(), order_.end(), group) == order_.end()) order_.push_back(group);
    const int n = total(group);
    if (n == 0) return;
    be::launch_random_actions(bx_, dE_, hE_, curmask_, group, seed * 0x9E3779B97F4A7C15ull + (++rand_calls_), n);
}

// Legal-action mask of one group
int Engine::get_action_mask(int group, unsigned char *buf) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_action_mask", group);
    if (!be::launch_action_mask) return refuse("the %s backend has no action-mask kernel", be::name());
    to_device();
    if (smem_refused(bx_, hE_, be::SMEM_ACTION_MASK, group, group, "get_action_mask")) return -1;
    const bool dev = be::is_device_ptr(buf);
    if (!dev) settle_counts();
    const int n = total(group);
    read_back(dev, {{buf, (size_t)n * group_type_[group]->n_action}}, [&](void **to) {
        be::launch_action_mask(bx_, dE_, hE_, curmask_, group, (unsigned char *)to[0], n);
    });
    return 0;
}

int Engine::random_legal_actions(int group, unsigned long long seed) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in random_legal_actions", group);
    if (!be::launch_random_legal_actions) return refuse("the %s backend has no legal-action sampler", be::name());
    to_device();
    if (std::find(order_.begin(), order_.end(), group) == order_.end()) order_.push_back(group);
    const int n = total(group);
    if (n == 0) return 0;
    // the seed the kernel sees (mask_phases.h legal_draw): shares the call counter of random_actions
    be::launch_random_legal_actions(bx_, dE_, hE_, curmask_, group, seed * 0x9E3779B97F4A7C15ull + (++rand_calls_), n);
    return 0;
}

// Mean neighbour action of one group over the agents of group `of` it sees
int Engine::get_mean_action(int group, int of, float *mean, int *count) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_mean_action", group);
    if (of < 0 || of >= G()) return refuse("invalid group handle %d for `of` in get_mean_action", of);
    if (!be::launch_mean_action) return refuse("the %s backend has no mean-action kernel", be::name());
    const int mem = out_memory("get_mean_action: mean and count", {mean, count});
    if (mem < 0) return -1;
    const bool dev = mean && mem;       // a null mean counts as host memory (refused below unless the group is empty)
    to_device();
    if (smem_refused(bx_, hE_, be::SMEM_MEAN_ACTION, group, of, "get_mean_action")) return -1;
    if (!dev) settle_counts();
    const int n = total(group);
    if (n == 0) return 0;
    if (!mean) return refuse("get_mean_action needs a mean buffer");
    read_back(dev, {{mean, (size_t)n * group_type_[of]->n_action * 4}, {count, (size_t)n * 4}}, [&](void **to) {
        be::launch_mean_action(bx_, dE_, hE_, curmask_, group, of, (float *)to[0], (int *)to[1], n);
    });
    return 0;
}

// The first k neighbours of one group in group `of`, nearest first
int Engine::get_neighbours(int group, int of, int k, int *idx, int *rel, int *count) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_neighbours", group);
    if (of < 0 || of >= G()) return refuse("invalid group handle %d for `of` in get_neighbours", of);
    if (k < 1 || k > 32) return refuse("get_neighbours: k = %d is outside [1, 32]", k);
    if (!idx) return refuse("get_neighbours needs an idx buffer");
    if (!be::launch_neighbours) return refuse("the %s backend has no neighbours kernel", be::name());
    const int mem = out_memory("get_neighbours: idx, rel and count", {idx, rel, count});
    if (mem < 0) return -1;
    to_device();
    if (!nbr_key_fits_[group])
        return refuse("get_neighbours: the view of group %d is too large to order its cells by an int key", group);
    if (!mem) settle_counts();
    const int n = total(group);
    const size_t idx_bytes = (size_t)n * k * 4;
    read_back(mem == 1, {{idx, idx_bytes}, {rel, 2 * idx_bytes}, {count, (size_t)n * 4}}, [&](void **to) {
        be::launch_neighbours(bx_, dE_, hE_, d_nbr_lut_ + nbr_lut_base_[group], curmask_, group, of, k, (int *)to[0],
                              (int *)to[1], (int *)to[2], n);
    });
    return 0;
}

// The stable slots of one group
int Engine::get_slots(int group, int *row_slot, int *slot_row) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_slots", group);
    if (!row_slot && !slot_row) return refuse("get_slots needs a row_slot or a slot_row buffer");
    if (!be::launch_slots || !be::launch_restore_slots) return refuse("the %s backend has no slots kernel", be::name());
    const int mem = out_memory("get_slots: row_slot and slot_row", {row_slot, slot_row});
    if (mem < 0) return -1;
    to_device();
    if (!mem) settle_counts();
    const int S = group < (int)slot_space_.size() ? slot_space_[group] : 0, nb = num_bound(group);
    read_back(mem == 1, {{row_slot, (size_t)nb * 4}, {slot_row, (size_t)A_ * S * 4}}, [&](void **to) {
        be::launch_slots(bx_, dE_, hE_, d_slot_dev_, curmask_, group, S, (int *)to[0], (int *)to[1], nb);
    });
    return 0;
}

// The observation of one group in slot order, [A][S] records and feature rows.  Its shape needs no counts (the device
// decides which slots hold rows), so neither pointer kind waits for them.  Device buffers: no staging, allocation or
// synchronisation once warm.  Host buffers: through the device staging of the dense observations, copied back.
int Engine::get_observation_slots(int group, void **bufs, int half) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_observation_slots", group);
    if (half != 0 && half != 1) return refuse("get_observation_slots: half must be 0 or 1, not %d", half);
    if (!bufs || !bufs[0] || !bufs[1]) return refuse("get_observation_slots needs a view and a feature buffer");
    if (!be::launch_obs_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered observation kernel", be::name());
    const int mem = out_memory("get_observation_slots: view and feature", {bufs[0], bufs[1]});
    if (mem < 0) return -1;
    to_device();
    const int S = group < (int)slot_space_.size() ? slot_space_[group] : 0;
    if (S == 0) return 0;
    const AgentTypeDef &t = *group_type_[group];
    const size_t esz = half ? 2 : 4, n = (size_t)A_ * S;
    const size_t vbytes = n * t.view.height * t.view.width * n_channel() * esz, fbytes = n * feature_size(group) * esz;
    prepare_obs(group);
    ObsArgs O;
    O.curmask = curmask_; O.group = group; O.half = half;
    O.grid = obs_grid_; O.chunk = obs_chunk_; O.tile = obs_tile_;
    if (mem == 1) {
        O.view = bufs[0]; O.feature = bufs[1];
    } else {
        stage_reserve(d_view_stage_, view_stage_bytes_, vbytes); O.view = d_view_stage_;
        stage_reserve(d_feat_stage_, feat_stage_bytes_, fbytes); O.feature = d_feat_stage_;
    }
    be::launch_obs_slots(bx_, dE_, hE_, d_slot_dev_, O, minimap_mode_ ? d_mm_val_ : nullptr, S);
    if (mem == 0) {
        be::d2h(bx_, bufs[0], d_view_stage_, vbytes); io_[IO_D2H] += (long long)vbytes;
        be::d2h(bx_, bufs[1], d_feat_stage_, fbytes); io_[IO_D2H] += (long long)fbytes;
    }
    return 0;
}

// The slot-ordered step loop.  [A][S] is known on the host and the device decides which slots hold rows, so none of the
// three calls waits for the counts; with CUDA pointers they neither synchronise nor allocate (the mask once warm).

// set_action in slot order: every row below the device-side count takes act[its slot].  It is the group's set_action
// for this step, registered in order_ as set_action registers it, once nothing can refuse the call any more.
int Engine::set_action_slots(int group, const int *act) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in set_action_slots", group);
    if (!be::launch_set_action_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered action kernel", be::name());
    const int S = slot_space(group);
    if (S > 0 && !act) return refuse("set_action_slots needs an action buffer");
    to_device();
    if (std::find(order_.begin(), order_.end(), group) == order_.end()) order_.push_back(group);
    if (S == 0) return 0;
    const void *src = act;
    if (!be::is_device_ptr(act)) {
        const size_t bytes = (size_t)A_ * S * 4;
        void *st = io_stage(bytes);
        be::h2d(bx_, st, act, bytes);
        io_[IO_H2D] += (long long)bytes;
        src = st;
    }
    be::launch_set_action_slots(bx_, dE_, hE_, d_slot_dev_, curmask_, group, S, (const int *)src);
    return 0;
}

// env_get_reward and the alive flag in slot order: float [A][S] and uint8 [A][S] (0 vacant, 1 alive, 2 dead)
int Engine::get_reward_slots(int group, float *reward, unsigned char *status) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_reward_slots", group);
    if (!reward && !status) return refuse("get_reward_slots needs a reward or a status buffer");
    if (!be::launch_reward_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered reward kernel", be::name());
    const int mem = out_memory("get_reward_slots: reward and status", {reward, status});
    if (mem < 0) return -1;
    to_device();
    const int S = slot_space(group);
    const size_t n = (size_t)A_ * S;
    read_back(mem == 1, {{reward, n * 4}, {status, n}}, [&](void **to) {
        be::launch_reward_slots(bx_, dE_, hE_, d_slot_dev_, curmask_, group, S, (float *)to[0], (unsigned char *)to[1]);
    });
    return 0;
}

// The legal-action mask in slot order: uint8 [A][S][n_action]
int Engine::get_action_mask_slots(int group, unsigned char *mask) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_action_mask_slots", group);
    if (!mask) return refuse("get_action_mask_slots needs a mask buffer");
    if (!be::launch_action_mask_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered action-mask kernel", be::name());
    const int mem = out_memory("get_action_mask_slots: mask", {mask});
    to_device();
    if (smem_refused(bx_, hE_, be::SMEM_ACTION_MASK_SLOTS, group, group, "get_action_mask_slots")) return -1;
    const int S = slot_space(group);
    read_back(mem == 1, {{mask, (size_t)A_ * S * group_type_[group]->n_action}}, [&](void **to) {
        be::launch_action_mask_slots(bx_, dE_, hE_, d_slot_dev_, curmask_, group, S, (unsigned char *)to[0]);
    });
    return 0;
}

// The mean neighbour action in slot order: float [A][S][n_action(of)] and int [A][S], zero in vacant slots
int Engine::get_mean_action_slots(int group, int of, float *mean, int *count) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_mean_action_slots", group);
    if (of < 0 || of >= G()) return refuse("invalid group handle %d for `of` in get_mean_action_slots", of);
    if (!mean) return refuse("get_mean_action_slots needs a mean buffer");
    if (!be::launch_mean_action_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered mean-action kernel", be::name());
    const int mem = out_memory("get_mean_action_slots: mean and count", {mean, count});
    if (mem < 0) return -1;
    to_device();
    if (smem_refused(bx_, hE_, be::SMEM_MEAN_ACTION_SLOTS, group, of, "get_mean_action_slots")) return -1;
    const int S = slot_space(group);
    const size_t n = (size_t)A_ * S;
    read_back(mem == 1, {{mean, n * group_type_[of]->n_action * 4}, {count, n * 4}}, [&](void **to) {
        be::launch_mean_action_slots(bx_, dE_, hE_, d_slot_dev_, curmask_, group, of, S, (float *)to[0], (int *)to[1]);
    });
    return 0;
}

// The first k neighbours in slot order: int [A][S][k] flat slots a * S_of + slot of `of`, int [A][S][k][2] view cells
// and int [A][S] counts, -1 and 0 in vacant slots
int Engine::get_neighbours_slots(int group, int of, int k, int *idx, int *rel, int *count) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in get_neighbours_slots", group);
    if (of < 0 || of >= G()) return refuse("invalid group handle %d for `of` in get_neighbours_slots", of);
    if (k < 1 || k > 32) return refuse("get_neighbours_slots: k = %d is outside [1, 32]", k);
    if (!idx) return refuse("get_neighbours_slots needs an idx buffer");
    if (!be::launch_neighbours_slots || !be::launch_restore_slots)
        return refuse("the %s backend has no slot-ordered neighbours kernel", be::name());
    const int mem = out_memory("get_neighbours_slots: idx, rel and count", {idx, rel, count});
    if (mem < 0) return -1;
    to_device();
    if (!nbr_key_fits_[group])
        return refuse("get_neighbours_slots: the view of group %d is too large to order its cells by an int key", group);
    const int S = slot_space(group);
    const size_t n = (size_t)A_ * S, idx_bytes = n * k * 4;
    read_back(mem == 1, {{idx, idx_bytes}, {rel, 2 * idx_bytes}, {count, n * 4}}, [&](void **to) {
        be::launch_neighbours_slots(bx_, dE_, hE_, d_slot_dev_, d_nbr_lut_ + nbr_lut_base_[group], curmask_, group, of,
                                    k, S, slot_space(of), (int *)to[0], (int *)to[1], (int *)to[2]);
    });
    return 0;
}

// The built-in scripted opponent.  The fallback draws as random_legal_actions would if it were called next: the seed it
// would see, without counting as one of its calls, so that the three variants agree and leave the draws of
// random_actions / random_legal_actions as they were.
bool Engine::rule_refused(int group, int target, int policy, bool slots, const char *what) {
    if (group < 0 || group >= G()) return refuse("invalid group handle %d in %s", group, what) < 0;
    if (target < 0 || target >= G()) return refuse("invalid group handle %d for `target` in %s", target, what) < 0;
    if (policy != RULE_RUSH && policy != RULE_FLEE)
        return refuse("%s: policy %d is neither rush (%d) nor flee (%d)", what, policy, RULE_RUSH, RULE_FLEE) < 0;
    if (slots ? !be::launch_rule_actions_slots || !be::launch_restore_slots : !be::launch_rule_actions)
        return refuse("the %s backend has no %srule-action kernel", be::name(), slots ? "slot-ordered " : "") < 0;
    to_device();
    if (!nbr_key_fits_[group])
        return refuse("%s: the view of group %d is too large to order its cells by an int key", what, group) < 0;
    return false;
}

int Engine::rule_actions(int group, int target, int policy, unsigned long long seed) {
    if (rule_refused(group, target, policy, false, "rule_actions")) return -1;
    if (std::find(order_.begin(), order_.end(), group) == order_.end()) order_.push_back(group);
    const int n = total(group);
    if (n == 0) return 0;
    be::launch_rule_actions(bx_, dE_, hE_, d_nbr_lut_ + nbr_lut_base_[group], curmask_, group, target, policy,
                            seed * 0x9E3779B97F4A7C15ull + rand_calls_ + 1, nullptr, n);
    return 0;
}

int Engine::get_rule_actions(int group, int target, int policy, unsigned long long seed, int *act) {
    if (rule_refused(group, target, policy, false, "get_rule_actions")) return -1;
    const bool dev = be::is_device_ptr(act);
    if (!dev) settle_counts();
    const int n = total(group);
    if (n > 0 && !act) return refuse("get_rule_actions needs an action buffer");
    read_back(dev, {{act, (size_t)n * 4}}, [&](void **to) {
        be::launch_rule_actions(bx_, dE_, hE_, d_nbr_lut_ + nbr_lut_base_[group], curmask_, group, target, policy,
                                seed * 0x9E3779B97F4A7C15ull + rand_calls_ + 1, (int *)to[0], n);
    });
    return 0;
}

int Engine::get_rule_actions_slots(int group, int target, int policy, unsigned long long seed, int *act) {
    if (rule_refused(group, target, policy, true, "get_rule_actions_slots")) return -1;
    const int S = slot_space(group);
    if (S > 0 && !act) return refuse("get_rule_actions_slots needs an action buffer");
    read_back(be::is_device_ptr(act), {{act, (size_t)A_ * S * 4}}, [&](void **to) {
        be::launch_rule_actions_slots(bx_, dE_, hE_, d_slot_dev_, d_nbr_lut_ + nbr_lut_base_[group], curmask_, group,
                                      target, policy, seed * 0x9E3779B97F4A7C15ull + rand_calls_ + 1, S, (int *)to[0]);
    });
    return 0;
}

void Engine::step(int *done) {                                        // GridWorld.cc:456-631
    to_device();
    StepArgs S;
    memset(&S, 0, sizeof S);
    S.curmask = curmask_;
    // GridWorld.cc:484: only once rendering has started, or while a replay recorder is live
    const bool replaying = live_replays() > 0;
    S.record_events = first_render_ && !replaying ? 0 : 1;
    S.n_order = (int)order_.size();
    for (int k = 0; k < S.n_order; ++k) S.order[k] = order_[k];
    be::launch_step(bx_, dE_, hE_, S, max_agents_per_arena());
    // the recorded arenas' events, before a cull renumbers the rows (an event list sized for another cap_total is left
    // alone: replay_record refuses then)
    if (replaying && hE_.cap_total == ev_stride_)
        be::launch_replay_events(bx_, dE_, hE_, curmask_, d_rep_, d_ev_, d_ev_arenas_, n_ev_arenas_);
    ++state_version_;
    order_.clear();
    if (be::is_device_ptr(done)) {
        // device-resident caller: the done word goes to its device int, nothing is read back and the host does not
        // wait for the step.  The host then cannot know whether anybody died: the next clear_dead re-reads the counts.
        be::launch_done_to_device(bx_, dE_, hE_, done);
        may_have_dead_ = true;
        done_stale_ = true;
        if (!first_render_) collect_attack_events();
        return;
    }
    std::vector<int> d(A_);
    be::read_done(bx_, hE_, d.data());
    io_[IO_D2H] += (long long)A_ * 4;
    done_stale_ = false;
    int all = 1;
    for (int a = 0; a < A_; ++a) { arenas_[a].done = d[a] & 1; all &= arenas_[a].done; may_have_dead_ |= (d[a] & 2) != 0; }
    *done = all;
    if (!first_render_) collect_attack_events();
}

void Engine::get_reward(int group, float *buf) {                      // GridWorld.cc:694-704
    check_group(group, "GridWorld::get_reward");
    to_device();
    const bool dev = be::is_device_ptr(buf);
    if (!dev) settle_counts();
    const int n = total(group);
    read_back(dev, {{buf, (size_t)n * 4}}, [&](void **to) {
        be::launch_info(bx_, dE_, hE_, curmask_, INFO_REWARD, group, to[0], n);
    });
}

void Engine::clear_dead() {                                           // GridWorld.cc:633-665
    to_device();
    settle_counts();                                  // a fetch still pending from the previous cull is long finished
    be::launch_cull(bx_, dE_, hE_, curmask_, max_agents_per_arena());
    ++state_version_;
    curmask_ ^= (1u << G()) - 1u;
    if (!may_have_dead_) return;                      // nobody died since the last cull: counts and offsets stand
    may_have_dead_ = false;
    // the new counts come back asynchronously: the call does not wait for the cull.  Until somebody needs exact
    // numbers (settle_counts), h_off_ holds the previous counts -- upper bounds, since a cull only removes agents --
    // and the kernels clamp to the device-side totals (EngineDev::off).
    be::launch_offsets(bx_, dE_, hE_);
    if (be::capturing(bx_)) { ++capture_culls_; counts_unknown_ = true; return; }      // no read-back inside a graph
    be::counts_fetch_begin(bx_, hE_.off, h_off_.size());
    counts_pending_ = true;
}

void Engine::settle_counts() {
    if (counts_unknown_ && !be::capturing(bx_)) {     // graphs advanced the state: read the offset table the last cull left
        counts_unknown_ = false;
        counts_pending_ = false;
        be::d2h(bx_, h_off_.data(), hE_.off, h_off_.size() * 4);
        io_[IO_D2H] += (long long)h_off_.size() * 4;
        return;
    }
    if (!counts_pending_) return;
    memcpy(h_off_.data(), be::counts_fetch_wait(bx_), h_off_.size() * sizeof(int));
    io_[IO_D2H] += (long long)h_off_.size() * 4;
    counts_pending_ = false;
}

void Engine::set_goal(int group, const char *method, const int *) {                  // GridWorld.cc:667-679 (deprecated)
    // Each agent of the group draws a goal position from the engine RNG.  Nothing in the reference ever reads
    // Agent::goal (the two goal_mode feature slots are never written), so the observable effect is exactly the
    // two draws per agent the RNG stream advances by.
    check_group(group, "GridWorld::set_goal");
    if (!strequ(method, "random")) fatal("invalid goal type in GridWorld::set_goal");
    if (!was_reset_) fatal("set_goal before reset");
    if (where_ == DEVICE) to_host(false);
    for (int a = 0; a < A_; ++a) {
        if (sel_arena_ >= 0 && sel_arena_ != a) continue;
        HostArena &ar = arenas_[a];
        for (int i = 0, n = ar.groups[group].size(); i < n; ++i) { rng_next(ar.rng); rng_next(ar.rng); }
    }
}

// ---------------------------------------------------------------------------------------------
// replay dump for the reference viewer (RenderGenerator.cc:63-185).  Cold path: works on a host snapshot of the
// selected arena (arena 0 by default); byte-identical files for identical runs.
void Engine::collect_attack_events() {                // the list GridWorld::step hands to the RenderGenerator (:471-509)
    settle_counts();
    const int a = sel_arena_ >= 0 ? sel_arena_ : 0;
    struct Ev { int rank, id, x, y; };
    std::vector<Ev> evs;
    for (int g = 0; g < G(); ++g) {
        const int n = count(g, a);
        if (n == 0) continue;
        const AgentTypeDef &t = *group_type_[g];
        const AgentSoA &s = hE_.grp[g].soa[(curmask_ >> g) & 1u];
        const size_t base = (size_t)a * cap_[g];
        std::vector<int> rank(n), x(n), y(n), act(n), id(n);
        be::d2h(bx_, rank.data(), hE_.grp[g].ev_rank + base, (size_t)n * 4);
        be::d2h(bx_, x.data(), s.x + base, (size_t)n * 4); be::d2h(bx_, y.data(), s.y + base, (size_t)n * 4);
        be::d2h(bx_, act.data(), s.act + base, (size_t)n * 4); be::d2h(bx_, id.data(), s.id + base, (size_t)n * 4);
        std::vector<unsigned char> dir(n, (unsigned char)DIR_NORTH);
        if (turn_mode_) be::d2h(bx_, dir.data(), s.dir + base, (size_t)n);
        for (int i = 0; i < n; ++i) {
            if (rank[i] < 0) continue;
            const int k = act[i] - t.attack_base;
            // an attacker neither moves nor turns in the step it attacks
            Ev e = {rank[i], id[i], 0, 0};
            replay_event_cell(hE_.grp[g], dir[i], x[i], y[i], t.att_x_offset + t.attack.dx[k], t.att_y_offset + t.attack.dy[k],
                              e.x, e.y);
            evs.push_back(e);
        }
    }
    std::sort(evs.begin(), evs.end(), [](const Ev &p, const Ev &q) { return p.rank < q.rank; });
    attack_events_.clear();
    for (const Ev &e : evs) attack_events_.push_back({e.id, e.x, e.y});
}

void Engine::render_next_file() { file_ct_++; frame_ct_ = 0; }

namespace {
template <typename T> void print_json(std::ostream &os, const char *key, T value, bool last = false) {
    os << "\"" << key << "\": " << value;
    os << (last ? "\n" : ",\n");
}
std::string rgba_string(int r, int g, int b, float alpha) {
    std::stringstream ss;
    ss << "\"rgba(" << r << "," << g << "," << b << "," << alpha << ")\"";
    return ss.str();
}
}  // namespace

void Engine::write_render_config(std::ostream &f) const {             // RenderGenerator::gen_config
    static const int colors[][3] = {{192, 64, 64}, {64, 64, 192}, {64, 192, 64}, {64, 64, 64}};
    f << "{\n";
    print_json(f, "width", W_);
    print_json(f, "height", H_);
    print_json(f, "static-file", "\"static.map\"");
    print_json(f, "obstacle-style", rgba_string(127, 127, 127, 1));
    print_json(f, "dynamic-file-directory", "\".\"");
    print_json(f, "attack-style", rgba_string(63, 63, 63, 0.8));
    print_json(f, "minimap-width", 300);
    print_json(f, "minimap-height", 250);
    f << "\"group\" : [\n";
    for (int i = 0; i < G(); i++) {
        const AgentTypeDef &t = *group_type_[i];
        const int *c = colors[i % 4];
        f << "{\n";
        print_json(f, "height", t.length);
        print_json(f, "width", t.width);
        print_json(f, "style", rgba_string(c[0], c[1], c[2], 1));
        print_json(f, "anchor", "[0, 0]");
        print_json(f, "max-speed", (int)t.speed);
        print_json(f, "speed-style", rgba_string(c[0], c[1], c[2], 0.01));
        print_json(f, "vision-radius", t.view_radius);
        print_json(f, "vision-angle", t.view_angle);
        print_json(f, "vision-style", rgba_string(c[0], c[1], c[2], 0.2));
        print_json(f, "attack-radius", t.attack_radius);
        print_json(f, "attack-angle", t.attack_angle);
        print_json(f, "attack-style", rgba_string(c[0], c[1], c[2], 0.1));
        print_json(f, "broadcast-radius", 1, true);
        f << (i == G() - 1 ? "}" : "},") << "\n";
    }
    f << "]\n}\n";
}

void Engine::write_render_frame(std::ostream &fout, const std::vector<int> *walls,       // RenderGenerator::render_a_frame
                                const std::vector<std::vector<RepAgent>> &agents,
                                const std::vector<AttackEvent> &events) const {
    if (walls) {
        fout << "W" << " " << walls->size() << "\n";
        for (int w : *walls) fout << w % W_ << " " << w / W_ << "\n";
    }
    int num_agents = 0;
    for (int g = 0; g < G(); g++) {
        num_agents += (int)agents[g].size();
        if (group_type_[g]->can_absorb)
            for (const RepAgent &r : agents[g]) if (!(r.dir_flags & (FLAG_ABSORBED << 8))) num_agents--;
    }
    fout << "F" << " " << num_agents << " " << (int)events.size() << " " << 0 << "\n";
    static const int dir2angle[] = {0, 90, 180, 270};
    for (int g = 0; g < G(); g++) {
        const AgentTypeDef &t = *group_type_[g];
        for (const RepAgent &r : agents[g]) {
            if (t.can_absorb && !(r.dir_flags & (FLAG_ABSORBED << 8))) continue;
            int hp = std::max(0, int(100 * r.hp / t.hp));
            hp = std::min(hp, 100);
            fout << r.id << " " << hp << " " << dir2angle[r.dir_flags & 3] << " " << r.x << " " << r.y << " " << g << "\n";
        }
    }
    for (const AttackEvent &e : events) fout << 0 << " " << e.id << " " << e.x << " " << e.y << "\n";
}

void Engine::render() {                               // GridWorld.cc:939-949
    if (render_dir_ == "___debug___") return;         // terminal dump of the reference's debug mode: not provided
    if (first_render_) {
        first_render_ = false;
        std::ofstream f(render_dir_ + "/" + "config.json");
        write_render_config(f);
    }
    if (render_dir_.empty()) return;
    if (was_reset_ && where_ == DEVICE) to_host(true);
    const HostArena &ar = arenas_[sel_arena_ >= 0 ? sel_arena_ : 0];
    std::ofstream fout(render_dir_ + "/" + "video_" + std::to_string(file_ct_) + ".txt",
                       frame_ct_ == 0 ? std::ios::out : std::ios::app);
    std::vector<int> walls;
    if (frame_ct_ == 0)
        for (int i = 0; i < W_ * H_; i++) if (ar.occ[i] == OCC_WALL) walls.push_back(i);
    std::vector<std::vector<RepAgent>> agents(G());
    for (int g = 0; g < G(); g++) {
        const HostGroup &hg = ar.groups[g];
        for (int j = 0; j < hg.size(); j++)
            agents[g].push_back({hg.id[j], hg.x[j], hg.y[j], hg.hp[j], (hg.dir[j] & 3) | (hg.flags[j] & FLAG_ABSORBED ? FLAG_ABSORBED << 8 : 0)});
    }
    write_render_frame(fout, frame_ct_ == 0 ? &walls : nullptr, agents, attack_events_);
    if (frame_ct_++ > frame_per_file_) { frame_ct_ = 0; file_ct_++; }
}

// ---------------------------------------------------------------------------------------------
// replay recorders (replay_phases.h): frames of chosen arenas gathered on the device without synchronisation or
// allocation, so that recording can sit inside a captured step loop; replay_write formats them as env_render would.
int Engine::live_replays() const {
    int n = 0;
    for (const ReplayRec &r : replays_) n += r.live ? 1 : 0;
    return n;
}

// the arenas whose attack events the step collects: the union of the live recorders' (read by the event kernel from
// device memory, so a captured step sees the set shrink when a recorder outside the graph is freed)
void Engine::update_ev_arenas() {
    std::vector<int> list(A_, -1);
    std::vector<char> in(A_, 0);
    n_ev_arenas_ = 0;
    for (const ReplayRec &r : replays_)
        if (r.live)
            for (int a : r.arenas) if (!in[a]) { in[a] = 1; list[n_ev_arenas_++] = a; }
    be::h2d(bx_, d_ev_arenas_, list.data(), (size_t)A_ * 4);
}

int Engine::replay_new(const int *arenas, int n_arenas, int max_frames) {
    if (bx_ && be::capturing(bx_)) return refuse("replay_new allocates device memory: not possible while a CUDA graph is being captured");
    if (graph_captured_)
        return refuse("replay_new after this game captured a CUDA graph: steps captured without a live recorder do not record "
                      "attack events, so create recorders before capturing");
    if (!was_reset_) return refuse("replay_new before reset");
    if (!be::launch_replay_events || !be::launch_replay_restore || !be::launch_replay_record)
        return refuse("the %s backend has no replay kernels", be::name());
    if (!arenas || n_arenas < 1) return refuse("replay_new: the arena list is empty");
    if (max_frames < 1) return refuse("replay_new: max_frames = %d, must be >= 1", max_frames);
    std::vector<char> seen(A_, 0);
    for (int k = 0; k < n_arenas; ++k) {
        const int a = arenas[k];
        if (a < 0 || a >= A_) return refuse("replay_new: arena %d is outside [0, %d)", a, A_);
        if (seen[a]) return refuse("replay_new: arena %d is listed twice", a);
        seen[a] = 1;
    }
    to_device();
    ReplayRec r;
    r.arenas.assign(arenas, arenas + n_arenas);
    r.max_frames = max_frames;
    r.cap = cap_;
    r.W = W_; r.H = H_;
    r.L.cap_total = hE_.cap_total;
    r.L.wall_words = (int)(((long)W_ * H_ + 127) / 128 * 4);      // a multiple of 4: every frame block starts 16-byte aligned
    r.file_ct.assign(n_arenas, 0);
    r.frame_ct.assign(n_arenas, 0);
    r.walls.assign(n_arenas, {});
    const size_t frame_bytes = (size_t)r.L.frame_ints() * 4;
    r.frames = (int *)be::dmalloc(bx_, frame_bytes * n_arenas * max_frames);
    r.d_arenas = (int *)be::dmalloc(bx_, (size_t)n_arenas * 4);
    be::h2d(bx_, r.d_arenas, arenas, (size_t)n_arenas * 4);
    r.last_ep = (int *)be::dmalloc(bx_, (size_t)n_arenas * 4);
    be::dmemset(bx_, r.last_ep, 0xff, (size_t)n_arenas * 4);      // -1: no frame yet (episodes count up from 0)
    r.ctl = (RepCtl *)be::dmalloc(bx_, sizeof(RepCtl));
    be::dmemset(bx_, r.ctl, 0, sizeof(RepCtl));
    if (!d_rep_) {
        d_rep_ = (RepArena *)be::dmalloc(bx_, sizeof(RepArena) * A_);
        be::dmemset(bx_, d_rep_, 0, sizeof(RepArena) * A_);
        d_ev_arenas_ = (int *)be::dmalloc(bx_, (size_t)A_ * 4);
    }
    // no events are known until the next step when none were being collected, or for a list of another width
    if (!live_replays() || ev_stride_ != hE_.cap_total) {
        if (ev_stride_ != hE_.cap_total) {
            if (d_ev_) be::dfree(bx_, d_ev_);
            ev_stride_ = hE_.cap_total;
            d_ev_ = (RepEvent *)be::dmalloc(bx_, sizeof(RepEvent) * std::max<size_t>((size_t)A_ * ev_stride_, 1));
        }
        std::vector<RepArena> rep(A_);
        be::d2h(bx_, rep.data(), d_rep_, sizeof(RepArena) * A_);
        for (RepArena &x : rep) for (int &n : x.ev_n) n = 0;
        be::h2d(bx_, d_rep_, rep.data(), sizeof(RepArena) * A_);
    }
    r.live = true;
    replays_.push_back(r);                            // ids are never reused: a freed id stays unknown
    update_ev_arenas();
    return (int)replays_.size() - 1;
}

int Engine::replay_record(int id) {
    if (id < 0 || id >= (int)replays_.size() || !replays_[id].live) return refuse("unknown or freed replay id %d", id);
    ReplayRec &r = replays_[id];
    to_device();
    if (r.cap != cap_ || r.L.cap_total != hE_.cap_total || ev_stride_ != hE_.cap_total || r.W != W_ || r.H != H_)
        return refuse("replay_record: the per-arena agent bound grew past what replay %d's frames were sized for "
                      "(create a new recorder)", id);
    be::RepRecord R;
    R.arenas = r.d_arenas;
    R.n_arenas = (int)r.arenas.size();
    R.max_frames = r.max_frames;
    R.L = r.L;
    R.frames = r.frames;
    R.last_ep = r.last_ep;
    R.ctl = r.ctl;
    be::launch_replay_record(bx_, dE_, hE_, curmask_, d_rep_, d_ev_, R);
    if (be::capturing(bx_)) r.in_graph = true;
    return 0;
}

static bool make_dir(const std::string &d) { return mkdir(d.c_str(), 0777) == 0 || errno == EEXIST; }

int Engine::replay_write(int id, const char *dir, long long *dropped) {
    if (id < 0 || id >= (int)replays_.size() || !replays_[id].live) return refuse("unknown or freed replay id %d", id);
    if (be::capturing(bx_)) return refuse("replay_write synchronises: not possible while a CUDA graph is being captured");
    if (!dir) return refuse("replay_write: no directory");
    ReplayRec &r = replays_[id];
    const int nk = (int)r.arenas.size();
    std::vector<std::string> sub(nk);
    if (!make_dir(dir)) return refuse("replay_write: cannot create %s", dir);
    for (int k = 0; k < nk; ++k) {
        sub[k] = std::string(dir) + "/arena_" + std::to_string(r.arenas[k]);
        if (!make_dir(sub[k])) return refuse("replay_write: cannot create %s", sub[k].c_str());
    }
    be::sync(bx_);
    RepCtl ctl;
    be::d2h(bx_, &ctl, r.ctl, sizeof ctl);
    const long fi = r.L.frame_ints();
    std::vector<int> buf((size_t)ctl.n_frames * nk * fi);
    be::d2h(bx_, buf.data(), r.frames, buf.size() * 4);
    const int Gn = G();
    std::vector<std::vector<RepAgent>> agents(Gn);
    std::vector<AttackEvent> events;
    std::vector<RepEvent> evs;
    for (int k = 0; k < nk; ++k) {
        std::ofstream cfg(sub[k] + "/config.json");
        write_render_config(cfg);
        std::ofstream out;
        int open_file = 0;
        for (int f = 0; f < ctl.n_frames; ++f) {
            const int *F = buf.data() + ((size_t)f * nk + k) * fi;
            if (F[REP_H_WALLS]) {                     // the first frame of an episode opens a file, unless a split just did
                if (r.file_ct[k] == 0 || r.frame_ct[k] != 0) r.file_ct[k]++;
                r.frame_ct[k] = 0;
                std::vector<int> &w = r.walls[k];
                w.clear();
                for (int q = 0; q < r.L.wall_words; ++q)
                    for (unsigned bits = (unsigned)F[r.L.wall_base() + q]; bits; bits &= bits - 1)
                        w.push_back(q * 32 + __builtin_ctz(bits));
            }
            if (open_file != r.file_ct[k]) {
                out.close();
                out.open(sub[k] + "/video_" + std::to_string(r.file_ct[k]) + ".txt", r.frame_ct[k] == 0 ? std::ios::out : std::ios::app);
                if (!out) return refuse("replay_write: cannot write %s/video_%d.txt", sub[k].c_str(), r.file_ct[k]);
                open_file = r.file_ct[k];
            }
            const RepAgent *ag = (const RepAgent *)(F + r.L.agent_base());
            const RepEvent *ev = (const RepEvent *)(F + r.L.event_base());
            evs.clear();
            for (int g = 0, base = 0; g < Gn; base += r.cap[g], ++g) {        // rows at the flat offsets of r.cap
                agents[g].assign(ag + base, ag + base + F[REP_H_N + g]);
                for (int i = 0; i < F[REP_H_EV_N + g]; ++i) if (ev[base + i].rank >= 0) evs.push_back(ev[base + i]);
            }
            std::sort(evs.begin(), evs.end(), [](const RepEvent &p, const RepEvent &q) { return p.rank < q.rank; });
            events.clear();
            for (const RepEvent &e : evs) events.push_back({e.id, e.x, e.y});
            write_render_frame(out, r.frame_ct[k] == 0 ? &r.walls[k] : nullptr, agents, events);
            if (r.frame_ct[k]++ > frame_per_file_) { r.frame_ct[k] = 0; r.file_ct[k]++; }
        }
        if (out.is_open() && !out.flush()) return refuse("replay_write: cannot write %s", sub[k].c_str());
    }
    if (dropped) *dropped = (long long)ctl.dropped;
    be::dmemset(bx_, r.ctl, 0, sizeof(RepCtl));
    return ctl.n_frames;
}

int Engine::replay_free(int id) {
    if (id < 0 || id >= (int)replays_.size() || !replays_[id].live) return refuse("unknown or freed replay id %d", id);
    ReplayRec &r = replays_[id];
    if (r.in_graph) return refuse("replay %d is recorded into from inside a CUDA graph: it lives as long as the game", id);
    if (be::capturing(bx_)) return refuse("replay_free is not possible while a CUDA graph is being captured");
    for (void *p : {(void *)r.frames, (void *)r.d_arenas, (void *)r.last_ep, (void *)r.ctl}) be::dfree(bx_, p);
    r = ReplayRec();
    update_ev_arenas();
    return 0;
}

void Engine::sync() { if (bx_) be::sync(bx_); }
void Engine::graph_begin() {
    to_device();
    settle_counts();
    if (!first_render_) fatal("graph capture while rendering is not supported");
    capture_mask_ = curmask_; capture_culls_ = 0;
    // a graph may restore arenas from any live snapshot, and a replay then starts from restored counts: while one
    // exists, every count-sized launch of the capture, before a restore or after it, is sized for them (num_bound)
    const std::vector<int> floor = restore_floor();
    capture_floor_ = std::any_of(floor.begin(), floor.end(), [](int v) { return v > 0; });
    if (capture_floor_) raise_counts(floor);
    if (!be::capture_begin(bx_)) fatal("this backend has no CUDA graph support");
    graph_captured_ = true;
}
int Engine::graph_end() {
    const int id = be::capture_end(bx_);
    if (capture_floor_) { counts_unknown_ = true; capture_floor_ = false; }      // nothing ran: re-read the exact counts
    // kernel arguments are baked into the graph, the ping-pong buffer selector among them: a replay is only right when
    // the captured sequence leaves the selector where it found it (an even number of clear_dead calls)
    if (curmask_ != capture_mask_) fatal("a captured step sequence must contain an even number of clear_dead calls (got %d)", capture_culls_);
    return id;
}
void Engine::graph_launch(int id, int times) {
    to_device();
    for (int k = 0; k < times; ++k) be::graph_launch(bx_, id);
    if (times > 0) { ++state_version_; counts_unknown_ = true; counts_pending_ = false; may_have_dead_ = true; done_stale_ = true; }
}
void Engine::get_io_stats(long long *out, int cap) { for (int i = 0; i < cap && i < IO_N; ++i) out[i] = io_[i]; }
void *Engine::stream() { ensure_backend(); return be::stream_handle(bx_); }
void Engine::set_profiling(bool on) { ensure_backend(); be::profile_enable(bx_, on); }
void Engine::get_profile(double *ms, long long *n) { *ms = 0; *n = 0; if (bx_) be::profile_read(bx_, ms, n); }

int Engine::get_counters(long long *out, int cap) {
    int n = std::min<int>(cap, MG_N_COUNTERS);
    if (where_ != DEVICE && dE_ == nullptr) { for (int i = 0; i < n; ++i) out[i] = 0; return n; }
    std::vector<long long> c(MG_N_COUNTERS);
    be::d2h(bx_, c.data(), hE_.counters, sizeof(long long) * MG_N_COUNTERS);
    for (int i = 0; i < n; ++i) out[i] = c[i];
    return n;
}

int Engine::get_info(int group, const char *name, void *void_buffer) {         // GridWorld.cc:709-894
    int *ib = (int *)void_buffer;
    if (strequ(name, "obs_override")) {                 // extension: the obs_grid, obs_chunk, obs_tile keys
        ib[0] = obs_grid_; ib[1] = obs_chunk_; ib[2] = obs_tile_;
        return 0;
    }
    if (strequ(name, "obs_launch")) {                   // extension: shape of this engine's last render launch
        if (!be::obs_launch_report) return refuse("the %s backend does not report its render launches", be::name());
        for (int i = 0; i < 8; ++i) ib[i] = 0;
        if (bx_) be::obs_launch_report(bx_, ib);
        return 0;
    }
    if (strequ(name, "step_launch")) {                  // extension: shape of this engine's last step and cull launches
        if (!be::step_launch_report) return refuse("the %s backend does not report its step launches", be::name());
        for (int i = 0; i < 10; ++i) ib[i] = 0;
        if (bx_) be::step_launch_report(bx_, ib);
        return 0;
    }
    if (strequ(name, "state_space")) {                  // extension: per-arena shape of magent_b200_get_global_state
        ib[0] = H_; ib[1] = W_; ib[2] = state_channels();               // fixed: no counts needed, nothing to wait for
        return 0;
    }
    if (strequ(name, "num_bound")) {                    // extension: per group, records a device-pointer call may write
        for (int g = 0; g < G(); ++g) ib[g] = num_bound(g);     // before the counts next settle (no waiting here)
        return 0;
    }
    if (strequ(name, "slot_space")) {                   // extension: per group, S of magent_b200_get_slots (no waiting)
        for (int g = 0; g < G(); ++g) ib[g] = g < (int)slot_space_.size() ? slot_space_[g] : 0;
        return 0;
    }
    if (strequ(name, "arena_rng")) {                    // extension: uint32 minstd state of every arena
        if (where_ == DEVICE) {
            std::vector<ArenaHdr> hdr(A_);
            be::d2h(bx_, hdr.data(), hE_.hdr, sizeof(ArenaHdr) * A_);
            for (int a = 0; a < A_; ++a) ((uint32_t *)void_buffer)[a] = hdr[a].rng;
        } else {
            for (int a = 0; a < A_; ++a) ((uint32_t *)void_buffer)[a] = arenas_[a].rng;
        }
        return 0;
    }
    settle_counts();
    float *fb = (float *)void_buffer;
    if (strequ(name, "num")) {
        check_group(group, "get_info(num)");
        ib[0] = total(group);
    } else if (strequ(name, "id") || strequ(name, "pos") || strequ(name, "alive") || strequ(name, "hp")) {
        check_group(group, "get_info");
        to_device();
        const int n = total(group);
        const int kind = strequ(name, "id") ? INFO_ID : strequ(name, "pos") ? INFO_POS : strequ(name, "alive") ? INFO_ALIVE : INFO_HP;
        const size_t bytes = kind == INFO_POS ? (size_t)n * 8 : kind == INFO_ALIVE ? (size_t)n : (size_t)n * 4;
        read_back(be::is_device_ptr(void_buffer), {{void_buffer, bytes}}, [&](void **to) {
            be::launch_info(bx_, dE_, hE_, curmask_, kind, group, to[0], n);
        });
    } else if (strequ(name, "arena_num")) {
        check_group(group, "get_info(arena_num)");
        for (int a = 0; a < A_; ++a) ib[a] = count(group, a);
    } else if (strequ(name, "arena_done")) {
        if (done_stale_ && where_ == DEVICE) {          // the last env_step wrote its result to a device int only
            std::vector<int> d(A_);
            be::read_done(bx_, hE_, d.data());
            for (int a = 0; a < A_; ++a) arenas_[a].done = d[a] & 1;
            done_stale_ = false;
        }
        for (int a = 0; a < A_; ++a) ib[a] = arenas_[a].done;
    } else if (strequ(name, "action_space")) {
        check_group(group, "get_info"); ib[0] = group_type_[group]->n_action;
    } else if (strequ(name, "view_space")) {
        check_group(group, "get_info");
        ib[0] = group_type_[group]->view.height; ib[1] = group_type_[group]->view.width; ib[2] = n_channel();
    } else if (strequ(name, "feature_space")) {
        check_group(group, "get_info"); ib[0] = feature_size(group);
    } else if (strequ(name, "view2attack")) {
        check_group(group, "get_info");
        const AgentTypeDef &t = *group_type_[group];
        for (int i = 0; i < t.view.height * t.view.width; ++i) ib[i] = -1;
        // ret.at(dy - y1, dx - x1) = i is a LINEAR index without a bounds check in the reference (utility.h NDPointer::at,
        // GridWorld.cc:864-870): an attack cell whose column lies outside the view rectangle lands, wrapped, on a
        // neighbouring row.  Same here for every index inside the buffer; indices outside it (the reference corrupts the
        // heap there) are dropped.
        const int cells = t.view.height * t.view.width;
        for (int i = 0; i < t.attack.count; ++i) {
            const long idx = (long)(t.attack.dy[i] - t.view.y1) * t.view.width + (t.attack.dx[i] - t.view.x1);
            if (idx >= 0 && idx < cells) ib[idx] = i;
        }
    } else if (strequ(name, "attack_base")) {
        check_group(group, "get_info"); ib[0] = group_type_[group]->attack_base;
    } else if (strequ(name, "both_attack")) {
        ib[0] = 0;                                    // `const bool stat = false` in the reference
    } else if (strequ(name, "groups_info")) {
        static const int colors[][3] = {{192, 64, 64}, {64, 64, 192}, {64, 192, 64}, {64, 64, 64}};
        for (int i = 0; i < G(); i++) {
            ib[i * 5 + 0] = group_type_[i]->width; ib[i * 5 + 1] = group_type_[i]->length;
            for (int c = 0; c < 3; ++c) ib[i * 5 + 2 + c] = colors[i % 4][c];
        }
    } else if (strequ(name, "walls_info") || strequ(name, "global_minimap") || strequ(name, "mean_info") ||
               strequ(name, "render_window_info") || strequ(name, "attack_event")) {
        // cold getters: served from a host snapshot of arena 0 (or the selected arena)
        to_host(true);
        const HostArena &ar = arenas_[sel_arena_ >= 0 ? sel_arena_ : 0];
        if (strequ(name, "walls_info")) {
            int ct = 0;
            for (int i = 0; i < W_ * H_; i++)
                if (ar.occ[i] == OCC_WALL) { ++ct; ib[ct * 2] = i % W_; ib[ct * 2 + 1] = i / W_; }
            ib[0] = ct;
        } else if (strequ(name, "global_minimap")) {
            int vh = (int)lround(fb[0]), vw = (int)lround(fb[1]);
            int ng = G();
            for (int i = 0; i < vh * vw * ng; ++i) fb[i] = 0.0f;
            int scale_h = (H_ + vh - 1) / vh, scale_w = (W_ + vw - 1) / vw;
            for (int i = 0; i < ng; i++) {
                int ch = ((i - group) % ng + ng) % ng;
                const HostGroup &hg = ar.groups[i];
                for (int j = 0; j < hg.size(); j++) fb[((hg.y[j] / scale_h) * vw + hg.x[j] / scale_w) * ng + ch] += 1.0f;
                for (int j = 0; j < vh * vw; j++) fb[j * ng + ch] /= (float)hg.size();
            }
        } else if (strequ(name, "mean_info")) {
            check_group(group, "get_info(mean_info)");
            const HostGroup &hg = ar.groups[group];
            int na = group_type_[group]->n_action;
            float sx = 0, sy = 0;
            std::vector<int> ctr(na + 1, 0);
            for (int i = 0; i < hg.size(); i++) { sx += hg.x[i]; sy += hg.y[i]; if (hg.act[i] >= 0 && hg.act[i] <= na) ctr[hg.act[i]]++; }
            fb[0] = sx / hg.size(); fb[1] = sy / hg.size();
            for (int i = 0; i < na; i++) fb[2 + i] = (float)(1.0 * ctr[i] / hg.size());
        } else if (strequ(name, "render_window_info")) {
            first_render_ = false;                     // GridWorld.cc:798
            int x1 = ib[0], y1 = ib[1], x2 = ib[2], y2 = ib[3], ct = 1;
            for (int g = 0; g < G(); g++) {
                const HostGroup &hg = ar.groups[g];
                for (int j = 0; j < hg.size(); j++) {
                    if (hg.x[j] < x1 || hg.x[j] > x2 || hg.y[j] < y1 || hg.y[j] > y2) continue;
                    if (group_type_[g]->can_absorb && !(hg.flags[j] & FLAG_ABSORBED)) continue;     // GridWorld.cc:821
                    ib[ct * 4] = hg.id[j]; ib[ct * 4 + 1] = hg.x[j]; ib[ct * 4 + 2] = hg.y[j]; ib[ct * 4 + 3] = g; ct++;
                }
            }
            ib[0] = ct - 1; ib[1] = (int)attack_events_.size();
        } else if (strequ(name, "attack_event")) {
            for (size_t i = 0; i < attack_events_.size(); i++) {
                ib[i * 3] = attack_events_[i].id; ib[i * 3 + 1] = attack_events_[i].x; ib[i * 3 + 2] = attack_events_[i].y;
            }
        }
    } else {
        fatal("unsupported info name in GridWorld::get_info : %s", name);
    }
    return 0;
}

}  // namespace mg
