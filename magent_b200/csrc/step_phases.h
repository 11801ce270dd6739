// step_phases.h -- the GridWorld step pipeline as data-parallel phases over one arena.
//
// Every function below is executed by a *team* of threads (Ctx: tid()/nth()/scan()/sync are provided
// by the caller: a CTA, a cooperative grid, or the single-threaded test emulation).  Phases are
// separated by team barriers in run_step()/run_cull(); inside a phase each thread only writes state it
// owns (its agent, its agent's cells) or uses atomics.
//
// The reference executes attack and move *sequentially* (attack order = a Fisher-Yates shuffle of the
// attack buffer, GridWorld.cc:464-506; move order = band buffers then boundary buffer in insertion
// order, GridWorld.cc:573-613).  The phases reproduce the OUTCOME of that sequential order:
//   * shuffle replay: closed-form position of every element after the swap loop (DESIGN.md §4.2),
//   * attack: per-victim timelines in rank order, relaxed to the unique fixpoint of the
//     "attacker still alive at its rank" dependency (triangular in rank => unique, reached by sweeps),
//   * move: per-cell claimant lists + relaxation of "claimant succeeds iff every target cell is free at
//     its turn" (triangular in order key).
#pragma once
#include "dev_types.h"

namespace mg {

struct GroupEnum {
    int cnt, k_n;
    int grp[MG_MAX_GROUPS];
    int pre[MG_MAX_GROUPS + 1];
};

MG_HD void enum_all(const EngineDev &E, int a, GroupEnum &e) {
    e.k_n = E.G; e.pre[0] = 0;
    for (int g = 0; g < E.G; ++g) { e.grp[g] = g; e.pre[g + 1] = e.pre[g] + E.n[g * E.A + a]; }
    e.cnt = e.pre[E.G];
}
MG_HD void enum_order(const EngineDev &E, const StepArgs &S, int a, GroupEnum &e) {
    e.k_n = S.n_order; e.pre[0] = 0;
    for (int k = 0; k < S.n_order; ++k) {
        e.grp[k] = S.order[k];
        e.pre[k + 1] = e.pre[k] + E.n[S.order[k] * E.A + a];
    }
    e.cnt = e.pre[S.n_order];
}
MG_HD void enum_locate(const GroupEnum &e, int idx, int &k, int &i) {
    k = 0;
    while (idx >= e.pre[k + 1]) ++k;
    i = idx - e.pre[k];
}

MG_HD const AgentSoA &cur_soa(const EngineDev &E, unsigned curmask, int g) {
    return E.grp[g].soa[(curmask >> g) & 1u];
}

// view of one arena: bases into the arena-major arrays
struct ArenaRef {
    int a;
    int *occ, *claim;
    long sb;            // base into per-agent scratch  (a * scratch_stride)
    long nb;            // base into claim nodes        (a * scratch_stride * max_body)
    ArenaHdr *hdr;
};
// claimant node -> the mover that owns it (nodes are numbered mover * max_body + body cell; 1x1 bodies skip the divide)
MG_HD int node_owner(const EngineDev &E, int node) { return E.max_body == 1 ? node : node / E.max_body; }
// the one-byte kind plane of the observation (dev_types.h) follows every occupancy write
MG_HD void kind_set(const EngineDev &E, int a, int x, int y, unsigned char k) {
    E.kind[a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad] = k;
}
// ... and so does the hp_norm plane: hp / max_hp of the occupant (Map.cc:197) at every occupied cell, written where an
// agent's hp changes (attack / starve / absorb) and where it takes new cells (move, turn, placement)
MG_HD void hpn_set(const EngineDev &E, int a, int x, int y, float v) {
#if !defined(MG_ABLATE_HPN)                          // (profiling variants only: results are WRONG without it)
    E.hpn[a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad] = v;
#endif
}
// the cells of a living agent show its group and hp: kind byte (with KIND_FULL when hp == max_hp) and, unless full, hp / max_hp
MG_HD void show_body(const EngineDev &E, int a, int g, const GroupDev &G, int x, int y, int bw, int bh, float hp) {
    const bool full = hp == G.max_hp;
    const unsigned char k = kind_agent(g, full);
    const float v = hp / G.max_hp;
    for (int bx = 0; bx < bw; ++bx)
        for (int by = 0; by < bh; ++by) {
            kind_set(E, a, x + bx, y + by, k);
            if (!full) hpn_set(E, a, x + bx, y + by, v);
        }
}
// ---- directions (turn_mode; reference Map.cc:515-607).  Without turn_mode every agent faces NORTH, for which
// relative = absolute and the body is width x length.
MG_HD int agent_dir(const EngineDev &E, const AgentSoA &s, long gi) { return E.turn_mode ? (int)s.dir[gi] : (int)DIR_NORTH; }
// get_size_for_dir: footprint of a body facing `dir`
MG_HD void body_dims(const GroupDev &G, int dir, int &w, int &h) {
    if (dir == DIR_NORTH || dir == DIR_SOUTH) { w = G.body_w; h = G.body_l; } else { w = G.body_l; h = G.body_w; }
}
// rela_to_abs: displacement (rx, ry) in the agent's frame -> map displacement
MG_HD void dir_rot(int dir, int rx, int ry, int &dx, int &dy) {
    switch (dir) {
        case DIR_NORTH: dx = rx; dy = ry; break;
        case DIR_SOUTH: dx = -rx; dy = -ry; break;
        case DIR_WEST: dx = ry; dy = -rx; break;
        default: dx = -ry; dy = rx; break;          // EAST
    }
}
// save_to_real: offset of the "real" (head) corner from the stored top-left corner
MG_HD void dir_real(const GroupDev &G, int dir, int &ox, int &oy) {
    switch (dir) {
        case DIR_NORTH: ox = 0; oy = 0; break;
        case DIR_SOUTH: ox = G.body_w - 1; oy = G.body_l - 1; break;
        case DIR_WEST: ox = 0; oy = G.body_w - 1; break;
        default: ox = G.body_l - 1; oy = 0; break;  // EAST
    }
}
MG_HD ArenaRef arena_ref(const EngineDev &E, int a) {
    ArenaRef r;
    r.a = a;
    r.occ = E.occ + (long)a * E.W * E.H;
    r.claim = E.claim_head + (long)a * E.W * E.H;
    r.sb = (long)a * E.scratch_stride;
    r.nb = (long)a * E.scratch_stride * E.max_body;
    r.hdr = E.hdr + a;
    return r;
}
MG_HD long gidx(const EngineDev &E, int a, int g, int i) { return (long)a * E.grp[g].cap + i; }
MG_HD int lflat(const EngineDev &E, int code) { return E.grp[code_group(code)].foff + code_index(code); }

// ------------------------------------------------------------------------------------------------
// phase 0: reset per-step scratch
template <class Ctx>
MG_HD void phase_init(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &all, const GroupEnum &ord) {
    ArenaRef R = arena_ref(E, a);
    for (int idx = c.tid(); idx < all.cnt; idx += c.nth()) {
        int g, i; enum_locate(all, idx, g, i);
        const AgentSoA &s = cur_soa(E, S.curmask, g);
        long f = R.sb + E.grp[g].foff + i;
        bool dead = s.flags[gidx(E, a, g, i)] & FLAG_DEAD;
        E.att_rank[f] = RANK_NONE;
        E.tgt[f] = -1;
        E.in_head[f] = -1;
        E.death[f] = dead ? DEATH_BEFORE : DEATH_NEVER;
        E.sh_head[R.sb + idx] = -1;          // shuffle scratch is indexed by buffer position < n_attack <= cnt
        E.sh_first[R.sb + idx] = DEATH_NEVER;
    }
    if (c.tid() == 0) {
        R.hdr->n_attack = 0;
        for (int r = 0; r < E.n_rules; ++r) R.hdr->rule_trig[r] = 0;
        for (int q = 0; q < E.n_allq; ++q) { R.hdr->allq_viol[q] = 0; R.hdr->allq_min[q] = 0x7fffffff; R.hdr->allq_max[q] = -0x7fffffff - 1; }
        R.hdr->rng_next = R.hdr->rng;
        c.add_count(E, CNT_AGENT_STEPS, ord.cnt);
        if (a == 0) c.add_count(E, CNT_STEPS, 1);
    }
}

// phase 1: position of every attack action in the attack buffer (reference GridWorld.cc:403-454 pushes
// in set_action call order, then agent index order; dead-but-unculled agents are pushed too)
template <class Ctx>
MG_HD int phase_attack_scan(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord) {
    ArenaRef R = arena_ref(E, a);
    auto pred = [&](int idx) -> int {
        int k, i; enum_locate(ord, idx, k, i);
        int g = ord.grp[k];
        int act = cur_soa(E, S.curmask, g).act[gidx(E, a, g, i)];
        return (act >= E.grp[g].attack_base && act < E.grp[g].n_action) ? 1 : 0;
    };
    auto emit = [&](int idx, int e) {
        int k, i; enum_locate(ord, idx, k, i);
        E.att_agent[R.sb + e] = code_make(ord.grp[k], i);
    };
    int total = c.scan(ord.cnt, pred, emit);
    if (c.tid() == 0) {
        R.hdr->n_attack = total;
        c.add_count(E, CNT_ATTACKS, total);
    }
    return total;
}

// phase 2: the A random draws of the shuffle, j_e = x_e mod (e+1)  (GridWorld.cc:465-468), by jump-ahead
template <class Ctx>
MG_HD void phase_rng(Ctx &c, const EngineDev &E, int a, int n_attack) {
    ArenaRef R = arena_ref(E, a);
    uint32_t x0 = R.hdr->rng;
    for (int e = c.tid(); e < n_attack; e += c.nth()) {
        uint32_t x = mulmod31(minstd_pow(E.pow2, (uint32_t)e + 1u), x0);
        int j = (int)(x % (uint32_t)(e + 1));
        E.jv[R.sb + e] = j;
        E.sh_next[R.sb + e] = atomic_exch(&E.sh_head[R.sb + j], e);
        if (e > j) atomic_min(&E.sh_first[R.sb + j], e);
        if (e == n_attack - 1) R.hdr->rng_next = x;
    }
}

// cell an attack action aims at (Map::get_attack_obj, Map.cc:209-221); may lie off the board
MG_HD void attack_cell_from(const EngineDev &E, const GroupDev &G, int act, int x, int y, int dir, int &tx, int &ty) {
    const int k = act - G.attack_base;
    const int adx = ld_ro(G.att_dx + k), ady = ld_ro(G.att_dy + k);
    tx = x + G.att_xoff + adx;
    ty = y + G.att_yoff + ady;
    if (E.turn_mode) {
        int rx, ry, dx, dy;
        dir_real(G, dir, rx, ry);
        dir_rot(dir, G.att_xoff + adx, G.att_yoff + ady, dx, dy);
        tx = x + rx + dx; ty = y + ry + dy;
    }
}
MG_HD void attack_cell(const EngineDev &E, const GroupDev &G, const AgentSoA &s, long gi, int &tx, int &ty) {
    attack_cell_from(E, G, s.act[gi], s.x[gi], s.y[gi], E.turn_mode ? (int)s.dir[gi] : (int)DIR_NORTH, tx, ty);
}
MG_HD int flat_group(const EngineDev &E, int flat) {
    int g = 0;
    while (g + 1 < E.G && flat >= E.grp[g + 1].foff) ++g;
    return g;
}
// target cell of the attacker with local flat id `flat`, as a linear cell index
MG_HD int attack_cell_of(const EngineDev &E, unsigned curmask, int a, int flat) {
    const int g = flat_group(E, flat);
    int tx, ty;
    attack_cell(E, E.grp[g], cur_soa(E, curmask, g), gidx(E, a, g, flat - E.grp[g].foff), tx, ty);
    return ty * E.W + tx;
}
// an attack on an agent of one's own group is refused unless the type has attack_in_group (Map.cc:236-240)
MG_HD bool friendly_fire_refused(const EngineDev &E, int att_group, int victim_group) {
    return att_group == victim_group && !E.grp[att_group].attack_in_group;
}

// ---- food_mode (Map.cc:245,276-303).  A kill leaves victim.food_supply units of food on the ATTACKED cell; every later
// attack on that cell -- this step or any later one, by any group -- eats min(eat_ability, food) and the food is gone
// once less than 0.1 is left.  Eating only depends on which eaters are still alive at their rank, so a cell's food
// level is a rank-ordered timeline like a victim's hp.
//   list: chain of attacker flat ids through in_next (a victim's in-list, or the cell list hung off the claim plane)
//   only eaters with start_rank < rank < upto that aim at `cell` and execute (death > rank) take their bite
// Returns the food left for an event at rank `upto`; gone = nothing (left) there.
MG_HD float food_timeline(const EngineDev &E, const ArenaRef &R, unsigned curmask, int cell, int list, float food0,
                          int start_rank, int upto, bool &gone) {
    float food = food0;
    gone = false;
    int last = start_rank;
    for (;;) {
        int best = upto, be = -1;
        for (int e = list; e != -1; e = E.in_next[R.sb + e]) {
            const int r = E.att_rank[R.sb + e];
            if (r > last && r < best) { best = r; be = e; }
        }
        if (be == -1) break;
        last = best;
        if (ld_volatile(&E.death[R.sb + be]) <= best) continue;             // dead before (or at) its turn: no bite
        if (attack_cell_of(E, curmask, R.a, be) != cell) continue;
        const float bite = E.grp[flat_group(E, be)].eat_ability;
        const float add = bite < food ? bite : food;                        // Map.cc:295-297
        food -= add;
        if ((double)food < 0.1) { gone = true; return 0.0f; }               // Map.cc:298-302
    }
    return food;
}
// food an attacker finds on its target cell when its turn (rank own_r) comes; found = false when the cell is blank or
// holds a living agent by then.  list_out / food0_out / start_out describe the cell's timeline for the commit phase.
MG_HD float food_found(const EngineDev &E, const ArenaRef &R, unsigned curmask, int my_tgt, int my_cell, int own_r, bool &found) {
    found = false;
    if (my_tgt == TGT_FOOD) {
        bool gone;
        const float f = food_timeline(E, R, curmask, my_cell, R.claim[my_cell], E.food[(long)R.a * E.W * E.H + my_cell], -1, own_r, gone);
        found = !gone;
        return f;
    }
    // the target agent died earlier this step: food lies here iff the killing blow landed on this very cell
    const int vflat = lflat(E, my_tgt);
    const int dv = ld_volatile(&E.death[R.sb + vflat]);
    if (dv >= own_r || dv < 0) return 0.0f;
    const int vg = code_group(my_tgt);
    for (int k = E.in_head[R.sb + vflat]; k != -1; k = E.in_next[R.sb + k]) {
        if (E.att_rank[R.sb + k] != dv) continue;
        if (attack_cell_of(E, curmask, R.a, k) != my_cell) return 0.0f;
        bool gone;
        const float f = food_timeline(E, R, curmask, my_cell, E.in_head[R.sb + vflat], E.grp[vg].food_supply, dv, own_r, gone);
        found = !gone;
        return f;
    }
    return 0.0f;
}

// phase 3: final buffer position (= execution rank) of each attack, and its target
template <class Ctx>
MG_HD void phase_rank_target(Ctx &c, const EngineDev &E, const StepArgs &S, int a, int n_attack) {
    ArenaRef R = arena_ref(E, a);
    for (int e = c.tid(); e < n_attack; e += c.nth()) {
        // element e is swapped to position v=j_e at step e; afterwards it moves whenever a later step
        // picks its current position: first to ne = next step with the same j, then along sh_first.
        // the attacker's own fields are requested first: their global round trip overlaps the shuffle walk below
        const int code = E.att_agent[R.sb + e];
        const int g = code_group(code), i = code_index(code);
        const GroupDev &G = E.grp[g];
        const AgentSoA &s = cur_soa(E, S.curmask, g);
        const long gi = gidx(E, a, g, i);
        const unsigned char fl = s.flags[gi];
        const int act = s.act[gi], ax = s.x[gi], ay = s.y[gi];
        const int adir = E.turn_mode ? (int)s.dir[gi] : (int)DIR_NORTH;
        int v = E.jv[R.sb + e];
        int ne = DEATH_NEVER;
        for (int q = E.sh_head[R.sb + v]; q != -1; q = E.sh_next[R.sb + q])
            if (q > e && q < ne) ne = q;
        int pos = v;
        if (ne != DEATH_NEVER) {
            pos = ne;
            for (int nx = E.sh_first[R.sb + pos]; nx != DEATH_NEVER; nx = E.sh_first[R.sb + pos]) pos = nx;
        }
        int fs = G.foff + i;
        E.att_rank[R.sb + fs] = pos;
        if (fl & FLAG_DEAD) continue;                   // skipped at execution (GridWorld.cc:479)
        // Map::get_attack_obj (Map.cc:209-252)
        int tx, ty;
        attack_cell_from(E, G, act, ax, ay, adir, tx, ty);
        if (tx < 0 || tx >= E.W || ty < 0 || ty >= E.H) continue;
        int t = R.occ[ty * E.W + tx];
        if (E.food_mode && t == OCC_FOOD) {             // eaters of one cell queue on the (idle) claim plane
            E.tgt[R.sb + fs] = TGT_FOOD;
            E.in_next[R.sb + fs] = atomic_exch(&R.claim[ty * E.W + tx], fs);
            continue;
        }
        if (t < 0) continue;
        // a refused in-group attack is a blank -- unless the cell holds food by the time its turn comes (food_mode),
        // so it still joins the occupant's list, as a non-damaging member
        if (friendly_fire_refused(E, g, code_group(t)) && !E.food_mode) continue;
        E.tgt[R.sb + fs] = t;
        E.in_next[R.sb + fs] = atomic_exch(&E.in_head[R.sb + lflat(E, t)], fs);
    }
}

// phase 4 (swept until stable): death rank of every agent that is hit or that attacks.
// Sequential semantics being reproduced: GridWorld.cc:475-506 + Map::do_attack (Map.cc:255-310) +
// Agent::be_attack/add_hp (GridWorld.h:185,203-209).
template <class Ctx>
MG_HD bool phase_attack_relax(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &all) {
    ArenaRef R = arena_ref(E, a);
    bool changed = false;
    for (int idx = c.tid(); idx < all.cnt; idx += c.nth()) {
        int g, i; enum_locate(all, idx, g, i);
        int ft = E.grp[g].foff + i;
        long f = R.sb + ft;
        int head = E.in_head[f];
        int my_tgt = E.tgt[f];
        if (head == -1 && my_tgt == TGT_NONE) continue;
        const GroupDev &G = E.grp[g];
        float hp = cur_soa(E, S.curmask, g).hp[gidx(E, a, g, i)];
        int own_r = my_tgt != TGT_NONE ? E.att_rank[f] : DEATH_NEVER;
        bool own_done = my_tgt == TGT_NONE;
        int last = -1, dn = DEATH_NEVER;
        for (;;) {
            int best = DEATH_NEVER, bs = -1;
            for (int s = head; s != -1; s = E.in_next[R.sb + s]) {
                int r = E.att_rank[R.sb + s];
                if (r > last && r < best) { best = r; bs = s; }
            }
            if (!own_done && own_r < best) {            // my own attack comes first: kill => supply
                own_done = true;
                if (my_tgt >= 0 && ld_volatile(&E.death[R.sb + lflat(E, my_tgt)]) == own_r) {
                    float sup = E.grp[code_group(my_tgt)].kill_supply;
                    float nh = hp + sup;                 // Agent::add_hp: min(type.hp, hp + add)
                    hp = G.max_hp < nh ? G.max_hp : nh;
                } else if (E.food_mode) {                // food on my target cell by now?  eat (Map.cc:292-297)
                    bool found;
                    const float food = food_found(E, R, S.curmask, my_tgt, attack_cell_of(E, S.curmask, a, ft), own_r, found);
                    if (found) {
                        const float add = G.eat_ability < food ? G.eat_ability : food;
                        const float nh = hp + add;
                        hp = G.max_hp < nh ? G.max_hp : nh;
                    }
                }
                continue;
            }
            if (bs == -1) break;
            last = best;
            // attacker dead by then?  (a long body with attack_in_group can aim at one of its own cells: if the walk got
            // this far the agent is alive at its own rank)
            if (bs != ft && ld_volatile(&E.death[R.sb + bs]) < best) continue;
            // attacker's group -> damage
            const int sg = flat_group(E, bs);
            if (E.food_mode && friendly_fire_refused(E, sg, g)) continue;   // listed only as a potential eater
            hp -= E.grp[sg].damage;
            if (hp < 0.0f) {
                dn = best;
                if (bs == ft) {                          // my own blow killed me: do_attack still feeds the (dead) killer the
                    const float nh = hp + G.kill_supply; // victim's kill_supply (Map.cc:268-273) -- visible only as the hp of
                    hp = G.max_hp < nh ? G.max_hp : nh;  // an un-culled corpse in the replay dump
                }
                break;
            }
        }
        E.hp_fin[f] = hp;
        if (dn != E.death[f]) { st_volatile(&E.death[f], dn); changed = true; }
    }
    return changed;
}

// phase 5: commit attacks (attacker side and victim side) and starvation (GridWorld.cc:519-542)
template <class Ctx>
MG_HD void phase_attack_apply_starve(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &all) {
    ArenaRef R = arena_ref(E, a);
    int kills = 0, hits = 0, starved = 0;
    for (int idx = c.tid(); idx < all.cnt; idx += c.nth()) {
        int g, i; enum_locate(all, idx, g, i);
        const GroupDev &G = E.grp[g];
        const AgentSoA &s = cur_soa(E, S.curmask, g);
        long gi = gidx(E, a, g, i);
        long f = R.sb + G.foff + i;
        // mover scratch is (re)initialised here, after the shuffle scratch it may share storage with is dead
        E.mv_key[f] = MVKEY_NONE;
        E.mv_state[f] = MV_NONE;
        if (S.record_events) G.ev_rank[gi] = -1;
        // requested together, before the first test needs one: one global round trip instead of three
        const unsigned char fl = s.flags[gi];
        const float hp0 = s.hp[gi];
        float nr = s.next_reward[gi];                    // only this thread writes this agent's reward in this phase
        if (fl & FLAG_DEAD) continue;
        int d = E.death[f];
        int r = E.att_rank[f];
        // my attack is executed iff I am alive when its rank comes; d == r can only mean that it is my own blow that
        // kills me (an in-group attack aimed at one of my own cells)
        const bool executed = r != RANK_NONE && (d > r || (d == r && E.tgt[f] == code_make(g, i)));
        const bool self_kill = executed && d == r;
        if (S.record_events && executed) G.ev_rank[gi] = r;                    // RenderAttackEvent, GridWorld.cc:484-485
        float late_reward = 0.0f;                        // a self-kill is rewarded AFTER the death assignment (Map.cc:265-283)
        if (executed) {
            int t = E.tgt[f];
            int dt = t >= 0 ? E.death[R.sb + lflat(E, t)] : DEATH_BEFORE;
            if (t >= 0 && E.food_mode && friendly_fire_refused(E, g, code_group(t))) dt = DEATH_BEFORE;
            if (t < 0 || dt < r) {                       // blank / already dead / food (eating earns nothing): penalty only
                nr += G.attack_penalty;
            } else if (dt == r) {                        // my hit kills
                s.last_op[gi] = OP_KILL;
                s.op_obj[gi] = t;
                if (self_kill) late_reward = E.grp[code_group(t)].kill_reward + G.attack_penalty;
                else nr += E.grp[code_group(t)].kill_reward + G.attack_penalty;
                ++kills; ++hits;
            } else {
                s.last_op[gi] = OP_ATTACK;
                s.op_obj[gi] = t;
                nr += 0.0f + G.attack_penalty;
                ++hits;
            }
        }
        bool evaluated = E.in_head[f] != -1 || E.tgt[f] != TGT_NONE;
        float hp = evaluated ? E.hp_fin[f] : hp0;
        bool dies = false;
        if (d != DEATH_NEVER) {                          // killed in the attack phase
            dies = true;
        } else {                                         // Agent::starve (GridWorld.h:194-201)
            if (G.step_recover > 0) {
                float nh = hp + G.step_recover;
                hp = G.max_hp < nh ? G.max_hp : nh;
            } else {
                hp -= -G.step_recover;
                if (hp < 0.0f) { dies = true; ++starved; }
            }
        }
        s.hp[gi] = hp;
        if (!dies && hp != hp0) {                        // keep the hp_norm plane of the observation current
            int bw, bh;
            body_dims(G, agent_dir(E, s, gi), bw, bh);
            show_body(E, a, g, G, s.x[gi], s.y[gi], bw, bh, hp);
        }
        if (dies) {
            s.flags[gi] = fl | FLAG_DEAD;
            R.hdr->any_dead = 1;
            nr = G.dead_penalty;                         // assignment (GridWorld.h:206)
            if (self_kill) nr += late_reward;
            int x = s.x[gi], y = s.y[gi], bw, bh;
            body_dims(G, agent_dir(E, s, gi), bw, bh);
            for (int bx = 0; bx < bw; ++bx)
                for (int by = 0; by < bh; ++by) {
                    R.occ[(y + by) * E.W + x + bx] = OCC_EMPTY;
                    kind_set(E, a, x + bx, y + by, 0);
                }
            atomic_add(&E.dead_ct[g * E.A + a], 1);
        }
        if (executed || dies) s.next_reward[gi] = nr;
    }
    c.add_count(E, CNT_KILLS, kills);
    c.add_count(E, CNT_HITS, hits);
    c.add_count(E, CNT_STARVED, starved);
}

// phase 5b/5c (food_mode only): what is left on every cell whose food was created or bitten this step.  Every
// participant of a cell's timeline computes the same final amount (5b, into hp_fin) and writes it (5c): the
// writes agree, so no owner has to be elected.  5c runs after the victims' bodies were cleared in phase 5.
template <class Ctx>
MG_HD void phase_food_commit(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &all, bool write) {
    ArenaRef R = arena_ref(E, a);
    float *foodp = E.food + (long)a * E.W * E.H;
    for (int idx = c.tid(); idx < all.cnt; idx += c.nth()) {
        int g, i; enum_locate(all, idx, g, i);
        const int ft = E.grp[g].foff + i;
        const long f = R.sb + ft;
        const int t = E.tgt[f], r = E.att_rank[f];
        if (t == TGT_FOOD && write) R.claim[attack_cell_of(E, S.curmask, a, ft)] = -1;    // unhook the eaters' queue, executed or not
        if (t == TGT_NONE || r == RANK_NONE || E.death[f] < r || (E.death[f] == r && t != code_make(g, i))) continue;   // not executed
        int list, start;
        float food0;
        if (t == TGT_FOOD) { start = -1; }
        else if (!friendly_fire_refused(E, g, code_group(t)) && E.death[R.sb + lflat(E, t)] == r) { start = r; }   // my kill
        else continue;
        const int cell = attack_cell_of(E, S.curmask, a, ft);
        if (!write) {
            if (t == TGT_FOOD) { list = R.claim[cell]; food0 = foodp[cell]; }
            else { list = E.in_head[R.sb + lflat(E, t)]; food0 = E.grp[code_group(t)].food_supply; }
            bool gone;
            const float left = food_timeline(E, R, S.curmask, cell, list, food0, start, DEATH_NEVER, gone);
            E.hp_fin[f] = gone ? -1.0f : left;
        } else {
            const float left = E.hp_fin[f];
            const bool gone = left < 0.0f;
            foodp[cell] = gone ? 0.0f : left;
            R.occ[cell] = gone ? OCC_EMPTY : OCC_FOOD;
            kind_set(E, a, cell % E.W, cell / E.W, gone ? (unsigned char)KIND_EMPTY : (unsigned char)KIND_FOOD);
        }
    }
}

// footprint a mover wants to occupy: its current footprint for a move, the rotated one for a turn
MG_HD void mover_dims(const EngineDev &E, const GroupDev &G, const AgentSoA &s, long gi, bool turn, int &w, int &h) {
    body_dims(G, agent_dir(E, s, gi), w, h);
    if (turn) { int t = w; w = h; h = t; }           // every turn is by 90 degrees (wise = 2 * act - 1 is odd)
}
// direction after a turn action (reference GridWorld.cc:556 passes act - move_base, so wise = 2 * act - 1 is neither
// -1 nor 1: Map::do_turn takes its "else" formula and new_dir = (dir + wise + 4) % 4, Map.cc:367)
MG_HD int turned_dir(int dir, int act) { return (dir + 2 * act - 1 + 4) % 4; }

// Where a move (turn == false) or turn (turn == true) action `act` would put an agent at (x, y) facing `dir`: top-left
// corner (nx, ny) and footprint bw x bh.  Returns the reference's in-board verdict for that footprint (Map.cc:455).
// Shared by the step (phase_move_register) and the legal-action mask (mask_phases.h).
MG_HD bool mover_target(const EngineDev &E, const GroupDev &G, int act, int x, int y, int dir, bool turn,
                        int &nx, int &ny, int &bw, int &bh) {
    if (turn) {
        // the body pivots about its "real" corner (turn offsets are 0, AgentType.cc:108): the stored top-left
        // corner follows from real_to_save with the new direction
        const int nd = turned_dir(dir, act);
        int rx, ry, qx, qy;
        dir_real(G, dir, rx, ry);
        dir_real(G, nd, qx, qy);
        nx = x + rx - qx; ny = y + ry - qy;
    } else {
        int dx = ld_ro(G.move_dx + act), dy = ld_ro(G.move_dy + act);
        if (E.turn_mode) { const int rx = dx, ry = dy; dir_rot(dir, rx, ry, dx, dy); }     // GridWorld.cc:587-598
        nx = x + dx; ny = y + dy;
    }
    body_dims(G, dir, bw, bh);
    if (turn) { int t = bw; bw = bh; bh = t; }       // every turn is by 90 degrees
    return !(nx < 0 || ny < 0 || nx + bw >= E.W || ny + bh >= E.H);
}

// phase 6: movers (turn == false) or turners (turn == true, turn_mode only) compute their target footprint and
// queue on every target cell.  Turn: Map::do_turn, Map.cc:361-406; move: Map::do_move, Map.cc:313-358.
// A thread owns ~4 movers.  One at a time each costs three dependent global round trips (own fields -> occupancy of
// the target -> claim exchange); the batch below issues each kind of request for all of the thread's movers
// before it consumes the first answer.  Everything indexed by `u` is unrolled into registers.
template <class Ctx>
MG_HD void phase_move_register(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord, bool turn) {
    ArenaRef R = arena_ref(E, a);
    constexpr int U = 4;
    for (int base = c.tid(); base < ord.cnt; base += U * c.nth()) {
        int act[U], x[U], y[U], fl[U], dir[U];
        // request 1: the agents' own fields
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) {
            const int idx = base + u * c.nth();
            act[u] = -1; x[u] = y[u] = fl[u] = 0; dir[u] = DIR_NORTH;
            if (idx < ord.cnt) {
                int k, i; enum_locate(ord, idx, k, i);
                const int g = ord.grp[k];
                const AgentSoA &s = cur_soa(E, S.curmask, g);
                const long gi = gidx(E, a, g, i);
                act[u] = s.act[gi]; fl[u] = s.flags[gi]; x[u] = s.x[gi]; y[u] = s.y[gi];
                if (E.turn_mode) dir[u] = s.dir[gi];
            }
        }
        int cell[U], node[U];                           // single-cell footprints wait here for requests 2 and 3
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) {
            cell[u] = -1; node[u] = 0;
            const int idx = base + u * c.nth();
            if (idx >= ord.cnt) continue;
            int k, i; enum_locate(ord, idx, k, i);
            const int g = ord.grp[k];
            const GroupDev &G = E.grp[g];
            const int av = act[u];
            if (turn ? (av < G.n_move || av >= G.attack_base) : (av < 0 || av >= G.n_move)) continue;
            if (fl[u] & (turn ? FLAG_DEAD : (FLAG_DEAD | FLAG_ABSORBED))) continue;     // GridWorld.cc:553,581
            const int fs = G.foff + i;
            const long f = R.sb + fs;
            // insertion order of the reference: band buffers 0..nsep-1, then the boundary buffer
            unsigned bucket = (unsigned)E.nsep;
            if (E.large_map) {
                int xm = x[u] % E.bandwidth;
                if (!(xm < 4 || xm > E.bandwidth - 4)) bucket = (unsigned)(x[u] / E.bandwidth);
            }
            E.mv_key[f] = (bucket << 27) | ((unsigned)k << 23) | (unsigned)i;
            int nx, ny, bw, bh;
            const bool in_board = mover_target(E, G, av, x[u], y[u], dir[u], turn, nx, ny, bw, bh);
            E.mv_nx[f] = nx; E.mv_ny[f] = ny;
            if (!in_board) {
                E.mv_state[f] = MV_OOB;
                continue;
            }
            if (bw == 1 && bh == 1) { cell[u] = ny * E.W + nx; node[u] = fs * E.max_body; continue; }
            // larger bodies: walls / food under the footprint (is_blank_area, Map.cc:461-465), then queue on every cell
            bool wall = false;
            for (int bx = 0; bx < bw; ++bx)
                for (int by = 0; by < bh; ++by)
                    if (R.occ[(ny + by) * E.W + nx + bx] <= OCC_WALL) wall = true;
            // with absorbing types around, a wall-blocked mover may still bump into an absorber: keep it in the relaxation
            if (wall && (turn || !E.any_absorb)) { E.mv_state[f] = MV_STATIC_FAIL; continue; }
            E.mv_state[f] = MV_PENDING_FAIL;
            int ci = 0;
            for (int bx = 0; bx < bw; ++bx)
                for (int by = 0; by < bh; ++by, ++ci) {
                    int nd = fs * E.max_body + ci;
                    E.cl_next[R.nb + nd] = atomic_exch(&R.claim[(ny + by) * E.W + nx + bx], nd);
                }
        }
        // request 2: occupancy of the single target cells
        int occv[U];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) occv[u] = cell[u] >= 0 ? R.occ[cell[u]] : 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) {
            if (cell[u] < 0) continue;
            const long f = R.sb + node[u] / E.max_body;
            if (occv[u] <= OCC_WALL && (turn || !E.any_absorb)) { E.mv_state[f] = MV_STATIC_FAIL; cell[u] = -1; }
            else E.mv_state[f] = MV_PENDING_FAIL;
        }
        // request 3: the claim exchanges
        int prev[U];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) prev[u] = cell[u] >= 0 ? atomic_exch(&R.claim[cell[u]], node[u]) : -1;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int u = 0; u < U; ++u) if (cell[u] >= 0) E.cl_next[R.nb + node[u]] = prev[u];
    }
}

// who stands on cell (cx,cy) when the mover with order key `key` takes its turn?  -1 = nobody.
// `self` (local flat id) is ignored.  Reads mover states with volatile loads.
// `stable` is cleared when the answer rests on the state of a mover that a later sweep may still change (an
// earlier-keyed mover that has not been refused for good): answers that stay stable need no re-evaluation.
MG_HD int occupant_at_turn(const EngineDev &E, const ArenaRef &R, unsigned curmask, int cx, int cy, unsigned key, int self, bool turn,
                           bool &stable) {
    int cell = cy * E.W + cx;
    int o = R.occ[cell];
    const int head = R.claim[cell];                   // issued with the occupancy load: one round trip, not two
    if (o >= 0) {
        int fo = lflat(E, o);
        if (fo != self) {
            const unsigned char so = ld_volatile(&E.mv_state[R.sb + fo]);
            if (so >= MV_PENDING_FAIL && E.mv_key[R.sb + fo] < key) stable = false;   // PENDING_FAIL / OK / ABSORBED / SKIPPED may flip
            if (so == MV_ABSORBED && E.mv_key[R.sb + fo] < key) goto claimants;     // it died into an absorber: cell vacated
            bool left = so == MV_OK && E.mv_key[R.sb + fo] < key;
            if (left) {
                const GroupDev &GO = E.grp[code_group(o)];
                int ox = E.mv_nx[R.sb + fo], oy = E.mv_ny[R.sb + fo], ow, oh;
                mover_dims(E, GO, cur_soa(E, curmask, code_group(o)), gidx(E, R.a, code_group(o), code_index(o)), turn, ow, oh);
                if (cx >= ox && cx < ox + ow && cy >= oy && cy < oy + oh) left = false;
            }
            if (!left) return fo;
        }
    }
claimants:
    for (int node = head; node != -1; node = E.cl_next[R.nb + node]) {
        int fm = node_owner(E, node);
        if (fm != self && E.mv_key[R.sb + fm] < key) {
            stable = false;
            if (ld_volatile(&E.mv_state[R.sb + fm]) == MV_OK) return fm;
        }
    }
    return -1;
}

// phase 7 (swept until stable): a mover succeeds iff all its target cells are free at its turn
// (Map::do_move / is_blank_area, Map.cc:313-358,454-470)
template <class Ctx>
MG_HD bool phase_move_relax(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord, bool turn,
                            SettledMask &settled) {
    ArenaRef R = arena_ref(E, a);
    bool changed = false;
    // `settled` is private to the thread and lives across the sweeps of one relaxation: bit j = the thread's j-th
    // mover got an answer that no later sweep can change (occupant_at_turn's `stable`), so it is not looked at again.
    // A thread visits the same movers in the same order in every sweep.
    int j = -1;
    for (int idx = c.tid(); idx < ord.cnt; idx += c.nth()) {
        ++j;
        if (settled.get(j)) continue;
        int k, i; enum_locate(ord, idx, k, i);
        int g = ord.grp[k];
        const GroupDev &G = E.grp[g];
        int fs = G.foff + i;
        long f = R.sb + fs;
        unsigned char st = E.mv_state[f];
        if (st != MV_PENDING_FAIL && st != MV_OK && st != MV_ABSORBED && st != MV_SKIPPED) continue;
        unsigned key = E.mv_key[f];
        int nx = E.mv_nx[f], ny = E.mv_ny[f];
        int bw, bh;                                   // footprint being claimed
        mover_dims(E, G, cur_soa(E, S.curmask, g), gidx(E, a, g, i), turn, bw, bh);
        bool ok = true;
        unsigned char ns;
        bool skipped = false;
        if (G.can_absorb && !turn) {
            // an absorber that swallowed somebody earlier in this move phase is `absorbed` by the time its own turn
            // comes and is skipped (GridWorld.cc:581): whoever bumped into it queued on one of its current cells
            const AgentSoA &sm = cur_soa(E, S.curmask, g);
            const long gm = gidx(E, a, g, i);
            const int mycode = code_make(g, i);
            const int x0 = sm.x[gm], y0 = sm.y[gm];
            for (int bx = 0; bx < bw && !skipped; ++bx)
                for (int by = 0; by < bh && !skipped; ++by)
                    for (int node = R.claim[(y0 + by) * E.W + x0 + bx]; node != -1; node = E.cl_next[R.nb + node]) {
                        const int fm = node_owner(E, node);
                        if (fm != fs && E.mv_key[R.sb + fm] < key && ld_volatile(&E.mv_state[R.sb + fm]) == MV_ABSORBED &&
                            ld_volatile(&E.tgt[R.sb + fm]) == mycode) { skipped = true; break; }
                    }
        }
        if (skipped) {
            ns = MV_SKIPPED;
        } else if (!E.any_absorb || turn) {
            bool stable = true;
            for (int bx = 0; bx < bw && ok; ++bx)
                for (int by = 0; by < bh && ok; ++by)
                    if (occupant_at_turn(E, R, S.curmask, nx + bx, ny + by, key, fs, turn, stable) != -1) ok = false;
            ns = ok ? MV_OK : MV_PENDING_FAIL;
            if (stable) settled.set(j);
        } else {
            // Map::do_move with can_absorb types (Map.cc:334-349): the first other agent in the footprint decides
            int hit = -1, hit_cell = -1;
            for (int bx = 0; bx < bw; ++bx)
                for (int by = 0; by < bh; ++by) {
                    const int cell = (ny + by) * E.W + nx + bx;
                    if (R.occ[cell] <= OCC_WALL) { ok = false; continue; }
                    bool unused = true;
                    const int o = occupant_at_turn(E, R, S.curmask, nx + bx, ny + by, key, fs, false, unused);
                    if (o != -1) { ok = false; if (hit == -1) { hit = o; hit_cell = cell; } }
                }
            ns = ok ? MV_OK : MV_PENDING_FAIL;
            if (!ok && hit != -1) {
                int hg = 0;
                while (hg + 1 < E.G && hit >= E.grp[hg + 1].foff) ++hg;
                const int hcode = code_make(hg, hit - E.grp[hg].foff);
                if (E.grp[hg].can_absorb &&
                    !(cur_soa(E, S.curmask, hg).flags[gidx(E, a, hg, code_index(hcode))] & FLAG_ABSORBED)) {
                    // absorbed already by an earlier mover of this step?  every mover that bumps into `hit` queues on hit_cell
                    bool taken = false;
                    for (int node = R.claim[hit_cell]; node != -1 && !taken; node = E.cl_next[R.nb + node]) {
                        const int fm = node_owner(E, node);
                        if (fm != fs && E.mv_key[R.sb + fm] < key && ld_volatile(&E.mv_state[R.sb + fm]) == MV_ABSORBED &&
                            ld_volatile(&E.tgt[R.sb + fm]) == hcode) taken = true;
                    }
                    if (!taken) {
                        // the absorber's identity is part of this mover's state: later movers compare against it
                        if (st == MV_ABSORBED && ld_volatile(&E.tgt[f]) != hcode) changed = true;
                        st_volatile(&E.tgt[f], hcode);
                        ns = MV_ABSORBED;
                    }
                }
            }
        }
        if (ns != st) { st_volatile(&E.mv_state[f], ns); changed = true; }
    }
    return changed;
}

// phase 8: losers record what they bumped into (Map::get_collide, Map.cc:486-501; GridWorld sets
// OP_COLLIDE, Map.cc:350-353)
template <class Ctx>
MG_HD void phase_move_collide(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord) {
    ArenaRef R = arena_ref(E, a);
    int ok_ct = 0, blocked = 0;
    for (int idx = c.tid(); idx < ord.cnt; idx += c.nth()) {
        int k, i; enum_locate(ord, idx, k, i);
        int g = ord.grp[k];
        const GroupDev &G = E.grp[g];
        int fs = G.foff + i;
        long f = R.sb + fs;
        unsigned char st = E.mv_state[f];
        if (st == MV_OK) { ++ok_ct; continue; }
        if (st == MV_NONE || st == MV_SKIPPED) continue;
        ++blocked;
        if (st == MV_OOB) continue;
        if (st == MV_ABSORBED) {                  // Map.cc:341-349: the absorber doubles its hp, the mover disappears
            const int obj = E.tgt[f];
            const int og = code_group(obj);
            const AgentSoA &so = cur_soa(E, S.curmask, og);
            const long oi = gidx(E, a, og, code_index(obj));
            so.flags[oi] |= FLAG_ABSORBED;
            const float hp2 = so.hp[oi] * 2;
            so.hp[oi] = hp2;
            {                                     // the absorber's cells show its new hp (if it moves, the fill rewrites them)
                int obw, obh;
                body_dims(E.grp[og], agent_dir(E, so, oi), obw, obh);
                show_body(E, a, og, E.grp[og], so.x[oi], so.y[oi], obw, obh, hp2);
            }
            const AgentSoA &s = cur_soa(E, S.curmask, g);
            const long gi = gidx(E, a, g, i);
            s.flags[gi] |= FLAG_DEAD;             // set_dead(true): no dead_penalty, dead_ct untouched (reference quirk)
            R.hdr->any_dead = 1;
            s.last_op[gi] = OP_COLLIDE;
            s.op_obj[gi] = obj;
            continue;
        }
        unsigned key = E.mv_key[f];
        int nx = E.mv_nx[f], ny = E.mv_ny[f];
        int bw, bh;
        mover_dims(E, G, cur_soa(E, S.curmask, g), gidx(E, a, g, i), false, bw, bh);
        int hit = -1;
        bool unused = true;
        for (int bx = 0; bx < bw && hit == -1; ++bx)
            for (int by = 0; by < bh && hit == -1; ++by)
                hit = occupant_at_turn(E, R, S.curmask, nx + bx, ny + by, key, fs, false, unused);
        if (hit != -1) {
            int hg = 0;
            while (hg + 1 < E.G && hit >= E.grp[hg + 1].foff) ++hg;
            if (E.grp[hg].can_absorb) continue;  // bumping into an already absorbed absorber records nothing
            const AgentSoA &s = cur_soa(E, S.curmask, g);
            long gi = gidx(E, a, g, i);
            s.last_op[gi] = OP_COLLIDE;
            s.op_obj[gi] = code_make(hg, hit - E.grp[hg].foff);
        }
    }
    c.add_count(E, CNT_MOVES_OK, ok_ct);
    c.add_count(E, CNT_MOVES_BLOCKED, blocked);
}

// phase 9a: winners vacate their old cells
template <class Ctx>
MG_HD void phase_move_clear(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord) {
    ArenaRef R = arena_ref(E, a);
    for (int idx = c.tid(); idx < ord.cnt; idx += c.nth()) {
        int k, i; enum_locate(ord, idx, k, i);
        int g = ord.grp[k];
        const GroupDev &G = E.grp[g];
        long f = R.sb + G.foff + i;
        if (E.mv_state[f] != MV_OK && E.mv_state[f] != MV_ABSORBED) continue;
        const AgentSoA &s = cur_soa(E, S.curmask, g);
        long gi = gidx(E, a, g, i);
        int x = s.x[gi], y = s.y[gi], bw, bh;
        body_dims(G, agent_dir(E, s, gi), bw, bh);
        for (int bx = 0; bx < bw; ++bx)
            for (int by = 0; by < bh; ++by) {
                R.occ[(y + by) * E.W + x + bx] = OCC_EMPTY;
                kind_set(E, a, x + bx, y + by, 0);
            }
    }
}

// phase 9b: winners occupy their new cells; every queued mover unhooks its claimant nodes
template <class Ctx>
MG_HD void phase_move_fill(Ctx &c, const EngineDev &E, const StepArgs &S, int a, const GroupEnum &ord, bool turn) {
    ArenaRef R = arena_ref(E, a);
    for (int idx = c.tid(); idx < ord.cnt; idx += c.nth()) {
        int k, i; enum_locate(ord, idx, k, i);
        int g = ord.grp[k];
        const GroupDev &G = E.grp[g];
        long f = R.sb + G.foff + i;
        unsigned char st = E.mv_state[f];
        if (turn && st != MV_NONE) { E.mv_state[f] = MV_NONE; E.mv_key[f] = MVKEY_NONE; }   // the move phase starts from a clean slate
        if (st != MV_OK && st != MV_PENDING_FAIL && st != MV_ABSORBED && st != MV_SKIPPED) continue;
        int nx = E.mv_nx[f], ny = E.mv_ny[f];
        bool ok = st == MV_OK;
        int code = code_make(g, i);
        const AgentSoA &s = cur_soa(E, S.curmask, g);
        long gi = gidx(E, a, g, i);
        int bw, bh;
        mover_dims(E, G, s, gi, turn, bw, bh);
        const float hp = ok ? s.hp[gi] : 0.0f;
        const bool full = hp == G.max_hp;
        const unsigned char kd = kind_agent(g, full);
        const float hpv = hp / G.max_hp;
        for (int bx = 0; bx < bw; ++bx)
            for (int by = 0; by < bh; ++by) {
                int cell = (ny + by) * E.W + nx + bx;
                R.claim[cell] = -1;
                if (ok) { R.occ[cell] = code; kind_set(E, a, nx + bx, ny + by, kd); if (!full) hpn_set(E, a, nx + bx, ny + by, hpv); }
            }
        if (ok) {
            s.x[gi] = nx; s.y[gi] = ny;
            if (turn) s.dir[gi] = (unsigned char)turned_dir(s.dir[gi], s.act[gi]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// phase 10: reward rules (reference GridWorld::calc_reward / calc_rule / calc_event_node,
// GridWorld.cc:681-692, RewardEngine.cc:216-443)
//
// Group-quantified event nodes ('all' subject, RewardEngine.cc:223-233,294-343): "every agent of the group,
// dead-but-unculled ones included, satisfies the predicate".  Reduced once per step and arena into
// ArenaHdr::allq_*; the binary ops (attack/kill/collide) compare every agent with agent 0 of the group, so
// the leaf only has to compare agent 0's op_obj with the bound object.
template <class Ctx>
MG_HD void phase_rule_allq(Ctx &c, const EngineDev &E, const StepArgs &S, int a) {
    ArenaRef R = arena_ref(E, a);
    for (int r = 0; r < E.n_rules; ++r) {
        const RuleDev &Ru = E.rules[r];
        for (int p = 0; p < Ru.n_prog; ++p) {
            const RuleInstr &I = Ru.prog[p];
            if (I.role_a != ROLE_ALL) continue;
            const int g = I.all_group, n = E.n[g * E.A + a];
            const AgentSoA &s = cur_soa(E, S.curmask, g);
            const long b0 = gidx(E, a, g, 0);
            int viol = 0, mn = 0x7fffffff, mx = -0x7fffffff - 1;
            int obj0 = -1, vertical = 0, base = 0;
            if (n > 0 && (I.op == OP_KILL || I.op == OP_ATTACK || I.op == OP_COLLIDE)) obj0 = s.op_obj[b0];
            if (I.op == OP_IN_A_LINE && n >= 2) {              // RewardEngine.cc:262-292
                int dx = s.x[b0] - s.x[b0 + 1], dy = s.y[b0] - s.y[b0 + 1];
                if (dx == 0 && dy != 0) { vertical = 1; base = s.x[b0]; }
                else if (dx != 0 && dy == 0) { vertical = 0; base = s.y[b0]; }
                else viol = 1;
            }
            for (int i = c.tid(); i < n; i += c.nth()) {
                const long gi = b0 + i;
                switch (I.op) {
                    case OP_KILL: case OP_ATTACK: case OP_COLLIDE:
                        viol |= !(s.last_op[gi] == I.op && s.op_obj[gi] == obj0); break;
                    case OP_DIE: viol |= !(s.flags[gi] & FLAG_DEAD); break;
                    case OP_AT: viol |= !(s.x[gi] == I.i0 && s.y[gi] == I.i1); break;
                    case OP_IN: { int x = s.x[gi], y = s.y[gi];
                        viol |= !(x > I.i0 && x < I.i2 && y > I.i1 && y < I.i3); break; }
                    case OP_IN_A_LINE: {
                        int fix = vertical ? s.x[gi] : s.y[gi], var = vertical ? s.y[gi] : s.x[gi];
                        viol |= fix != base;
                        mn = var < mn ? var : mn; mx = var > mx ? var : mx; break; }
                    default: break;
                }
            }
            if (viol) atomic_or(&R.hdr->allq_viol[I.allq], 1);
            if (I.op == OP_IN_A_LINE && mn <= mx) { atomic_min(&R.hdr->allq_min[I.allq], mn); atomic_max(&R.hdr->allq_max[I.allq], mx); }
        }
    }
}

// calc_event_node on the bound entities (postfix program; no short-circuit needed: nodes have no side effects)
MG_HD bool rule_eval(const EngineDev &E, const ArenaRef &R, const RuleInstr *prog, int n_prog, unsigned curmask, int a, const int *codes) {
    bool stack[MG_MAX_PROG];
    int sp = 0;
    for (int p = 0; p < n_prog; ++p) {
        const RuleInstr &I = prog[p];
        switch (I.op) {
            case OP_AND: { bool b = stack[--sp]; bool x = stack[--sp]; stack[sp++] = x && b; break; }
            case OP_OR:  { bool b = stack[--sp]; bool x = stack[--sp]; stack[sp++] = x || b; break; }
            case OP_NOT: { stack[sp - 1] = !stack[sp - 1]; break; }
            default: {
                bool v = false;
                if (I.role_a == ROLE_ALL) {
                    const int g = I.all_group, n = E.n[g * E.A + a];
                    const bool clean = R.hdr->allq_viol[I.allq] == 0;
                    if (I.op == OP_KILL || I.op == OP_ATTACK || I.op == OP_COLLIDE)
                        v = n == 0 || (clean && cur_soa(E, curmask, g).op_obj[gidx(E, a, g, 0)] == codes[I.role_b]);
                    else if (I.op == OP_IN_A_LINE)
                        v = n < 2 || (clean && R.hdr->allq_max[I.allq] - R.hdr->allq_min[I.allq] + 1 == n);
                    else
                        v = clean;
                } else {
                    int ca = codes[I.role_a];
                    int ga = code_group(ca);
                    const AgentSoA &s = cur_soa(E, curmask, ga);
                    long gi = gidx(E, a, ga, code_index(ca));
                    if (I.op == OP_KILL || I.op == OP_ATTACK || I.op == OP_COLLIDE) {
                        v = s.last_op[gi] == I.op && s.op_obj[gi] == codes[I.role_b];
                    } else if (I.op == OP_DIE) {
                        v = (s.flags[gi] & FLAG_DEAD) != 0;
                    } else if (I.op == OP_AT) {
                        v = s.x[gi] == I.i0 && s.y[gi] == I.i1;
                    } else if (I.op == OP_IN) {
                        int x = s.x[gi], y = s.y[gi];
                        v = x > I.i0 && x < I.i2 && y > I.i1 && y < I.i3;
                    }
                }
                stack[sp++] = v;
            }
        }
    }
    return sp > 0 && stack[sp - 1];
}

// AgentSymbol::bind_with_check (RewardEngine.cc:14-23) for an inferred object
// Agent::get_index() as the reference keeps it: the position after the last clear_dead, 0 for agents added since
MG_HD int stale_index(const ArenaRef &R, int code) {
    int i = code_index(code);
    return i < R.hdr->n_cull[code_group(code)] ? i : 0;
}
MG_HD bool rule_bind(const ArenaRef &R, int obj, int group, int index) {
    if (obj < 0) return false;
    if (code_group(obj) != group) return false;
    return index == -1 || stale_index(R, obj) == index;
}

MG_HD void rule_pay(const EngineDev &E, const ArenaRef &R, const RuleRecv *recv, int n_recv, unsigned curmask, int a, const int *codes) {
    for (int q = 0; q < n_recv; ++q) {
        const RuleRecv &rc = recv[q];
        if (rc.role == ROLE_GROUP) {
            atomic_addf(&R.hdr->grp_reward[rc.group], rc.value);
        } else {
            int cd = codes[rc.role];
            if (cd < 0) continue;
            int gg = code_group(cd);
            atomic_addf(&cur_soa(E, curmask, gg).next_reward[gidx(E, a, gg, code_index(cd))], rc.value);
        }
    }
}

// One rule: the reference's depth-first binding (calc_rule, RewardEngine.cc:373-443) flattened.  The 'all' and
// fixed-index levels bind the same entities whatever the enclosing loops hold, so they are resolved first (a
// failed bind there kills the rule for this step); the 'any' levels span a mixed-radix index space that the team
// strides over -- one level for the shipped games, two for double_attack, O(n^k) in general exactly like the
// reference.  An agent cannot fill two 'any' levels at once (be_involved, RewardEngine.cc:401-403).
template <class Ctx>
MG_HD void phase_reward_rule(Ctx &c, const EngineDev &E, const StepArgs &S, int a, int r, const GroupEnum &all) {
    ArenaRef R = arena_ref(E, a);
    const RuleDev &Ru = E.rules[r];                     // in HBM: only touched by candidates that pass the bind
    const RuleHot H = E.rule_hot[r];
    if (H.shape == RULE_DEAD) return;
    int codes[2 * MG_MAX_IN];
    bool any = false;
    const bool small = r < MG_HOT_RULES && E.rule_small[r].n_prog >= 0;
    const RuleInstr *prog = small ? E.rule_small[r].prog : Ru.prog;
    const RuleRecv *recv = small ? E.rule_small[r].recv : Ru.recv;
    const int n_prog = small ? E.rule_small[r].n_prog : Ru.n_prog, n_recv = small ? E.rule_small[r].n_recv : Ru.n_recv;
    if (H.shape == RULE_ONE_ANY) {
        // one free subject, optionally binding its op_obj: every shipped game's rules.  One thread per subject; the
        // only global round trip before the verdict is the subject's op_obj.
        const int n = all.pre[H.group + 1] - all.pre[H.group];
        const AgentSoA &s = cur_soa(E, S.curmask, H.group);
        const long b0 = gidx(E, a, H.group, 0);
        for (int i = c.tid(); i < n; i += c.nth()) {
            codes[1] = -1;
            if (H.has_obj) {
                const int obj = s.op_obj[b0 + i];
                const int lop = H.simple_op ? (int)s.last_op[b0 + i] : 0;    // requested together with op_obj
                if (!rule_bind(R, obj, H.obj_group, H.obj_index)) continue;
                if (H.simple_op && lop != H.simple_op) continue;
                codes[1] = obj;
            }
            codes[0] = code_make(H.group, i);
            if (!H.simple_op && !rule_eval(E, R, prog, n_prog, S.curmask, a, codes)) continue;
            any = true;
            rule_pay(E, R, recv, n_recv, S.curmask, a, codes);
        }
        if (any) R.hdr->rule_trig[r] = 1;
        return;
    }
    for (int k = 0; k < 2 * MG_MAX_IN; ++k) codes[k] = -1;
    for (int k = 0; k < Ru.n_in; ++k) {
        const RuleInput &in = Ru.in[k];
        if (in.kind == IN_ANY) continue;
        const int n = E.n[in.group * E.A + a];
        int who = 0;
        if (in.kind == IN_FIXED) {
            if (in.index >= n) return;
            who = in.index;
            codes[2 * k] = code_make(in.group, who);
        }
        if (in.has_obj) {
            if (n == 0) return;                       // 'all': the first agent of the group infers (:414-421)
            int obj = cur_soa(E, S.curmask, in.group).op_obj[gidx(E, a, in.group, who)];
            if (!rule_bind(R, obj, in.obj_group, in.obj_index)) return;
            codes[2 * k + 1] = obj;
        }
    }
    long long combos = 1;
    int radix[MG_MAX_IN];
    for (int q = 0; q < Ru.n_any; ++q) {
        radix[q] = E.n[Ru.in[Ru.any_in[q]].group * E.A + a];
        combos *= radix[q];
    }
    for (long long p = c.tid(); p < combos; p += c.nth()) {
        long long rest = p;
        bool ok = true;
        for (int q = Ru.n_any - 1; q >= 0; --q) {
            const int k = Ru.any_in[q];
            const RuleInput &in = Ru.in[k];
            const int i = (int)(rest % radix[q]);
            rest /= radix[q];
            codes[2 * k] = code_make(in.group, i);
            if (in.has_obj) {
                int obj = cur_soa(E, S.curmask, in.group).op_obj[gidx(E, a, in.group, i)];
                if (!rule_bind(R, obj, in.obj_group, in.obj_index)) { ok = false; break; }
                codes[2 * k + 1] = obj;
            }
        }
        if (!ok) continue;
        for (int q = 1; q < Ru.n_any && ok; ++q)
            for (int q2 = 0; q2 < q; ++q2)
                if (codes[2 * Ru.any_in[q]] == codes[2 * Ru.any_in[q2]]) ok = false;
        if (!ok) continue;
        if (!rule_eval(E, R, prog, n_prog, S.curmask, a, codes)) continue;
        any = true;
        rule_pay(E, R, recv, n_recv, S.curmask, a, codes);
    }
    if (any) R.hdr->rule_trig[r] = 1;             // every writer stores the same byte
}

// phase 11: game-over check (GridWorld.cc:618-630) and rng commit
template <class Ctx>
MG_HD void phase_done(Ctx &c, const EngineDev &E, int a) {
    if (c.tid() != 0) return;
    ArenaRef R = arena_ref(E, a);
    int live = 0;
    for (int g = 0; g < E.G; ++g)
        if (E.n[g * E.A + a] - E.dead_ct[g * E.A + a] > 0) ++live;
    int done = live < E.G;
    for (int r = 0; r < E.n_rules; ++r)
        if (E.rule_hot[r].terminal && R.hdr->rule_trig[r]) done = 1;
    R.hdr->done = done;
    // bit 1 tells the host whether this arena holds dead agents: when no arena does, clear_dead cannot change a
    // count and the host skips re-reading the offsets (one blocking copy less per step)
    E.done[a] = done | (R.hdr->any_dead ? 2 : 0);
    R.hdr->rng = R.hdr->rng_next;
}

// MG_PHASE_TIMING (profiling variants only, built with -DMG_PHASE_TIMING): thread 0 of the team
// stamps the SM clock after every phase of the first arenas into a device array the profiling script reads back
#if defined(MG_PHASE_TIMING) && defined(__CUDA_ARCH__)
#define MG_MARK(k) do { if (c.tid() == 0 && a < 8) mg_phase_clock[a * 32 + (k)] = clock64(); } while (0)
#define MG_MARKV(k, v) do { if (c.tid() == 0 && a < 8) mg_phase_clock[a * 32 + (k)] = (v); } while (0)
#else
#define MG_MARK(k) do { } while (0)
#define MG_MARKV(k, v) do { (void)(v); } while (0)
#endif

// relaxation driver: sweep until a full sweep changes nothing.  One team barrier per sweep; the
// rotating flag triple makes the reset of the next flag race-free (DESIGN.md §4.3).  The flags live where the
// team can see them cheaply: shared memory for a CTA team, the arena header in HBM for the grid team.
template <class Ctx, class Sweep>
MG_HD int relax_until_stable(Ctx &c, int *flags, Sweep sweep, int a = 0, int mark = -1) {
    if (c.tid() == 0) { st_volatile(&flags[0], 0); st_volatile(&flags[1], 0); st_volatile(&flags[2], 0); }
    c.sync();
    for (int it = 0;; ++it) {
        int cur = it % 3, nxt = (it + 1) % 3;
        if (c.tid() == 0) st_volatile(&flags[nxt], 0);
        if (sweep()) st_volatile(&flags[cur], 1);
        c.sync();
        if (it == 0 && mark >= 0) { MG_MARK(mark); }
        if (!ld_volatile(&flags[cur])) return it + 1;
    }
}

// the whole step for one arena (reference GridWorld::step, GridWorld.cc:456-631)
template <class Ctx>
MG_HD void run_step(Ctx &c, const EngineDev &E, const StepArgs &S, int a) {
    ArenaHdr *hdr = E.hdr + a;
    int *flags = c.flags(hdr);
    // group sizes are constant during a step: read them once, into storage every thread of the CTA can index
    // cheaply (shared memory on the device: a dynamically indexed per-thread struct would live in local memory)
    GroupEnum *en = c.enums();
    if (c.is_cta_leader()) { enum_all(E, a, en[0]); enum_order(E, S, a, en[1]); }
    c.sync_cta();
    const GroupEnum &all = en[0], &ord = en[1];
    MG_MARK(0);
    phase_init(c, E, S, a, all, ord);
    c.sync();
    MG_MARK(1);
    int n_attack = phase_attack_scan(c, E, S, a, ord);
    c.sync();
    MG_MARK(2);
    if (n_attack > 0) {
        phase_rng(c, E, a, n_attack);
        c.sync();
        MG_MARK(3);
        phase_rank_target(c, E, S, a, n_attack);
        MG_MARK(4);
        int sweeps = relax_until_stable(c, flags, [&]() { return phase_attack_relax(c, E, S, a, all); });
        MG_MARKV(14, sweeps);
    }
    MG_MARK(5);
    phase_attack_apply_starve(c, E, S, a, all);
    c.sync();
    MG_MARK(6);
    if (E.food_mode && n_attack > 0) {
        phase_food_commit(c, E, S, a, all, false);
        c.sync();
        phase_food_commit(c, E, S, a, all, true);
        c.sync();
    }
    if (E.turn_mode) {                                   // GridWorld.cc:544-571: all turns, then all moves
        phase_move_register(c, E, S, a, ord, true);
        SettledMask turn_settled;
        relax_until_stable(c, flags, [&]() { return phase_move_relax(c, E, S, a, ord, true, turn_settled); });
        phase_move_clear(c, E, S, a, ord);
        c.sync();
        phase_move_fill(c, E, S, a, ord, true);
        c.sync();
    }
    phase_move_register(c, E, S, a, ord, false);
    MG_MARK(7);
    SettledMask mv_settled;
    int mv_sweeps = relax_until_stable(c, flags, [&]() { return phase_move_relax(c, E, S, a, ord, false, mv_settled); }, a, 16);
    MG_MARKV(15, mv_sweeps);
    MG_MARK(8);
    phase_move_collide(c, E, S, a, ord);
    c.sync();
    MG_MARK(9);
    phase_move_clear(c, E, S, a, ord);
    c.sync();
    MG_MARK(10);
    phase_move_fill(c, E, S, a, ord, false);
    c.sync();
    MG_MARK(11);
    if (E.n_allq > 0) {
        phase_rule_allq(c, E, S, a);
        c.sync();
    }
    for (int r = 0; r < E.n_rules; ++r) {
        phase_reward_rule(c, E, S, a, r, all);
        c.sync();
    }
    MG_MARK(12);
    phase_done(c, E, a);
    c.flush_counts(E);
    c.sync();
    MG_MARK(13);
}

// clear_dead for one arena: stable compaction of every group into the other SoA buffer
// (reference GridWorld::clear_dead, GridWorld.cc:633-665, Agent::init_reward GridWorld.h:168-174)
template <class Ctx>
MG_HD void run_cull(Ctx &c, const EngineDev &E, unsigned curmask, int a) {
    ArenaRef R = arena_ref(E, a);
    for (int g = 0; g < E.G; ++g) {
        const GroupDev &G = E.grp[g];
        const AgentSoA &src = G.soa[(curmask >> g) & 1u];
        const AgentSoA &dst = G.soa[((curmask >> g) & 1u) ^ 1u];
        int n = E.n[g * E.A + a];
        c.sync();
        auto pred = [&](int i) -> int { return (src.flags[gidx(E, a, g, i)] & FLAG_DEAD) ? 0 : 1; };
        auto emit = [&](int i, int j) {
            long si = gidx(E, a, g, i), di = gidx(E, a, g, j);
            int x = src.x[si], y = src.y[si];
            dst.x[di] = x; dst.y[di] = y;
            dst.hp[di] = src.hp[si];
            dst.act[di] = src.act[si];
            dst.id[di] = src.id[si];
            dst.last_reward[di] = src.next_reward[si];
            dst.next_reward[di] = G.step_reward;
            dst.op_obj[di] = -1;
            dst.last_op[di] = OP_NULL;
            dst.flags[di] = src.flags[si];
            dst.dir[di] = src.dir[si];
            if (i != j) {
                int code = code_make(g, j), bw, bh;
                body_dims(G, agent_dir(E, src, si), bw, bh);
                for (int bx = 0; bx < bw; ++bx)
                    for (int by = 0; by < bh; ++by)
                        R.occ[(y + by) * E.W + x + bx] = code;
            }
        };
        int total = c.scan(n, pred, emit);
        c.sync();
        if (c.tid() == 0) {
            E.n[g * E.A + a] = total;
            E.dead_ct[g * E.A + a] = 0;
            R.hdr->grp_reward[g] = 0.0f;
            R.hdr->n_cull[g] = total;
            R.hdr->any_dead = 0;
        }
    }
    c.sync();
}

}  // namespace mg
