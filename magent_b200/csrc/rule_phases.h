// rule_phases.h -- the built-in scripted opponents: the per-agent decision behind magent_b200_rule_actions and
// magent_b200_get_rule_actions(_slots).
//
// For agent i of group g and a target group t (t == g allowed), on the state as it is now (include/magent_b200_ext.h has
// the full statement):
//   rush  1. attack: among the legal attacks (action_legal) whose aimed cell (attack_cell_from) holds an agent of t other
//            than i, the one whose target has the lowest hp; ties to the lowest action;
//         2. approach: else, when i sees an agent of t, the legal move (k < n_move) whose moved footprint (mover_target)
//            is nearest (nbr_box_d2) to the cell get_neighbours(g, of=t, k=1) lists for i; ties to the lowest action;
//         3. else the action random_legal_actions would draw for i (legal_draw).
//   flee  2 with the farthest move instead, else 3.
// A dead agent and an agent without a legal action take action 0.  One function, rule_action(), serves the CUDA kernels
// (backend_cuda.cu rule_actions_kernel, rule_actions_slots_kernel) and the test emulation (tests/emu/rule_actions_emu.cc).
#pragma once
#include "mask_phases.h"
#include "nbr_phases.h"

namespace mg {

enum { RULE_RUSH = 0, RULE_FLEE = 1 };

// step 1: the legal attack on the agent of group t with the lowest hp, or -1
MG_HD int rule_attack(const EngineDev &E, unsigned curmask, int a, const int *occ, int g, int t, const MaskAgent &m) {
    const GroupDev &G = E.grp[g];
    const float *hp = cur_soa(E, curmask, t).hp;
    int best = -1;
    float best_hp = 0.0f;
    for (int k = G.attack_base; k < G.n_action; ++k) {
        if (!action_legal(E, curmask, a, occ, g, m, k)) continue;
        int tx, ty;
        attack_cell_from(E, G, k, m.x, m.y, m.dir, tx, ty);          // on the board: action_legal checked
        const int c = occ[ty * E.W + tx];
        if (c < 0 || code_group(c) != t || c == m.code) continue;
        const float v = hp[gidx(E, a, t, code_index(c))];
        if (best < 0 || v < best_hp) { best = k; best_hp = v; }
    }
    return best;
}

// The map cell (cx, cy) that magent_b200_get_neighbours(g, of = t, k = 1) lists for agent m: the first cell of its view
// LUT (key order, struct NbrCell) that lists a neighbour of group t.  False when it sees no agent of t.
MG_HD bool rule_nearest(const EngineDev &E, const NbrCell *lut, unsigned curmask, int a, int g, int t, const MaskAgent &m,
                        int &cx, int &cy) {
    NbrObserver o;
    o.x = m.x; o.y = m.y; o.dir = m.dir; o.code = m.code; o.flags = m.flags;
    const int n = E.grp[g].view_count;
    const NbrCell *l = lut + (E.turn_mode ? m.dir * n : 0);
    const unsigned char *kp = E.kind + (long)a * E.kplane + (long)(m.y + E.kpad) * E.kw + m.x + E.kpad;
    for (int q = 0; q < n; ++q) {
        if (!nbr_kind_of(kp[ld_ro(&l[q].off)], t)) continue;
        const int d = ld_ro(&l[q].delta);
        const int x = m.x + (short)(d & 0xffff), y = m.y + (d >> 16);
        if (nbr_nearest_at(E, curmask, a, g, t, o, x, y, ld_ro(&l[q].key)) >= 0) { cx = x; cy = y; return true; }
    }
    return false;
}

// step 2: the legal move whose moved footprint is nearest to (flee: farthest from) cell (cx, cy), or -1
MG_HD int rule_move(const EngineDev &E, unsigned curmask, int a, const int *occ, int g, const MaskAgent &m, int cx, int cy,
                    bool flee) {
    const GroupDev &G = E.grp[g];
    int best = -1, best_d = 0;
    for (int k = 0; k < G.n_move; ++k) {
        if (!action_legal(E, curmask, a, occ, g, m, k)) continue;
        int nx, ny, bw, bh;
        mover_target(E, G, k, m.x, m.y, m.dir, false, nx, ny, bw, bh);
        const int d = nbr_box_d2(bw, bh, cx - nx, cy - ny);
        if (best < 0 || (flee ? d > best_d : d < best_d)) { best = k; best_d = d; }
    }
    return best;
}

// step 3: the action magent_b200_random_legal_actions draws for agent m at ABI ordinal o (seed and steps as legal_draw
// takes them); 0 without a legal action
MG_HD int rule_fallback(const EngineDev &E, unsigned curmask, int a, const int *occ, int g, const MaskAgent &m,
                        unsigned long long seed, long long steps, int o) {
    const int na = E.grp[g].n_action;
    int n_legal = 0;
    for (int k = 0; k < na; ++k) n_legal += action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
    if (n_legal == 0) return 0;
    int r = legal_draw(seed, steps, o, n_legal), act = 0;
    for (; r >= 0; ++act) r -= action_legal(E, curmask, a, occ, g, m, act) ? 1 : 0;
    return act - 1;
}

// The action of agent m (group g, arena a, ABI ordinal o) under `policy` against group t.  `lut`: group g's view LUT in
// key order, one run of view_count cells per heading in turn_mode (Engine::upload_nbr_luts).
MG_HD int rule_action(const EngineDev &E, const NbrCell *lut, unsigned curmask, int a, int g, int t, int policy,
                      const MaskAgent &m, unsigned long long seed, long long steps, int o) {
    if (m.flags & FLAG_DEAD) return 0;
    const int *occ = E.occ + (long)a * E.W * E.H;
    if (policy == RULE_RUSH) {
        const int k = rule_attack(E, curmask, a, occ, g, t, m);
        if (k >= 0) return k;
    }
    int cx, cy;
    if (rule_nearest(E, lut, curmask, a, g, t, m, cx, cy)) {
        const int k = rule_move(E, curmask, a, occ, g, m, cx, cy, policy == RULE_FLEE);
        if (k >= 0) return k;
    }
    return rule_fallback(E, curmask, a, occ, g, m, seed, steps, o);
}

}  // namespace mg
