// mask_phases.h -- which actions of an agent would do anything: the per-(agent, action) decision behind
// magent_b200_get_action_mask and magent_b200_random_legal_actions.
//
// "Legal" is a pure function of the state now: the reference, executing action k for this agent ALONE on this state,
// would take the success branch of Map::do_move / Map::do_turn / Map::get_attack_obj.  What other agents do in the same
// step is ignored (that is the step itself).  One function, action_legal(), serves the two CUDA kernels
// (backend_cuda.cu) and the test emulation (tests/emu/action_mask_emu.cc); the geometry comes from the helpers the
// step phases use (step_phases.h mover_target, attack_cell_from, friendly_fire_refused).
#pragma once
#include "step_phases.h"

namespace mg {

// what the decision needs to know about the agent itself; loaded once per agent
struct MaskAgent {
    int x, y, dir, code;         // code: the agent's own cell code in `occ`
    unsigned char flags;
};
MG_HD MaskAgent mask_agent(const EngineDev &E, unsigned curmask, int a, int g, int i) {
    const AgentSoA &s = cur_soa(E, curmask, g);
    const long gi = gidx(E, a, g, i);
    MaskAgent m;
    m.x = s.x[gi]; m.y = s.y[gi]; m.flags = s.flags[gi];
    m.dir = agent_dir(E, s, gi);
    m.code = code_make(g, i);
    return m;
}

// the draw of magent_b200_random_legal_actions
MG_HD unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
// Agent with ABI ordinal `o` (its row in env_set_action), `n_legal` > 0 legal actions: the rank, in ascending action
// number, of the legal action it takes.  `seed` is the call's seed as the engine passes it on (Engine::
// random_legal_actions), `steps` the device step counter (CNT_STEPS), which makes a replayed CUDA graph draw afresh.
MG_HD int legal_draw(unsigned long long seed, long long steps, int o, int n_legal) {
    seed += (unsigned long long)steps * 0xA24BAED4963EE407ull;
    return (int)((unsigned)(splitmix64(seed ^ ((unsigned long long)o * 0xD1342543DE82EF95ull)) >> 33) % (unsigned)n_legal);
}

// Would action k of agent `m` (group g, arena a; occ = the arena's occupancy plane) succeed if taken alone now?
MG_HD bool action_legal(const EngineDev &E, unsigned curmask, int a, const int *occ, int g, const MaskAgent &m, int k) {
    const GroupDev &G = E.grp[g];
    if (m.flags & FLAG_DEAD) return false;                 // attack, turn and move all skip it (GridWorld.cc:479,553,581)
    if (k >= G.attack_base) {                              // Map::get_attack_obj (Map.cc:209-252)
        int tx, ty;
        attack_cell_from(E, G, k, m.x, m.y, m.dir, tx, ty);
        if (tx < 0 || tx >= E.W || ty < 0 || ty >= E.H) return false;
        const int t = occ[ty * E.W + tx];
        if (t == OCC_FOOD) return E.food_mode != 0;        // anybody may eat
        if (t < 0) return false;
        return !friendly_fire_refused(E, g, code_group(t));   // own cells of a long body with attack_in_group included
    }
    const bool turn = k >= G.n_move;                       // turn_mode only: the two actions between moves and attacks
    if (!turn && (m.flags & FLAG_ABSORBED)) return false;  // an absorbed absorber's move is skipped (GridWorld.cc:581)
    int nx, ny, bw, bh;
    if (!mover_target(E, G, k, m.x, m.y, m.dir, turn, nx, ny, bw, bh)) return false;
    // is_blank_area (Map.cc:454-470): every cell empty or the mover's own; else the first other agent in get_collide's
    // scan order (Map.cc:486-501, walls and food are passed over) decides
    bool blank = true;
    int hit = -1;
    for (int bx = 0; bx < bw; ++bx)
        for (int by = 0; by < bh; ++by) {
            const int o = occ[(ny + by) * E.W + nx + bx];
            if (o == OCC_EMPTY || o == m.code) continue;
            blank = false;
            if (o >= 0 && hit < 0) hit = o;
        }
    if (blank) return true;
    if (turn || hit < 0) return false;
    // bumping into an absorber that has not swallowed anybody yet: the mover disappears into it (Map.cc:341-349)
    const int hg = code_group(hit);
    if (!E.grp[hg].can_absorb) return false;
    return !(cur_soa(E, curmask, hg).flags[gidx(E, a, hg, code_index(hit))] & FLAG_ABSORBED);
}

}  // namespace mg
