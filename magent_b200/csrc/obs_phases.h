// obs_phases.h -- per-cell / per-agent pieces of get_observation, shared by the CUDA render kernel and
// the test-only host emulation.
//
// Reference being restated: GridWorld::get_observation (src/gridworld/GridWorld.cc:292-401) and
// Map::extract_view (src/gridworld/Map.cc:129-207).
#pragma once
#include "step_phases.h"

namespace mg {

// coarse minimap cell of a map position for an observer whose view is vw x vh (GridWorld.cc:328-329,349)
MG_HD void minimap_cell(const EngineDev &E, int vw, int vh, int x, int y, int &cx, int &cy) {
    int scale_h = (E.H + vh - 1) / vh;
    int scale_w = (E.W + vw - 1) / vw;
    cx = x / scale_w;
    cy = y / scale_h;
}

// channel of group `other` as seen by group `me` (GridWorld::make_channel_trans, GridWorld.cc:897-913)
MG_HD int obs_channel(const EngineDev &E, int me, int other) {
    int stride = 2 + (E.minimap_mode ? 1 : 0);
    int rel = other - me; if (rel < 0) rel += E.G;
    return E.channel_base + rel * stride;
}

// Compose the n_channel floats of view cell (vy, vx) of one observer.
//   mm   : normalised minimap of the observer's arena, [G][vh*vw], or nullptr when minimap is off
//   out  : n_channel floats, fully written
MG_HD void obs_compose_cell(const EngineDev &E, unsigned curmask, int a, int g, int ax, int ay, int dir,
                            int self_cx, int self_cy, int vy, int vx, const float *mm, float *out) {
    const GroupDev &G = E.grp[g];
    const int C = E.n_channel;
    for (int ch = 0; ch < C; ++ch) out[ch] = 0.0f;
    int cell = vy * G.view_w + vx;
    if (mm) {
        int cells = G.view_w * G.view_h;
        for (int j = 0; j < E.G; ++j) {
            float v = mm[j * cells + cell];
            if (vy == self_cy && vx == self_cx) v += 1.0f;            // GridWorld.cc:382
            out[obs_channel(E, g, j) + 2] = v;
        }
    }
    if (!G.view_mask[cell]) return;
    int x = ax + G.view_xoff + G.view_x1 + vx;
    int y = ay + G.view_yoff + G.view_y1 + vy;
    if (E.turn_mode) {                   // the window is laid out in the observer's frame (Map.cc:140-146)
        int ox, oy, dx, dy;
        dir_real(G, dir, ox, oy);
        dir_rot(dir, G.view_xoff + G.view_x1 + vx, G.view_yoff + G.view_y1 + vy, dx, dy);
        x = ax + ox + dx; y = ay + oy + dy;
    }
    if (x < 0 || x >= E.W || y < 0 || y >= E.H) return;
    int t = (E.occ + (long)a * E.W * E.H)[y * E.W + x];
    if (t == OCC_EMPTY) return;
    if (t == OCC_WALL) { out[0] = 1.0f; return; }
    if (t == OCC_FOOD) { out[1] = 1.0f; return; }                     // food channel, no hp (Map.cc:191-199)
    int tg = code_group(t);
    int ch = obs_channel(E, g, tg);
    out[ch] = 1.0f;
    // hp / max_hp of the occupant (Map.cc:197), from the planes the step phases keep current (step_phases.h show_body): an
    // agent at exactly max_hp carries KIND_FULL in its kind byte instead of a value in the hp_norm plane
    const long pc = a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad;
    out[ch + 1] = (E.kind[pc] & KIND_FULL) ? 1.0f : E.hpn[pc];
}

// ---- global state (magent_b200_get_global_state): the whole map of every arena, [A][H][W][state_channels] floats.
// Channel 0 is the wall, 1 the food (food_mode only), then per group g in ABSOLUTE order base + 2g is presence and
// base + 2g + 1 the occupant's hp / max_hp.  Every value equals what Map::extract_view (Map.cc:191-199) writes for that map
// cell into any view covering it; only the channel order differs from a view's observer-relative one (obs_channel).
MG_HD int state_base(const EngineDev &E) { return 1 + (E.food_mode ? 1 : 0); }
MG_HD int state_channels(const EngineDev &E) { return state_base(E) + 2 * E.G; }
// the cell's hp / max_hp lives in the hp_norm plane: an agent below max_hp (KIND_FULL agents show 1.0f)
MG_HD bool state_needs_hpn(int t) { return kind_is_agent(t) && !(t & KIND_FULL); }
// channel ch of a cell whose kind byte is t; hp is the hp / max_hp the cell shows when it holds an agent
MG_HD float state_cell_value(int t, float hp, int ch, int base) {
    if (t == KIND_EMPTY) return 0.0f;
    if (t == KIND_WALL) return ch == 0 ? 1.0f : 0.0f;
    if (t == KIND_FOOD) return ch == 1 ? 1.0f : 0.0f;
    const int c = base + 2 * kind_group(t);
    return ch == c ? 1.0f : ch == c + 1 ? hp : 0.0f;
}
// the state_channels floats of map cell (x, y) of arena a, read from the padded planes the render reads
MG_HD void state_compose_cell(const EngineDev &E, int a, int x, int y, float *out) {
    const long pc = a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad;
    const int t = E.kind[pc];
    const float hp = state_needs_hpn(t) ? E.hpn[pc] : 1.0f;
    const int base = state_base(E), C = state_channels(E);
    for (int ch = 0; ch < C; ++ch) out[ch] = state_cell_value(t, hp, ch, base);
}

// non-spatial feature vector of agent (a, g, i)  (GridWorld.cc:386-396, Agent::get_embedding GridWorld.h:155-164)
MG_HD void obs_feature(const EngineDev &E, unsigned curmask, int a, int g, int i, float *out) {
    const GroupDev &G = E.grp[g];
    const AgentSoA &s = cur_soa(E, curmask, g);
    long gi = gidx(E, a, g, i);
    for (int k = 0; k < G.feature_size; ++k) out[k] = 0.0f;
    int id = s.id[gi];
    for (int k = 0; k < E.embedding_size; ++k, id >>= 1) out[k] = (float)(id & 1);
    int act = s.act[gi];
    if (act >= 0 && act <= G.n_action) out[E.embedding_size + act] = 1.0f;      // fresh agents: act == n_action
    out[E.embedding_size + G.n_action] = s.last_reward[gi];
    if (E.minimap_mode) {
        out[E.embedding_size + G.n_action + 1] = (float)s.x[gi] / (float)E.W;
        out[E.embedding_size + G.n_action + 2] = (float)s.y[gi] / (float)E.H;
    }
}

// one element of the feature vector (same values as obs_feature, element-wise for coalesced stores)
MG_HD float obs_feature_elem(const EngineDev &E, unsigned curmask, int a, int g, int i, int k) {
    const GroupDev &G = E.grp[g];
    const AgentSoA &s = cur_soa(E, curmask, g);
    long gi = gidx(E, a, g, i);
    if (k < E.embedding_size) return k < 31 ? (float)((s.id[gi] >> k) & 1) : 0.0f;
    int kk = k - E.embedding_size;
    if (kk < G.n_action) return kk == s.act[gi] ? 1.0f : 0.0f;
    if (kk == G.n_action) return s.last_reward[gi];
    if (E.minimap_mode) {
        if (kk == G.n_action + 1) return (float)s.x[gi] / (float)E.W;
        if (kk == G.n_action + 2) return (float)s.y[gi] / (float)E.H;
    }
    return 0.0f;
}

}  // namespace mg
