// nbr_phases.h -- who an observer's neighbours are: the per-observer pieces behind magent_b200_get_mean_action.
//
// The neighbours N(i) of observer i (group g) in group `of` are the distinct agents j != i of `of` whose presence i's own
// view channel for `of` shows: some in-range cell of i's view window maps, as in obs_phases.h obs_compose_cell, to an
// on-board map cell that j's body covers in `occ`.  A body larger than 1 x 1 counts once, at the first of its cells in
// row-major order over its footprint that i sees.  magent_b200_get_neighbours orders N(i) by key (nbr_cell_key) and
// lists a longer body at its smallest-key cell instead.  One set of functions serves the CUDA kernels (backend_cuda.cu
// mean_action_kernel, neighbours_kernel) and the test emulations (tests/emu/mean_action_emu.cc, neighbours_emu.cc).
#pragma once
#include "step_phases.h"

namespace mg {

// what the decision needs to know about the observer itself; loaded once per observer
struct NbrObserver {
    int x, y, dir, code;         // code: the observer's own cell code in `occ`
    unsigned char flags;
};
MG_HD NbrObserver nbr_observer(const EngineDev &E, unsigned curmask, int a, int g, int i) {
    const AgentSoA &s = cur_soa(E, curmask, g);
    const long gi = gidx(E, a, g, i);
    NbrObserver o;
    o.x = s.x[gi]; o.y = s.y[gi]; o.flags = s.flags[gi];
    o.dir = agent_dir(E, s, gi);
    o.code = code_make(g, i);
    return o;
}

// Map displacement, from the observer's stored top-left corner, of view cell (vx, vy) of an observer of group G facing
// `dir`: the window mapping of obs_compose_cell (turn_mode: laid out in the observer's frame, Map.cc:140-146).
MG_HD void nbr_view_delta(const EngineDev &E, const GroupDev &G, int dir, int vx, int vy, int &dx, int &dy) {
    const int ex = G.view_xoff + G.view_x1 + vx, ey = G.view_yoff + G.view_y1 + vy;
    if (!E.turn_mode) { dx = ex; dy = ey; return; }
    int ox, oy, rx, ry;
    dir_real(G, dir, ox, oy);
    dir_rot(dir, ex, ey, rx, ry);
    dx = ox + rx; dy = oy + ry;
}

// The inverse: the view cell (vx, vy) that map displacement (dx, dy) from the observer falls on, and whether that is an
// in-range cell of its view window (vx, vy are set either way).
MG_HD bool nbr_view_cell(const EngineDev &E, const GroupDev &G, int dir, int dx, int dy, int &vx, int &vy) {
    int ex = dx, ey = dy;
    if (E.turn_mode) {
        int ox, oy;
        dir_real(G, dir, ox, oy);
        // undoing a quarter turn one way is the quarter turn the other way
        dir_rot(dir == DIR_WEST ? DIR_EAST : dir == DIR_EAST ? DIR_WEST : dir, dx - ox, dy - oy, ex, ey);
    }
    vx = ex - G.view_xoff - G.view_x1; vy = ey - G.view_yoff - G.view_y1;
    if (vx < 0 || vx >= G.view_w || vy < 0 || vy >= G.view_h) return false;
    return G.view_mask[vy * G.view_w + vx] != 0;
}
MG_HD bool nbr_in_view(const EngineDev &E, const GroupDev &G, int dir, int dx, int dy) {
    int vx, vy;
    return nbr_view_cell(E, G, dir, dx, dy, vx, vy);
}

// ---- the order of magent_b200_get_neighbours
// The key of view cell (vx, vy) of an observer of group G facing `dir`, whose map cell lies at displacement (dx, dy) from
// the observer's stored top-left corner: first d2, the squared Euclidean distance from that cell to the observer's
// footprint [0, bw) x [0, bh) (0 on the footprint), then the row-major view index.  Packed as d2 * view cells + index,
// which keeps the order; the host checks that the largest key of a group fits an int (Engine::to_device).
MG_HD int nbr_cell_key(const GroupDev &G, int dir, int dx, int dy, int vx, int vy) {
    int bw, bh;
    body_dims(G, dir, bw, bh);
    const int ex = dx < 0 ? -dx : dx >= bw ? dx - bw + 1 : 0;
    const int ey = dy < 0 ? -dy : dy >= bh ? dy - bh + 1 : 0;
    return (ex * ex + ey * ey) * (G.view_w * G.view_h) + vy * G.view_w + vx;
}
// the key of map displacement (dx, dy), or -1 when it is not on an in-range cell of the window
MG_HD int nbr_key(const EngineDev &E, const GroupDev &G, int dir, int dx, int dy) {
    int vx, vy;
    if (!nbr_view_cell(E, G, dir, dx, dy, vx, vy)) return -1;
    return nbr_cell_key(G, dir, dx, dy, vx, vy);
}

// Map cell (x, y) of arena a, seen through an in-range view cell of observer `o` of group g whose key is `key`: the index
// in group `of` of the neighbour this cell lists, or -1 when it lists none (off the board, no agent of `of` there, the
// observer itself, or a cell of a longer body with a smaller key that the observer also sees).  Stateless: a longer body
// is listed at its smallest-key visible cell whichever order the cells are visited in.
MG_HD int nbr_nearest_at(const EngineDev &E, unsigned curmask, int a, int g, int of, const NbrObserver &o, int x, int y,
                         int key) {
    if (x < 0 || x >= E.W || y < 0 || y >= E.H) return -1;
    const int t = E.occ[(long)a * E.W * E.H + (long)y * E.W + x];
    if (t < 0 || code_group(t) != of || t == o.code) return -1;
    const int j = code_index(t);
    const GroupDev &F = E.grp[of];
    if (F.body_w == 1 && F.body_l == 1) return j;
    const AgentSoA &s = cur_soa(E, curmask, of);
    const long gj = gidx(E, a, of, j);
    const int jx = s.x[gj], jy = s.y[gj];
    int bw, bh;
    body_dims(F, agent_dir(E, s, gj), bw, bh);
    const GroupDev &G = E.grp[g];
    for (int by = 0; by < bh; ++by)
        for (int bx = 0; bx < bw; ++bx) {
            const int k = nbr_key(E, G, o.dir, jx + bx - o.x, jy + by - o.y);
            if (k >= 0 && k < key) return -1;
        }
    return j;
}

// The cell's byte in the padded `kind` plane can show an agent of group `of`: the cheap filter before `occ` is read.
MG_HD bool nbr_kind_of(int t, int of) { return kind_is_agent(t) && kind_group(t) == of; }

// Map cell (x, y) of arena a, seen through an in-range view cell of observer `o` of group g: the index in group `of` of
// the neighbour it contributes to N(o), or -1 when it contributes none (off the board, no agent of `of` there, the
// observer itself, or a cell of a longer body that an earlier cell of the same body already contributes).
MG_HD int nbr_at(const EngineDev &E, unsigned curmask, int a, int g, int of, const NbrObserver &o, int x, int y) {
    if (x < 0 || x >= E.W || y < 0 || y >= E.H) return -1;
    const int t = E.occ[(long)a * E.W * E.H + (long)y * E.W + x];
    if (t < 0 || code_group(t) != of || t == o.code) return -1;
    const int j = code_index(t);
    const GroupDev &F = E.grp[of];
    if (F.body_w == 1 && F.body_l == 1) return j;
    // the first cell of j's footprint, row-major, that the observer sees counts j
    const AgentSoA &s = cur_soa(E, curmask, of);
    const long gj = gidx(E, a, of, j);
    const int jx = s.x[gj], jy = s.y[gj];
    int bw, bh;
    body_dims(F, agent_dir(E, s, gj), bw, bh);
    const GroupDev &G = E.grp[g];
    for (int by = 0; by < bh; ++by)
        for (int bx = 0; bx < bw; ++bx) {
            if (jx + bx == x && jy + by == y) return j;
            if (nbr_in_view(E, G, o.dir, jx + bx - o.x, jy + by - o.y)) return -1;
        }
    return -1;
}

// the bin neighbour j (group `of`) falls in: its action, or -1 when that is outside [0, n_action) (an agent added since
// the last step holds n_action; an id the step ignores stays as it was set)
MG_HD int nbr_bin(const EngineDev &E, unsigned curmask, int a, int of, int j) {
    const int k = cur_soa(E, curmask, of).act[gidx(E, a, of, j)];
    return k >= 0 && k < E.grp[of].n_action ? k : -1;
}

// one element of a row: IEEE round-to-nearest division, 0 for an observer without neighbours
MG_HD float nbr_mean(int bin, int count) { return count > 0 ? (float)bin / (float)count : 0.0f; }

}  // namespace mg
