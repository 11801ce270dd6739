// replay_phases.h -- the per-item logic of the replay recorder (magent_b200_replay_*), shared by the CUDA kernels
// (backend_cuda.cu replay_events_kernel, replay_record_kernel), the test emulation (tests/emu/replay_emu.cc) and, for
// the attack cell, the host collector of env_render (Engine::collect_attack_events).
//
// A recorder frame of one arena is a fixed-size block of ints (dev_types.h struct RepLayout): a header, one RepAgent per agent row
// of the live SoA at its group's flat offset (GroupDev::foff), one RepEvent per agent row of the last step's event list
// at the same offsets, and a wall bitmap of the map (present only in the first frame of an episode).  Which rows and
// events are used, their order, the filtering of absorbers and the hp percentage are left to the host writer.
#pragma once
#include "step_phases.h"

namespace mg {

// the cell an executed attack aims at, as the viewer's attack event lists it (Map::get_attack_obj, Map.cc:209-221):
// (ax, ay) = the attack offset of the type plus the action's attack delta, in the agent's frame
MG_HD void replay_event_cell(const GroupDev &G, int dir, int x, int y, int ax, int ay, int &tx, int &ty) {
    int rx, ry, dx, dy;
    dir_real(G, dir, rx, ry);
    dir_rot(dir, ax, ay, dx, dy);
    tx = x + rx + dx;
    ty = y + ry + dy;
}

// the event-list row of agent row i of group g (executed: its ev_rank >= 0)
MG_HD RepEvent replay_event(const GroupDev &G, const AgentSoA &s, int turn_mode, long gi, int rank) {
    RepEvent e = {rank, -1, 0, 0};
    if (rank < 0) return e;
    const int act = s.act[gi];
    const int k = act - G.attack_base;
    const int dir = turn_mode ? (int)s.dir[gi] : (int)DIR_NORTH;
    e.id = s.id[gi];
    replay_event_cell(G, dir, s.x[gi], s.y[gi], G.att_xoff + G.att_dx[k], G.att_yoff + G.att_dy[k], e.x, e.y);
    return e;
}

MG_HD RepAgent replay_agent(const AgentSoA &s, int turn_mode, long gi) {
    RepAgent r;
    r.id = s.id[gi];
    r.x = s.x[gi];
    r.y = s.y[gi];
    r.hp = s.hp[gi];
    r.dir_flags = (turn_mode ? (int)s.dir[gi] : (int)DIR_NORTH) | ((s.flags[gi] & FLAG_ABSORBED) ? FLAG_ABSORBED << 8 : 0);
    return r;
}

// bit b of word w: cell 32 w + b of the arena's occ is a wall
MG_HD unsigned replay_wall_word(const int *occ, long cells, int w) {
    unsigned bits = 0;
    for (int b = 0; b < 32; ++b) {
        const long c = (long)w * 32 + b;
        if (c < cells && occ[c] == OCC_WALL) bits |= 1u << b;
    }
    return bits;
}

// the group of flat row f (GroupDev::foff <= f < foff + cap), or -1 beyond the last group
MG_HD int replay_group_of(const EngineDev &E, int f) {
    for (int g = 0; g < E.G; ++g)
        if (f >= E.grp[g].foff && f < E.grp[g].foff + E.grp[g].cap) return g;
    return -1;
}

}  // namespace mg
