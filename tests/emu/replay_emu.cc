// replay_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_replay_events, be::launch_replay_restore and be::launch_replay_record: single-threaded
// statements of what replay_events_kernel, replay_restore_kernel and replay_record_kernel do (backend_cuda.cu), with the
// per-item functions of replay_phases.h.  tests/test_replay_cpu.py links it with the other emulated loops, so that the
// recorder's bookkeeping (episodes, event lists, frame buffer, writer) is pinned to env_render without a GPU.
#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/replay_phases.h"

namespace mg {
namespace be {

void launch_replay_events(Ctx *, const EngineDev *dE, const EngineDev &, unsigned curmask, RepArena *rep, RepEvent *ev,
                          const int *arenas, int n_arenas) {
    const EngineDev &E = *dE;
    for (int k = 0; k < n_arenas; ++k) {
        const int a = arenas[k];
        if (a < 0) continue;
        for (int g = 0; g < E.G; ++g) {
            const GroupDev &G = E.grp[g];
            const AgentSoA &s = G.soa[(curmask >> g) & 1u];
            const int n = E.n[(long)g * E.A + a];
            rep[a].ev_n[g] = n;
            for (int i = 0; i < n; ++i) {
                const long gi = (long)a * G.cap + i;
                ev[(long)a * E.cap_total + G.foff + i] = replay_event(G, s, E.turn_mode, gi, G.ev_rank[gi]);
            }
        }
    }
}

void launch_replay_restore(Ctx *, const EngineDev &hE, RepArena *rep, const int *src) {
    for (int a = 0; a < hE.A; ++a) {
        const int s = src ? src[a] : ((hE.done[a] & 1) ? a : -1);
        if (s < 0 || s >= hE.A) continue;
        rep[a].episode += 1;
        for (int &n : rep[a].ev_n) n = 0;
    }
}

void launch_replay_record(Ctx *, const EngineDev *dE, const EngineDev &, unsigned curmask, const RepArena *rep,
                          const RepEvent *ev, const RepRecord &R) {
    const EngineDev &E = *dE;
    const int frame = R.ctl->n_frames;
    if (frame >= R.max_frames) { R.ctl->dropped += 1; return; }
    const long cells = (long)E.W * E.H;
    for (int k = 0; k < R.n_arenas; ++k) {
        const int a = R.arenas[k];
        const int episode = rep[a].episode;
        const bool walls = episode != R.last_ep[k];
        int *F = R.frames + ((long)frame * R.n_arenas + k) * R.L.frame_ints();
        F[REP_H_EPISODE] = episode;
        F[REP_H_WALLS] = walls ? 1 : 0;
        for (int g = 0; g < MG_MAX_GROUPS; ++g) {
            F[REP_H_N + g] = g < E.G ? E.n[(long)g * E.A + a] : 0;
            F[REP_H_EV_N + g] = g < E.G ? rep[a].ev_n[g] : 0;
        }
        for (int g = 0; g < E.G; ++g) {
            const GroupDev &G = E.grp[g];
            RepAgent *ag = reinterpret_cast<RepAgent *>(F + R.L.agent_base()) + G.foff;
            RepEvent *fe = reinterpret_cast<RepEvent *>(F + R.L.event_base()) + G.foff;
            for (int i = 0; i < E.n[(long)g * E.A + a]; ++i)
                ag[i] = replay_agent(G.soa[(curmask >> g) & 1u], E.turn_mode, (long)a * G.cap + i);
            for (int i = 0; i < rep[a].ev_n[g]; ++i) fe[i] = ev[(long)a * R.L.cap_total + G.foff + i];
        }
        if (walls)
            for (int w = 0; w < R.L.wall_words; ++w) F[R.L.wall_base() + w] = (int)replay_wall_word(E.occ + a * cells, cells, w);
        R.last_ep[k] = episode;
    }
    R.ctl->n_frames = frame + 1;
}

}  // namespace be
}  // namespace mg
