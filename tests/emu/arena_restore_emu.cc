// arena_restore_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_restore and be::launch_arena_done: single-threaded statements of what restore_kernel,
// restore_finish_kernel and arena_done_kernel do (backend_cuda.cu).  tests/test_arena_restore_cpu.py links it together
// with backend_emu.cc and global_state_emu.cc into tests/_emu/libmagent_emu_restore.so, so that the engine's snapshot
// and restore logic (storage, strides, counts, RNG, id counter) is pinned to the reference without a GPU.
#include <string.h>
#include "../../magent_b200/csrc/backend.h"

namespace mg {
namespace be {

void launch_restore(Ctx *c, const EngineDev *dE, const EngineDev &hE, unsigned curmask, const SnapDev &S, const int *src,
                    int keep_rng) {
    const EngineDev &E = *dE;
    const long cells = (long)E.W * E.H;
    for (int a = 0; a < E.A; ++a) {
        int s = src ? src[a] : ((E.done[a] & 1) ? a : -1);
        if (s < 0 || s >= E.A) continue;
        memcpy(E.occ + a * cells, S.occ + s * cells, cells * 4);
        memset(E.claim_head + a * cells, 0xff, cells * 4);
        memcpy(E.kind + a * E.kplane, S.kind + s * E.kplane, E.kplane);
        memcpy(E.hpn + a * E.kplane, S.hpn + s * E.kplane, E.kplane * 4);
        if (E.food) memcpy(E.food + a * cells, S.food + s * cells, cells * 4);
        for (int g = 0; g < E.G; ++g) {
            const int n = S.n[g * E.A + s];
            const AgentSoA &d = E.grp[g].soa[(curmask >> g) & 1u], &f = S.soa[g];
            const long da = (long)a * E.grp[g].cap, sa = (long)s * S.cap[g];
            memcpy(d.x + da, f.x + sa, n * 4); memcpy(d.y + da, f.y + sa, n * 4);
            memcpy(d.hp + da, f.hp + sa, n * 4); memcpy(d.act + da, f.act + sa, n * 4);
            memcpy(d.id + da, f.id + sa, n * 4);
            memcpy(d.next_reward + da, f.next_reward + sa, n * 4); memcpy(d.last_reward + da, f.last_reward + sa, n * 4);
            memcpy(d.op_obj + da, f.op_obj + sa, n * 4);
            memcpy(d.last_op + da, f.last_op + sa, n); memcpy(d.flags + da, f.flags + sa, n); memcpy(d.dir + da, f.dir + sa, n);
            E.n[g * E.A + a] = n;
            E.dead_ct[g * E.A + a] = S.dead_ct[g * E.A + s];
        }
        const ArenaHdr keep = E.hdr[a];
        E.hdr[a] = S.hdr[s];
        if (keep_rng) { E.hdr[a].rng = keep.rng; E.hdr[a].rng_next = keep.rng_next; }
        E.done[a] = S.done[s];
    }
    launch_offsets(c, dE, hE);
}

void launch_arena_done(Ctx *, const EngineDev *dE, const EngineDev &, int *out) {
    for (int a = 0; a < dE->A; ++a) out[a] = dE->done[a] & 1;
}

}  // namespace be
}  // namespace mg
