// slot_loop_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_set_action_slots, be::launch_reward_slots and be::launch_action_mask_slots:
// single-threaded statements of what set_action_slots_kernel, reward_slots_kernel and action_mask_slots_kernel do
// (backend_cuda.cu), with the per-row slot lookup of slot_phases.h and the legality of mask_phases.h action_legal.
// Every output slot starts vacant (+0.0, 0, an all-zero mask row); every row below the device-side count then writes its
// slot.  It defines only these three symbols, so that it links next to every other *_emu.cc;
// tests/test_slot_loop_cpu.py links it with backend_emu.cc, arena_restore_emu.cc, slots_emu.cc and the emulations of
// the outputs it compares.
#include <string.h>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/mask_phases.h"
#include "../../magent_b200/csrc/slot_phases.h"

namespace mg {
namespace be {

void launch_set_action_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, unsigned curmask, int g,
                             int S, const int *act) {
    const EngineDev &E = *dE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, curmask, g);
    for (int a = 0; a < E.A; ++a)
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const long gi = gidx(E, a, g, i);
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gi], S);
            if (flat >= 0) s.act[gi] = act[flat];
        }
}

void launch_reward_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, unsigned curmask, int g,
                         int S, float *reward, unsigned char *status) {
    const EngineDev &E = *dE;
    const size_t n = (size_t)E.A * S;
    if (reward) for (size_t q = 0; q < n; ++q) reward[q] = 0.0f;
    if (status) memset(status, 0, n);
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, curmask, g);
    for (int a = 0; a < E.A; ++a)
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const long gi = gidx(E, a, g, i);
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gi], S);
            if (flat < 0) continue;
            if (reward) reward[flat] = s.next_reward[gi] + E.hdr[a].grp_reward[g];
            if (status) status[flat] = (s.flags[gi] & FLAG_DEAD) ? 2 : 1;
        }
}

void launch_action_mask_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, unsigned curmask, int g,
                              int S, unsigned char *mask) {
    const EngineDev &E = *dE;
    const int na = E.grp[g].n_action;
    memset(mask, 0, (size_t)E.A * S * na);
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, curmask, g);
    for (int a = 0; a < E.A; ++a) {
        const int *occ = E.occ + (long)a * E.W * E.H;
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gidx(E, a, g, i)], S);
            if (flat < 0) continue;
            const MaskAgent m = mask_agent(E, curmask, a, g, i);
            for (int k = 0; k < na; ++k) mask[(size_t)flat * na + k] = action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
        }
    }
}

}  // namespace be
}  // namespace mg
