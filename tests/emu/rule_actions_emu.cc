// rule_actions_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_rule_actions and be::launch_rule_actions_slots: single-threaded loops over
// rule_phases.h rule_action, the function the CUDA kernels (rule_actions_kernel, rule_actions_slots_kernel) run, with
// the engine's view LUT (host memory in the emulation).  Every output slot starts vacant (-1); every row below the
// device-side count then writes its action into its slot (slot_phases.h slot_flat).  tests/test_rule_actions_cpu.py
// links it with backend_emu.cc and every other *_emu.cc, so the CPU tests pin rule_action to the numpy restatement.
#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/rule_phases.h"
#include "../../magent_b200/csrc/slot_phases.h"

namespace mg {
namespace be {

void launch_rule_actions(Ctx *, const EngineDev *dE, const EngineDev &, const NbrCell *lut, unsigned curmask, int g,
                         int t, int policy, unsigned long long seed, int *out, int) {
    const EngineDev &E = *dE;
    for (int a = 0; a < E.A; ++a) {
        const int o0 = E.off[(size_t)g * (E.A + 1) + a];
        for (int i = 0; i < E.n[g * E.A + a]; ++i) {
            const int act = rule_action(E, lut, curmask, a, g, t, policy, mask_agent(E, curmask, a, g, i), seed,
                                        E.counters[CNT_STEPS], o0 + i);
            if (out) out[o0 + i] = act;
            else cur_soa(E, curmask, g).act[gidx(E, a, g, i)] = act;
        }
    }
}

void launch_rule_actions_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, const NbrCell *lut,
                               unsigned curmask, int g, int t, int policy, unsigned long long seed, int S, int *out) {
    const EngineDev &E = *dE;
    for (size_t q = 0; q < (size_t)E.A * S; ++q) out[q] = -1;
    const AgentSoA &s = cur_soa(E, curmask, g);
    for (int a = 0; a < E.A; ++a) {
        const int o0 = E.off[(size_t)g * (E.A + 1) + a];
        for (int i = 0; i < E.off[(size_t)g * (E.A + 1) + a + 1] - o0; ++i) {
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gidx(E, a, g, i)], S);
            if (flat < 0) continue;
            out[flat] = rule_action(E, lut, curmask, a, g, t, policy, mask_agent(E, curmask, a, g, i), seed,
                                    E.counters[CNT_STEPS], o0 + i);
        }
    }
}

}  // namespace be
}  // namespace mg
