// action_mask_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_action_mask and be::launch_random_legal_actions: single-threaded loops over
// mask_phases.h action_legal / legal_draw, the functions the CUDA kernels (action_mask_kernel,
// random_legal_actions_kernel) run.  tests/test_action_mask_cpu.py links it together with backend_emu.cc into
// tests/_emu/libmagent_emu_mask.so, so the CPU tests pin those functions to the reference.
#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/mask_phases.h"

namespace mg {
namespace be {

void launch_action_mask(Ctx *, const EngineDev *dE, const EngineDev &, unsigned curmask, int g, unsigned char *out, int) {
    const EngineDev &E = *dE;
    const int na = E.grp[g].n_action;
    for (int a = 0; a < E.A; ++a) {
        const int *occ = E.occ + (long)a * E.W * E.H;
        unsigned char *rows = out + (size_t)E.off[(size_t)g * (E.A + 1) + a] * na;
        for (int i = 0; i < E.n[g * E.A + a]; ++i) {
            const MaskAgent m = mask_agent(E, curmask, a, g, i);
            for (int k = 0; k < na; ++k) rows[(size_t)i * na + k] = action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
        }
    }
}

void launch_random_legal_actions(Ctx *, const EngineDev *dE, const EngineDev &, unsigned curmask, int g,
                                 unsigned long long seed, int) {
    const EngineDev &E = *dE;
    const int na = E.grp[g].n_action;
    for (int a = 0; a < E.A; ++a) {
        const int *occ = E.occ + (long)a * E.W * E.H;
        const int o0 = E.off[(size_t)g * (E.A + 1) + a];
        for (int i = 0; i < E.n[g * E.A + a]; ++i) {
            const MaskAgent m = mask_agent(E, curmask, a, g, i);
            int n_legal = 0;
            for (int k = 0; k < na; ++k) n_legal += action_legal(E, curmask, a, occ, g, m, k) ? 1 : 0;
            int act = 0;
            if (n_legal > 0) {
                int r = legal_draw(seed, E.counters[CNT_STEPS], o0 + i, n_legal);
                for (; r >= 0; ++act) r -= action_legal(E, curmask, a, occ, g, m, act) ? 1 : 0;
                --act;
            }
            cur_soa(E, curmask, g).act[gidx(E, a, g, i)] = act;
        }
    }
}

}  // namespace be
}  // namespace mg
