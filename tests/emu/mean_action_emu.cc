// mean_action_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_mean_action: a single-threaded loop over nbr_phases.h, the functions the CUDA kernel
// (mean_action_kernel) runs: every in-range view cell mapped by nbr_view_delta, filtered on the `kind` byte by
// nbr_kind_of, decided by nbr_at, binned by nbr_bin.  tests/test_mean_action_cpu.py links it together with
// backend_emu.cc into tests/_emu/libmagent_emu_mean.so, so the CPU tests pin those functions to the reference.
#include <algorithm>
#include <vector>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/nbr_phases.h"

namespace mg {
namespace be {

void launch_mean_action(Ctx *, const EngineDev *dE, const EngineDev &, unsigned curmask, int g, int of, float *mean,
                        int *count, int) {
    const EngineDev &E = *dE;
    const GroupDev &G = E.grp[g];
    const int na = E.grp[of].n_action;
    std::vector<int> bins(na);
    for (int a = 0; a < E.A; ++a) {
        const int o0 = E.off[(size_t)g * (E.A + 1) + a];
        for (int i = 0; i < E.n[g * E.A + a]; ++i) {
            const NbrObserver o = nbr_observer(E, curmask, a, g, i);
            std::fill(bins.begin(), bins.end(), 0);
            int cnt = 0;
            for (int vy = 0; vy < G.view_h && !(o.flags & FLAG_DEAD); ++vy)
                for (int vx = 0; vx < G.view_w; ++vx) {
                    if (!G.view_mask[vy * G.view_w + vx]) continue;
                    int dx, dy;
                    nbr_view_delta(E, G, o.dir, vx, vy, dx, dy);
                    const int x = o.x + dx, y = o.y + dy;
                    const int t = E.kind[a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad];
                    if (!nbr_kind_of(t, of)) continue;
                    const int j = nbr_at(E, curmask, a, g, of, o, x, y);
                    if (j < 0) continue;
                    ++cnt;
                    const int k = nbr_bin(E, curmask, a, of, j);
                    if (k >= 0) ++bins[k];
                }
            for (int k = 0; k < na; ++k) mean[(size_t)(o0 + i) * na + k] = nbr_mean(bins[k], cnt);
            if (count) count[o0 + i] = cnt;
        }
    }
}

}  // namespace be
}  // namespace mg
