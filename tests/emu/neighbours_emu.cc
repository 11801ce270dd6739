// neighbours_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_neighbours: a single-threaded loop over nbr_phases.h, the functions the CUDA kernel
// (neighbours_kernel) runs, without its sorted view LUT: every in-range view cell mapped by nbr_view_delta and keyed by
// nbr_cell_key, filtered on the `kind` byte by nbr_kind_of, decided by nbr_nearest_at; the cells that list a neighbour
// are then sorted by key.  tests/test_neighbours_cpu.py links it together with backend_emu.cc into
// tests/_emu/libmagent_emu_nbr.so, so the CPU tests pin those functions to the reference.
#include <algorithm>
#include <vector>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/nbr_phases.h"

namespace mg {
namespace be {

void launch_neighbours(Ctx *, const EngineDev *dE, const EngineDev &, const NbrCell *, unsigned curmask, int g, int of,
                       int k, int *idx, int *rel, int *count, int) {
    const EngineDev &E = *dE;
    const GroupDev &G = E.grp[g];
    struct Hit { int key, j, vx, vy; };
    std::vector<Hit> hits;
    for (int a = 0; a < E.A; ++a) {
        const int o0 = E.off[(size_t)g * (E.A + 1) + a], base = E.off[(size_t)of * (E.A + 1) + a];
        for (int i = 0; i < E.n[g * E.A + a]; ++i) {
            const NbrObserver o = nbr_observer(E, curmask, a, g, i);
            hits.clear();
            for (int vy = 0; vy < G.view_h && !(o.flags & FLAG_DEAD); ++vy)
                for (int vx = 0; vx < G.view_w; ++vx) {
                    if (!G.view_mask[vy * G.view_w + vx]) continue;
                    int dx, dy;
                    nbr_view_delta(E, G, o.dir, vx, vy, dx, dy);
                    const int x = o.x + dx, y = o.y + dy;
                    const int t = E.kind[a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad];
                    if (!nbr_kind_of(t, of)) continue;
                    const int key = nbr_cell_key(G, o.dir, dx, dy, vx, vy);
                    const int j = nbr_nearest_at(E, curmask, a, g, of, o, x, y, key);
                    if (j >= 0) hits.push_back({key, j, vx, vy});
                }
            std::sort(hits.begin(), hits.end(), [](const Hit &p, const Hit &q) { return p.key < q.key; });
            const size_t row = (size_t)(o0 + i) * k;
            for (int s = 0; s < k; ++s) {
                const bool used = s < (int)hits.size();
                idx[row + s] = used ? base + hits[s].j : -1;
                if (rel) {
                    rel[2 * (row + s)] = used ? hits[s].vy : -1;
                    rel[2 * (row + s) + 1] = used ? hits[s].vx : -1;
                }
            }
            if (count) count[o0 + i] = (int)hits.size();
        }
    }
}

}  // namespace be
}  // namespace mg
