// nbr_slots_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_mean_action_slots and be::launch_neighbours_slots: single-threaded statements of what
// mean_action_slots_kernel and neighbours_slots_kernel do (backend_cuda.cu), over nbr_phases.h for the per-observer
// decisions and slot_phases.h for the slots.  Every output slot starts vacant (a +0.0 row / all -1, count 0); every row
// below the device-side count then writes the row of its observer into its slot, each listed neighbour given as its
// flat slot a * S_of + slot in group `of`.  The observers' walks are mean_action_emu.cc's and neighbours_emu.cc's,
// restated here as static helpers, so that this file defines only these two symbols and links next to every other
// *_emu.cc; tests/test_nbr_slots_cpu.py links it with backend_emu.cc, arena_restore_emu.cc, slots_emu.cc and the
// emulations of the row-ordered outputs it compares against.
#include <algorithm>
#include <vector>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/nbr_phases.h"
#include "../../magent_b200/csrc/slot_phases.h"

namespace mg {
namespace be {

// the cell of view cell (vx, vy) of observer o: map position and its `kind` byte
static int view_cell(const EngineDev &E, const GroupDev &G, int a, const NbrObserver &o, int vx, int vy, int &x, int &y,
                     int &dx, int &dy) {
    nbr_view_delta(E, G, o.dir, vx, vy, dx, dy);
    x = o.x + dx; y = o.y + dy;
    return E.kind[a * E.kplane + (long)(y + E.kpad) * E.kw + x + E.kpad];
}

// bins[k] += 1 for every neighbour of o in group `of` acting k; returns |N(o)|
static int mean_walk(const EngineDev &E, unsigned curmask, int a, int g, int of, const NbrObserver &o,
                     std::vector<int> &bins) {
    const GroupDev &G = E.grp[g];
    std::fill(bins.begin(), bins.end(), 0);
    int cnt = 0;
    for (int vy = 0; vy < G.view_h && !(o.flags & FLAG_DEAD); ++vy)
        for (int vx = 0; vx < G.view_w; ++vx) {
            if (!G.view_mask[vy * G.view_w + vx]) continue;
            int x, y, dx, dy;
            if (!nbr_kind_of(view_cell(E, G, a, o, vx, vy, x, y, dx, dy), of)) continue;
            const int j = nbr_at(E, curmask, a, g, of, o, x, y);
            if (j < 0) continue;
            ++cnt;
            const int k = nbr_bin(E, curmask, a, of, j);
            if (k >= 0) ++bins[k];
        }
    return cnt;
}

struct Hit { int key, j, vx, vy; };

// N(o) in group `of`, sorted by key
static void nbr_walk(const EngineDev &E, unsigned curmask, int a, int g, int of, const NbrObserver &o,
                     std::vector<Hit> &hits) {
    const GroupDev &G = E.grp[g];
    hits.clear();
    for (int vy = 0; vy < G.view_h && !(o.flags & FLAG_DEAD); ++vy)
        for (int vx = 0; vx < G.view_w; ++vx) {
            if (!G.view_mask[vy * G.view_w + vx]) continue;
            int x, y, dx, dy;
            if (!nbr_kind_of(view_cell(E, G, a, o, vx, vy, x, y, dx, dy), of)) continue;
            const int key = nbr_cell_key(G, o.dir, dx, dy, vx, vy);
            const int j = nbr_nearest_at(E, curmask, a, g, of, o, x, y, key);
            if (j >= 0) hits.push_back({key, j, vx, vy});
        }
    std::sort(hits.begin(), hits.end(), [](const Hit &p, const Hit &q) { return p.key < q.key; });
}

void launch_mean_action_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, unsigned curmask, int g,
                              int of, int S, float *mean, int *count) {
    const EngineDev &E = *dE;
    const int na = E.grp[of].n_action;
    const size_t n = (size_t)E.A * S;
    for (size_t q = 0; q < n * na; ++q) mean[q] = 0.0f;
    if (count) for (size_t q = 0; q < n; ++q) count[q] = 0;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, curmask, g);
    std::vector<int> bins(na);
    for (int a = 0; a < E.A; ++a)
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gidx(E, a, g, i)], S);
            if (flat < 0) continue;
            const int cnt = mean_walk(E, curmask, a, g, of, nbr_observer(E, curmask, a, g, i), bins);
            for (int k = 0; k < na; ++k) mean[(size_t)flat * na + k] = nbr_mean(bins[k], cnt);
            if (count) count[flat] = cnt;
        }
}

void launch_neighbours_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, const NbrCell *,
                             unsigned curmask, int g, int of, int k, int S, int S_of, int *idx, int *rel, int *count) {
    const EngineDev &E = *dE;
    const size_t n = (size_t)E.A * S;
    for (size_t q = 0; q < n * k; ++q) idx[q] = -1;
    if (rel) for (size_t q = 0; q < 2 * n * k; ++q) rel[q] = -1;
    if (count) for (size_t q = 0; q < n; ++q) count[q] = 0;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, curmask, g), &f = cur_soa(E, curmask, of);
    std::vector<Hit> hits;
    for (int a = 0; a < E.A; ++a)
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gidx(E, a, g, i)], S);
            if (flat < 0) continue;
            nbr_walk(E, curmask, a, g, of, nbr_observer(E, curmask, a, g, i), hits);
            const size_t row = (size_t)flat * k;
            for (int r = 0; r < k && r < (int)hits.size(); ++r) {
                idx[row + r] = slot_flat(T->tab, T->id_cap, a, f.id[gidx(E, a, of, hits[r].j)], S_of);
                if (rel) { rel[2 * (row + r)] = hits[r].vy; rel[2 * (row + r) + 1] = hits[r].vx; }
            }
            if (count) count[flat] = (int)hits.size();
        }
}

}  // namespace be
}  // namespace mg
