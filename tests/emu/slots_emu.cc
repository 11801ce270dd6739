// slots_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_slots and be::launch_restore_slots: single-threaded statements of what slots_kernel
// and restore_slots_kernel do (backend_cuda.cu), with the per-row lookup of slot_phases.h.  tests/test_slots_cpu.py links
// it together with backend_emu.cc and arena_restore_emu.cc into tests/_emu/libmagent_emu_slots.so, so that the engine's
// slot bookkeeping (placement, table width, snapshots, restores, read-back) is pinned to a restatement without a GPU.
#include <algorithm>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/slot_phases.h"

namespace mg {
namespace be {

void launch_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, unsigned curmask, int g, int S,
                  int *row_slot, int *slot_row, int n_bound) {
    const EngineDev &E = *dE;
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = E.grp[g].soa[(curmask >> g) & 1u];
    for (int a = 0; a < E.A; ++a) {
        if (slot_row) std::fill(slot_row + (long)a * S, slot_row + (long)(a + 1) * S, -1);
        const int cnt = std::min(off[a + 1] - off[a], n_bound - off[a]);
        for (int i = 0; i < cnt; ++i) {
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[(long)a * E.grp[g].cap + i], S);
            if (row_slot) row_slot[off[a] + i] = flat;
            if (slot_row && flat >= 0) slot_row[flat] = off[a] + i;
        }
    }
    if (row_slot)
        for (int r = off[E.A]; r < n_bound; ++r) row_slot[r] = -1;
}

void launch_restore_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, const int *snap_tab,
                          int snap_id_cap, const int *src) {
    const EngineDev &E = *dE;
    for (int a = 0; a < E.A; ++a) {
        const int s = src ? src[a] : ((E.done[a] & 1) ? a : -1);
        if (s < 0 || s >= E.A) continue;
        const int *from = snap_tab + s * slot_row_stride(snap_id_cap);
        std::copy(from, from + slot_row_stride(std::min(T->id_cap, snap_id_cap)), T->tab + a * slot_row_stride(T->id_cap));
    }
}

}  // namespace be
}  // namespace mg
