// slot_phases.h -- the per-row logic of magent_b200_get_slots, shared by slots_kernel (backend_cuda.cu) and the test
// emulation (tests/emu/slots_emu.cc).
//
// An agent's slot is the number of agents of its group placed into its arena before it since the arena's last reset
// (Engine::host_add_agent hands them out).  The table row of arena a (struct SlotDev) maps every id the arena has handed
// out to its slot, so a row needs its agent's id and nothing else: the step, cull and render kernels never see slots.
#pragma once
#include "dev_types.h"

namespace mg {

MG_HD long slot_row_stride(int id_cap) { return (long)SLOT_HDR + id_cap; }

// [A][S] position of row i of arena a (whose agent has id `id`), or -1 when the table has no slot for it below S.  The
// engine keeps every slot below S and every id below id_cap; the checks only keep a broken table from writing outside
// the caller's buffers.
MG_HD int slot_flat(const int *tab, int id_cap, int a, int id, int S) {
    if (id < 0 || id >= id_cap) return -1;
    const int s = tab[(long)a * slot_row_stride(id_cap) + SLOT_HDR + id];
    return s >= 0 && s < S ? a * S + s : -1;
}

}  // namespace mg
