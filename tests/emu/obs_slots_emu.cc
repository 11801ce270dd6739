// obs_slots_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_obs_slots: a single-threaded statement of the slot-ordered observation
// (backend_cuda.cu launch_obs_slots) built from the pieces backend_emu.cc's launch_obs uses (obs_phases.h
// obs_compose_cell and obs_feature) and the per-row slot lookup of slot_phases.h.  Every slot starts as an all-zero
// record and feature row; every row below the device-side count then writes its record into its slot.
// tests/test_obs_slots_cpu.py links it with backend_emu.cc, arena_restore_emu.cc and slots_emu.cc.
#include <string.h>
#include <vector>

#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/obs_phases.h"
#include "../../magent_b200/csrc/slot_phases.h"

namespace mg {
namespace be {

// n float32 values into element o of a float32 or binary16 buffer.  The compiler's binary16 conversion rounds to
// nearest-even and keeps a quiet NaN's sign and top payload bits, as the f16 hand-off does.
static void put(void *buf, int half, size_t o, const float *v, size_t n) {
    if (!half) { memcpy((float *)buf + o, v, n * sizeof(float)); return; }
    for (size_t q = 0; q < n; ++q) ((_Float16 *)buf)[o + q] = (_Float16)v[q];
}

void launch_obs_slots(Ctx *, const EngineDev *dE, const EngineDev &, const SlotDev *T, const ObsArgs &O,
                      const float *mm_val, int S) {
    const EngineDev &E = *dE;
    const int g = O.group;
    const GroupDev &G = E.grp[g];
    const int cells = G.view_w * G.view_h, C = E.n_channel, F = G.feature_size;
    const size_t rec = (size_t)cells * C, n = (size_t)E.A * S;
    memset(O.view, 0, n * rec * (O.half ? 2 : 4));
    memset(O.feature, 0, n * F * (O.half ? 2 : 4));
    const int *off = E.off + (size_t)g * (E.A + 1);
    const AgentSoA &s = cur_soa(E, O.curmask, g);
    std::vector<float> view(rec), feat(F);
    for (int a = 0; a < E.A; ++a) {
        const float *mm = mm_val ? mm_val + (size_t)a * E.G * cells : nullptr;
        for (int i = 0; i < off[a + 1] - off[a]; ++i) {
            const long gi = gidx(E, a, g, i);
            const int flat = slot_flat(T->tab, T->id_cap, a, s.id[gi], S);
            if (flat < 0) continue;
            int cx = -1, cy = -1;
            if (mm) minimap_cell(E, G.view_w, G.view_h, s.x[gi], s.y[gi], cx, cy);
            for (int vy = 0; vy < G.view_h; ++vy)
                for (int vx = 0; vx < G.view_w; ++vx)
                    obs_compose_cell(E, O.curmask, a, g, s.x[gi], s.y[gi], s.dir[gi], cx, cy, vy, vx, mm,
                                     view.data() + (size_t)(vy * G.view_w + vx) * C);
            obs_feature(E, O.curmask, a, g, i, feat.data());
            put(O.view, O.half, (size_t)flat * rec, view.data(), rec);
            put(O.feature, O.half, (size_t)flat * F, feat.data(), F);
        }
    }
}

}  // namespace be
}  // namespace mg
