// global_state_emu.cc -- TEST INFRASTRUCTURE ONLY.
//
// The host emulation's be::launch_global_state: a single-threaded loop over obs_phases.h state_compose_cell, the per-cell
// function the CUDA kernel (global_state_kernel) runs.  tests/test_global_state_cpu.py links it together with
// backend_emu.cc into tests/_emu/libmagent_emu_state.so, so the CPU tests pin that function to the reference.
#include <string.h>
#include <vector>
#include "../../magent_b200/csrc/backend.h"
#include "../../magent_b200/csrc/obs_phases.h"

namespace mg {
namespace be {

void launch_global_state(Ctx *, const EngineDev *dE, const EngineDev &, void *out, int half) {
    const EngineDev &E = *dE;
    const int C = state_channels(E);
    std::vector<float> cell(C);
    size_t o = 0;
    for (int a = 0; a < E.A; ++a)
        for (int y = 0; y < E.H; ++y)
            for (int x = 0; x < E.W; ++x) {
                state_compose_cell(E, a, x, y, cell.data());
                for (int ch = 0; ch < C; ++ch) {
                    if (half) ((_Float16 *)out)[o + ch] = (_Float16)cell[ch];      // round to nearest even
                    else ((float *)out)[o + ch] = cell[ch];
                }
                o += C;
            }
}

}  // namespace be
}  // namespace mg
