"""The grid-size scenarios of tests/test_step_shapes_gpu.py on the host emulation (tests/emu/) against the reference: the
scenario builders and the phase code at 34,000 agents per arena on machines without a GPU.  The emulation does not
report step launches, so it refuses the "step_launch" info key."""
import os

import numpy as np
import pytest

import parity_common as pc
import step_shapes_common as sc
from test_render_launch_cpu import emu  # noqa: F401  (module fixture: builds the emulation library)

STEPS = 3


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


@pytest.mark.parametrize("name", list(sc.GRID_SCENARIOS))
def test_grid_size_scenario_on_the_emulation(emu, name):
    make, _, seed, kw = sc.GRID_SCENARIOS[name]
    want = pc.run_trace(make(checker_lib()), STEPS, seed, **kw)
    got = pc.run_trace(make(emu), STEPS, seed, **kw)
    assert max(sc.arena_sizes(want[0])) > sc.GRID_THRESHOLD
    pc.compare_traces(want, got, name)


def test_grid_size_battle_batch_on_the_emulation(emu):
    want = sc.arena_trace(sc.Games(sc.make_grid_battle_games(checker_lib())), STEPS, 5)
    got = sc.arena_trace(sc.Batch(sc.make_grid_battle(emu)), STEPS, 5)
    assert sc.arena_sizes(want[0]) == [2 * n for n in sc.GRID_BATTLE_AGENTS]
    pc.compare_traces(want, got, "grid battle")


def test_step_launch_is_refused_without_the_backend_report(emu):
    env = pc.make_battle(emu, 24, 30, 1)
    env.step()
    env.clear_dead()
    buf = np.full((10,), 7, np.int32)
    assert env._lib.env_get_info(env.game, -1, b"step_launch", buf.ctypes.data) == -1
    assert "step launches" in env._lib.magent_b200_last_error().decode()
    assert (buf == 7).all()
    with pytest.raises(RuntimeError, match="step_launch refused"):
        env._get_step_launch()
