"""The global state (magent_b200_get_global_state) pinned to the reference on the CPU.

The test-only host emulation (tests/emu/) computes the state with the same per-cell function the CUDA kernel uses
(obs_phases.h state_compose_cell).  It runs in lockstep with the compiled reference (or the oracle's C restatement
where that is absent), and tests/global_state_common.py checks the state against every reference view and the
reference's own getters at every step."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import global_state_common as gs
import parity_common as pc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
STATE_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_state.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation (tests/emu/build.sh's sources) plus its global-state loop (tests/emu/global_state_emu.cc)"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "global_state_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(STATE_EMU_LIB) or os.path.getmtime(STATE_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(STATE_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", STATE_EMU_LIB], check=True, capture_output=True)
    return STATE_EMU_LIB


def checker():
    return pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB


def f16_state(env):
    out = np.empty((env.num_arenas,) + env.get_state_space(), dtype=np.float16)
    env._lib.magent_b200_get_global_state(env.game, ctypes.c_void_p(out.ctypes.data), 1)
    return out


def read_f32(env):
    return [env.get_global_state().copy()]


SCENARIOS = {
    "battle": lambda lib: pc.make_battle(lib, 30, 120, 3),
    "battle_rect": lambda lib: pc.make_battle_rect(lib),
    "pursuit": lambda lib: pc.make_pursuit(lib),
    "gather": lambda lib: pc.make_gather(lib, 30, 1),
    "food": lambda lib: pc.make_food(lib, 30, 3),
    "sector": lambda lib: pc.make_sector(lib),
    "multi4": lambda lib: pc.make_multi4(lib),
    "arrange": lambda lib: pc.make_arrange(lib),
}


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_state_matches_the_reference_views_and_getters(emu, name):
    assert gs.play_lockstep(SCENARIOS[name], emu, checker(), 15, 4, read_f32) == 15


def test_state_in_turn_mode(emu, tmp_path):
    """rotated view windows and bodies: headings read from the reference's replay frames"""
    gs.play_lockstep(lambda lib: pc.make_turn(lib, 30, 5), emu, checker(), 15, 5, read_f32, str(tmp_path), turn=True)


def test_arena_batch_equals_single_arena_references(emu):
    gs.play_batch_lockstep(lambda lib, seed, **kw: pc.make_battle(lib, 30, 80, seed, **kw), emu, checker(), 4, 12, 7,
                           read_f32)


@pytest.mark.parametrize("name", ["battle", "pursuit", "food"])
def test_f16_state_is_the_rounded_f32_state(emu, name):
    env = SCENARIOS[name](emu)
    rs = np.random.RandomState(2)
    for _ in range(8):
        s32 = env.get_global_state().copy()
        s16 = f16_state(env)
        np.testing.assert_array_equal(s16.view(np.uint16), s32.astype(np.float16).view(np.uint16))
        for h in env.get_handles():
            env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
        env.step()
        env.clear_dead()


def test_state_space_and_io_accounting(emu):
    """(H, W, C) for a non-square food_mode map; a host read counts its bytes as device->host traffic and leaves
    the observations alone"""
    env = pc.make_food(emu, 30, 3)
    assert env.get_state_space() == (30, 30, 1 + 1 + 2 * 3)
    rect = pc.make_battle_rect(emu, 56, 34)
    assert rect.get_state_space() == (34, 56, 5)
    h = env.get_handles()[1]
    v0 = env.get_observation(h)[0].copy()
    d0 = env.get_io_stats()["d2h"]
    s = env.get_global_state()
    assert s.shape == (1, 30, 30, 8) and s.dtype == np.float32
    assert env.get_io_stats()["d2h"] - d0 == s.nbytes
    np.testing.assert_array_equal(env.get_observation(h)[0], v0)


def test_select_arena_does_not_narrow_the_state(emu):
    env = pc.make_battle(emu, 20, 30, 1, _num_arenas=3)
    want = env.get_global_state().copy()
    env.select_arena(1)
    got = env.get_global_state()
    env.select_arena(-1)
    assert got.shape == (3, 20, 20, 5)
    np.testing.assert_array_equal(got, want)


# the ptxas report of both instantiations (test_render_spills_cpu.py reads the same file)
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")
KERNELS = {"float": "_ZN2mg2be19global_state_kernelIfEEvNS0_11StateParamsE",
           "__half": "_ZN2mg2be19global_state_kernelI6__halfEEvNS0_11StateParamsE"}


@pytest.mark.parametrize("T", sorted(KERNELS))
def test_global_state_kernel_has_no_stack_or_spills(T):
    import re
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    text = open(LOG).read()
    m = re.search(r"Function properties for %s\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % re.escape(KERNELS[T]), text)
    assert m, "global_state_kernel<%s> not in the ptxas report" % T
    assert tuple(int(v) for v in m.groups()) == (0, 0, 0), "global_state_kernel<%s>: %s" % (T, m.groups())
