"""The reset pool (snapshot_arenas / restore_arenas) pinned to the reference on the CPU.

The test-only host emulation (tests/emu/) restores arenas with a single-threaded statement of the CUDA restore kernel
(tests/emu/arena_restore_emu.cc); everything else -- snapshot storage, capacities, counts, RNG, id counter, refusals
-- is the engine's own host code.  tests/arena_restore_common.py checks every arena against a reference game at every
step, and every restored arena against a fresh reference twin of its source arena."""
import os
import re
import subprocess

import numpy as np
import pytest

import arena_restore_common as ar
import parity_common as pc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
RESTORE_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_restore.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation plus its restore and global-state loops"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "global_state_emu.cc", "arena_restore_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest, os.path.getmtime(os.path.join(pc.REPO, "include", "magent_b200_ext.h"))] +
                 [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(RESTORE_EMU_LIB) or os.path.getmtime(RESTORE_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(RESTORE_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", RESTORE_EMU_LIB], check=True, capture_output=True)
    return RESTORE_EMU_LIB


def checker():
    return pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB


@pytest.mark.parametrize("name", sorted(ar.SCENARIOS))
def test_restart_equals_a_fresh_episode(emu, name):
    assert ar.play_restarts(ar.SCENARIOS[name], emu, checker()) >= 8


def test_done_arenas_restart_on_their_own(emu):
    """src = NULL: the arenas that finished (one army wiped out) restart; the others play on"""
    n = ar.play_restarts(ar.make_duel, emu, checker(), steps=60, seed=3, plan={t: None for t in range(60)}, arenas=8)
    assert n >= 3, "no arena finished: the scenario no longer exercises the done-driven restore"


@pytest.mark.parametrize("name", ["battle", "pursuit", "turn"])
def test_keep_rng_continues_the_arenas_own_stream(emu, name):
    assert ar.play_restarts(ar.SCENARIOS[name], emu, checker(), keep_rng=True) >= 8


@pytest.mark.parametrize("name", ["battle", "food", "arrange"])
def test_mid_episode_snapshot_replays_identically(emu, name):
    ar.mid_episode_replay(ar.SCENARIOS[name], emu)


def test_add_agents_after_a_restore_continues_the_ids(emu):
    L = ar.Lockstep(ar.make_duel, emu, checker(), 4, 9)
    pool = L.snapshot()
    for _ in range(12):
        L.step()
    # the restored arenas' counts are exact at once, without a step
    nums = [L.eng.get_arena_nums(h).copy() for h in L.eng.get_handles()]
    assert L.restore(pool, [1, -1, 3, 0]) == 3
    for g, h in enumerate(L.eng.get_handles()):
        want = [ref.get_num(ref.get_handles()[g]) for ref in L.refs]
        np.testing.assert_array_equal(L.eng.get_arena_nums(h), want)
        assert L.eng.get_num(h) == sum(want)
    assert any(list(L.eng.get_arena_nums(h)) != list(x) for h, x in zip(L.eng.get_handles(), nums)), \
        "the restore was supposed to change the counts"
    L.eng.add_agents(L.eng.get_handles()[0], method="random", n=3)
    for ref in L.refs:
        ref.add_agents(ref.get_handles()[0], method="random", n=3)
    L.check(" (after add_agents)")
    for _ in range(3):
        L.step()
        L.check()


def test_restore_after_capacity_growth(emu):
    """a snapshot taken from the other ping-pong buffer at 64 per group, restored after a late add_agents re-allocated
    the device image at a larger capacity (which also resets the buffer selector): source and destination strides
    differ"""
    L = ar.Lockstep(ar.SCENARIOS["battle"], emu, checker(), 4, 11)
    L.step()
    pool = L.snapshot()
    L.step()
    L.step()
    L.eng.add_agents(L.eng.get_handles()[0], method="random", n=60)
    for ref in L.refs:
        ref.add_agents(ref.get_handles()[0], method="random", n=60)
    assert max(L.eng.get_arena_nums(L.eng.get_handles()[0])) > 64
    L.check()
    L.step()
    assert L.restore(pool, [2, -1, 0, 1]) == 3
    for _ in range(4):
        L.check()
        L.step()


def _fingerprint(env):
    hs = env.get_handles()
    return ([env.get_arena_nums(h).copy() for h in hs] + [env.get_agent_id(h).copy() for h in hs] +
            [env.get_pos(h).copy() for h in hs] + [env.get_global_state().copy(), env.get_arena_rng().copy()])


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_refusals_leave_the_state_alone(emu, tmp_path):
    env = ar.SCENARIOS["battle"](emu, 4, _num_arenas=3)
    pool = env.snapshot_arenas()
    hs = env.get_handles()
    for h in hs:
        env.set_action(h, np.zeros((env.get_num(h),), np.int32))
    env.step()
    env.clear_dead()
    before = _fingerprint(env)
    for bad in ([0, 1, 3], [-2, 0, 0]):                 # host values outside [-1, A)
        with pytest.raises(RuntimeError, match="outside"):
            env.restore_arenas(pool, np.asarray(bad, np.int32))
    with pytest.raises(RuntimeError, match="unknown or freed"):
        env.restore_arenas(pool + 7)
    env.set_action(hs[0], np.zeros((env.get_num(hs[0]),), np.int32))
    with pytest.raises(RuntimeError, match="actions are set"):
        env.restore_arenas(pool, np.arange(3, dtype=np.int32))
    env.step()
    env.clear_dead()
    before = _fingerprint(env)
    other = env.snapshot_arenas()
    env.free_snapshot(other)
    for call in (lambda: env.restore_arenas(other), lambda: env.free_snapshot(other)):
        with pytest.raises(RuntimeError, match="unknown or freed"):
            call()
    _same(before, _fingerprint(env))
    # another geometry: one more group
    env.new_group("small")
    with pytest.raises(RuntimeError, match="different geometry"):
        env.restore_arenas(pool)
    # rendering started
    ren = ar.SCENARIOS["battle"](emu, 4, _num_arenas=2)
    rp = ren.snapshot_arenas()
    ren.set_render_dir(str(tmp_path))
    ren.render()
    before = _fingerprint(ren)
    with pytest.raises(RuntimeError, match="rendering"):
        ren.restore_arenas(rp, np.zeros((2,), np.int32))
    _same(before, _fingerprint(ren))


def test_turn_mode_change_is_another_geometry(emu):
    env = ar.SCENARIOS["battle"](emu, 4, _num_arenas=2)
    pool = env.snapshot_arenas()
    import ctypes
    env._lib.env_config_game(env.game, b"turn_mode", ctypes.byref(ctypes.c_bool(True)))
    with pytest.raises(RuntimeError, match="different geometry"):
        env.restore_arenas(pool)


def test_num_bound_covers_the_snapshot(emu):
    env = ar.make_duel(emu, 2, _num_arenas=3)
    hs = env.get_handles()
    rs = np.random.RandomState(0)
    assert [env.get_num_bound(h) for h in hs] == [env.get_num(h) for h in hs]
    pool = env.snapshot_arenas()
    for _ in range(12):
        for h in hs:
            env.set_action(h, rs.randint(0, 21, size=env.get_num(h)).astype(np.int32))
        env.step()
        env.clear_dead()
    nums = [env.get_arena_nums(h) for h in hs]
    assert sum(int(x.sum()) for x in nums) < 2 * 3 * 8, "agents are supposed to die"
    for g, h in enumerate(hs):
        assert env.get_num_bound(h) == 3 * 8             # every arena may be restored to its 8 per group
    env.free_snapshot(pool)
    assert [env.get_num_bound(h) for h in hs] == [env.get_num(h) for h in hs]


# the ptxas report (test_render_spills_cpu.py reads the same file)
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")
KERNELS = {"restore_kernel": "_ZN2mg2be14restore_kernelENS0_13RestoreParamsE",
           "restore_finish_kernel": "_ZN2mg2be21restore_finish_kernelEPKNS_9EngineDevEPKiS5_",
           "arena_done_kernel": "_ZN2mg2be17arena_done_kernelEPKNS_9EngineDevEPi"}


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_restore_kernels_have_no_stack_or_spills(kernel):
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    text = open(LOG).read()
    m = re.search(r"Function properties for %s\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % re.escape(KERNELS[kernel]), text)
    assert m, "%s not in the ptxas report" % kernel
    assert tuple(int(v) for v in m.groups()) == (0, 0, 0), "%s: %s" % (kernel, m.groups())
