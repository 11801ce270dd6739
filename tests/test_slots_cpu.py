"""The stable agent slots (magent_b200_get_slots) on the CPU.

The test-only host emulation (tests/emu/slots_emu.cc) runs the per-row lookup the CUDA kernel runs (slot_phases.h) over
the engine's own slot table, so these tests pin the engine's bookkeeping (placement, the table's width, snapshots,
restores, read-back before a mid-episode placement) to the restatement of tests/slots_common.py: in every game mode,
under the fuzz configs and an irregular batched caller, across restores and resets, and on the refusals."""
import os
import re
import subprocess

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import parity_common as pc
import slots_common as sc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SLOTS_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_slots.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation plus its restore loop (snapshots) and its slots loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "arena_restore_emu.cc", "slots_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(SLOTS_EMU_LIB) or os.path.getmtime(SLOTS_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(SLOTS_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", SLOTS_EMU_LIB], check=True, capture_output=True)
    return SLOTS_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the default emulation library, which has no slots loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    if not os.path.exists(pc.EMU_LIB) or os.path.getmtime(pc.EMU_LIB) < newest:
        subprocess.run([os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


# ---------------------------------------------------------------- every game mode
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_slots_equal_the_restatement_in_every_game_mode(emu, name):
    """every step, between the step and its clear_dead and after it; then agents added into one arena mid-episode and
    more play"""
    env = arc.SCENARIOS[name](emu, 5, _num_arenas=3)
    tr = sc.Slots(env)
    n = sc.play_and_check(tr, 5, 3)
    sc.add_somewhere(tr, 1, seed=6)
    n += sc.play_and_check(tr, 3, 4)
    assert n > 0


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


def test_slots_under_the_irregular_and_batch_fuzz_callers(emu):
    """random configs (5-8 groups, long and turning bodies, custom and fill placements, a group that stays empty), four
    arenas, driven by the irregular caller: skipped clear_dead, adds into every arena or one"""
    empty = 0
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed, _num_arenas=4)
        tr = sc.Slots(env)
        empty += any(env.get_num(h) == 0 for h in tr.hs)
        sc.play_irregular(tr, 8, seed)
    assert empty


def test_ragged_batch_with_an_empty_group(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=4)
    tr = sc.Slots(env)
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        tr.add(tr.hs[0], method="random", n=extra)
    env.select_arena(-1)
    assert sc.play_and_check(tr, 4, 1) > 0
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # 9 per arena; group 1 stays empty
    tr = sc.Slots(lone)
    sc.check(tr)
    h0, h1 = lone.get_handles()
    assert lone.get_slot_space(h1) == 0
    r, m = lone.get_slots(h1)
    assert r.shape == (0,) and m.shape == (2, 0)
    r, m = lone.get_slots(h0)
    np.testing.assert_array_equal(r, np.concatenate([np.arange(9), 9 + np.arange(9)]))
    np.testing.assert_array_equal(m, np.arange(18).reshape(2, 9))


# ---------------------------------------------------------------- restores, resets, snapshots
def test_slots_across_restores(emu):
    """cross-arena, self, subset and done-driven (NULL src) restores, keep_rng, a snapshot taken after mid-episode adds,
    adds after restores"""
    env = arc.make_duel(emu, 3, n=6, _num_arenas=4)
    tr = sc.Slots(env)
    pool = tr.snapshot()
    rs = np.random.RandomState(2)
    done_restores = 0
    for t in range(40):
        sc.random_step(env, rs)
        sc.check(tr, "step %d" % t)
        if t == 1:
            env.select_arena(2)
            tr.add(tr.hs[1], method="random", n=2)
            env.select_arena(-1)
            late = tr.snapshot()                      # holds arena 2's larger slot count
            sc.check(tr, "after the late snapshot")
        if t in (2, 5):
            tr.restore(pool, [-1, 2, -1, 0])          # cross-arena, a subset
        if t == 3:
            tr.restore(late, [2, 2, -1, -1], keep_rng=True)
        if t == 4:
            tr.restore(pool, [0, 1, 2, 3])            # every arena from itself
        if t >= 6:
            done_restores += sum(env.get_arena_done())
            tr.restore(pool, None)                    # the arenas whose step reported done
        sc.check(tr, "step %d after the restores" % t)
        if t == 7:
            tr.add(tr.hs[0], method="random", n=2)
            sc.check(tr, "after adding into restored arenas")
    assert done_restores > 0
    # freeing the snapshot that held the largest slot count shrinks the slot space once no arena holds it either
    S = [env.get_slot_space(h) for h in tr.hs]
    tr.restore(pool, [0, 1, 2, 3])
    tr.free(late)
    sc.check(tr, "after free_snapshot")
    assert [env.get_slot_space(h) for h in tr.hs] != S


def test_reset_starts_over(emu):
    env = pc.make_battle(emu, 16, 12, 3, _num_arenas=3)
    tr = sc.Slots(env)
    pool = tr.snapshot()
    rs = np.random.RandomState(5)
    for _ in range(3):
        sc.random_step(env, rs)
    env.select_arena(0)
    tr.add(tr.hs[0], method="random", n=4)
    env.select_arena(-1)
    sc.check(tr)
    tr.reset()
    # the snapshot keeps its slots in the slot space; the arenas start at 0
    assert [env.get_slot_space(h) for h in tr.hs] == [12, 12]
    for h in tr.hs:
        tr.add(h, method="random", n=5)
    sc.check(tr, "after reset")
    r, m = env.get_slots(tr.hs[1])
    np.testing.assert_array_equal(r, (np.arange(3).reshape(-1, 1) * 12 + np.arange(5)).reshape(-1))
    tr.free(pool)
    assert [env.get_slot_space(h) for h in tr.hs] == [5, 5]
    sc.check(tr, "after free_snapshot")
    tr.restore(tr.snapshot(), [2, -1, 0])
    sc.check(tr, "after a restore in the new episode")


def test_slots_survive_many_adds(emu):
    """ids far beyond the table's first width, culls in between: the table grows and keeps every slot"""
    import magent_b200 as magent
    env = magent.GridWorld(arc.duel_config(16), _lib=emu, _num_arenas=2)
    env.set_seed(1)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=6)
    tr = sc.Slots(env)
    rs = np.random.RandomState(9)
    for t in range(48):
        sc.random_step(env, rs)
        h = tr.hs[t % 2]
        if env.get_num(h) < 50:
            env.select_arena((t // 2) % 2)
            tr.add(h, method="random", n=4)
            env.select_arena(-1)
        if t % 6 == 5:
            sc.check(tr, "step %d" % t)
    sc.check(tr, "at the end")
    assert min(sum(len(d) for d in tr.state[a]) for a in range(2)) > 64, "the ids stayed within the first width"


# ---------------------------------------------------------------- refusals
def test_refusals_leave_the_buffers_untouched(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=2)
    tr = sc.Slots(env)
    h = tr.hs[0]
    want = sc.read_host(env, h)
    rows = np.full(4096, 7, dtype=np.int32)
    slots = np.full(4096, 7, dtype=np.int32)
    L = env._lib
    for g in (-1, 2, 9):
        assert L.magent_b200_get_slots(env.game, g, rows.ctypes.data, slots.ctypes.data) == -1
        assert b"invalid group handle" in L.magent_b200_last_error()
    assert L.magent_b200_get_slots(env.game, 0, None, None) == -1
    assert b"needs a row_slot or a slot_row buffer" in L.magent_b200_last_error()
    assert (rows == 7).all() and (slots == 7).all()
    for x, y in zip(sc.read_host(env, h), want):
        np.testing.assert_array_equal(x, y)
    # either buffer alone
    n, S = env.get_num(h), env.get_slot_space(h)
    assert L.magent_b200_get_slots(env.game, 0, rows.ctypes.data, None) == 0
    np.testing.assert_array_equal(rows[:n], want[0])
    assert (rows[n:] == 7).all()
    assert L.magent_b200_get_slots(env.game, 0, None, slots.ctypes.data) == 0
    np.testing.assert_array_equal(slots[:2 * S].reshape(2, S), want[1])
    assert (slots[2 * S:] == 7).all()


def test_a_backend_without_the_slots_loop_refuses_the_call(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    h = env.get_handles()[0]
    assert env.get_slot_space(h) == 20
    with pytest.raises(RuntimeError, match="no slots kernel"):
        env.get_slots(h)
    rows = np.full(64, 7, dtype=np.int32)
    assert env._lib.magent_b200_get_slots(env.game, 0, rows.ctypes.data, None) == -1
    assert (rows == 7).all()
    sc.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernel
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


@pytest.mark.parametrize("kernel", ["slots_kernel", "restore_slots_kernel"])
def test_slots_kernels_have_no_stack_or_spills(kernel):
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    m = re.search(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, open(LOG).read())
    assert m, kernel + " not in the ptxas report"
    assert tuple(int(v) for v in m.groups()[1:]) == (0, 0, 0), "%s: %s" % (kernel, m.groups()[1:])
