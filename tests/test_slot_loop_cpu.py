"""The slot-ordered step loop (magent_b200_set_action_slots, _get_reward_slots, _get_action_mask_slots) on the CPU.

The test-only host emulation (tests/emu/slot_loop_emu.cc) states the three launches single-threaded over the engine's
own slot table and counts.  These tests pin the engine's side of the calls (the action order, staging and copy-back,
the byte counts, refusals) and the definitions: an engine driven through set_action_slots stays bit for bit the twin of
one driven through set_action in rows, and the reward, status and mask equal the row-ordered outputs gathered through
get_slots (tests/slot_loop_common.py)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import parity_common as pc
import slot_loop_common as lc
import slots_common as sc


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SRC_DIR = os.path.join(pc.REPO, "magent_b200", "csrc")
SLOT_LOOP_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_slot_loop.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation with every per-feature loop, the slot-ordered step loop included"""
    emu_srcs = [os.path.join(EMU_DIR, f) for f in sorted(os.listdir(EMU_DIR)) if f.endswith("_emu.cc")]
    assert os.path.join(EMU_DIR, "slot_loop_emu.cc") in emu_srcs
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(SLOT_LOOP_EMU_LIB) or os.path.getmtime(SLOT_LOOP_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(SLOT_LOOP_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(SRC_DIR, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", SLOT_LOOP_EMU_LIB], check=True,
                       capture_output=True)
    return SLOT_LOOP_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the plain emulation (tests/emu/build.sh): no slot kernels at all"""
    subprocess.run(["bash", os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


# ---------------------------------------------------------------- twin equivalence
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_twin_in_every_game_mode(emu, name):
    """every step and cull; outputs checked on the slot-driven engine; then agents added into one arena"""
    tw = lc.Twin(lambda lib: arc.SCENARIOS[name](lib, 5, _num_arenas=3), emu)
    rs = np.random.RandomState(2)
    tally = []
    for t in range(4):
        tw.step(rs, t, cull=False)
        lc.check_outputs(tw.s, tally, "step %d before clear_dead" % t)
        tw.both(lambda e: e.clear_dead())
        tw.check("step %d after clear_dead" % t)
        lc.check_outputs(tw.s, tally, "step %d" % t)
    for e in (tw.s, tw.r):
        sc.add_somewhere(sc.Slots(e), 1, seed=6)
    tw.check("after adding into arena 1")
    for t in range(4, 6):
        tw.step(rs, t)
        lc.check_outputs(tw.s, tally, "step %d" % t)
    assert sum(tally) > 0


MANY_GROUP_SEEDS = [70001, 70003, 70005, 70006]


@pytest.mark.parametrize("seed", MANY_GROUP_SEEDS + [2, 6, 13, 1004, 100002])
def test_twin_under_the_irregular_caller(emu, seed):
    """fuzz configs (70000-seeds: 5-8 groups), skipped culls, agents added mid-episode into every arena or one, groups
    acting in a random order, slot and row actions mixed"""
    tw = lc.Twin(lambda lib: fz.make_env(lib, seed, _num_arenas=4), emu)
    if seed in MANY_GROUP_SEEDS:
        assert 5 <= len(tw.hs) <= 8
    rs = np.random.RandomState(seed ^ 0x5107)
    H, W, _C = tw.s.get_state_space()
    for t in range(6):
        tw.step(rs, t, cull=rs.rand() < 0.65, order=list(rs.permutation(len(tw.hs))), mix=True)
        lc.check_outputs(tw.s, what="seed %d step %d" % (seed, t))
        if rs.rand() < 0.4:
            arena = int(rs.randint(-1, 4))
            g = int(rs.randint(0, len(tw.hs)))
            pos = [[int(rs.randint(1, W - 1)), int(rs.randint(1, H - 1)), int(rs.randint(0, 4))] for _ in range(6)]
            for e in (tw.s, tw.r):
                e.select_arena(arena)
                e.add_agents(e.get_handles()[g], method="custom", pos=pos)
                e.select_arena(-1)
            tw.check("seed %d step %d after adding into arena %d" % (seed, t, arena))
            lc.check_outputs(tw.s, what="seed %d step %d after adding" % (seed, t))
    assert tw.checked > 6


@pytest.mark.parametrize("keep_rng", [False, True])
def test_twin_across_restores(emu, keep_rng):
    """restores with a host src, the done flags (NULL src) and every arena from itself, between steps"""
    tw = lc.Twin(lambda lib: arc.make_duel(lib, 3, n=6, _num_arenas=4), emu)
    pools = tw.both(lambda e: e.snapshot_arenas())
    assert pools[0] == pools[1]
    rs = np.random.RandomState(4)
    plan = {1: [-1, 2, -1, 0], 3: None, 5: [0, 1, 2, 3], 6: [3, 3, -1, 1]}
    for t in range(8):
        tw.step(rs, t, mix=t % 2 == 1)
        if t in plan:
            src = None if plan[t] is None else np.asarray(plan[t], np.int32)
            for e, p in zip((tw.s, tw.r), pools):
                e.restore_arenas(p, src, keep_rng=keep_rng)
            tw.check("step %d after restoring %s" % (t, plan[t]))
            lc.check_outputs(tw.s, what="step %d after restoring" % t)


def test_two_groups_in_both_orders(emu):
    """the step's action order is the order of the first set_action or set_action_slots per group, whichever kind"""
    for order in ([0, 1], [1, 0]):
        tw = lc.Twin(lambda lib: pc.make_battle(lib, 16, 24, 5, _num_arenas=2), emu)
        rs = np.random.RandomState(sum(order) + order[0])
        for t in range(5):
            tw.step(rs, t, order=order, mix=True)


# ---------------------------------------------------------------- reward and status
def test_status_marks_the_dead_until_the_cull(emu):
    """the slot-native loop with actions drawn from the slot-ordered mask, dense enough that agents die"""
    env = pc.make_battle(emu, 16, 50, 1, _num_arenas=3)
    rs = np.random.RandomState(0)
    seen_dead = 0
    for t in range(12):
        for h in env.get_handles():
            mask = env.get_action_mask_slots(h)
            env.set_action_slots(h, (rs.rand(*mask.shape) * mask).argmax(-1).astype(np.int32))
        env.step()
        for h in env.get_handles():
            lc.check_reward(env, h, what="step %d" % t)
            seen_dead += int((env.get_reward_slots(h)[1] == 2).sum())
        env.clear_dead()
        for h in env.get_handles():
            lc.check_reward(env, h, what="step %d after the cull" % t)
            assert not (env.get_reward_slots(h)[1] == 2).any()
    assert seen_dead > 0


def test_vacant_rewards_are_positive_zero(emu):
    """a negative shared reward (the step penalty) in every occupied slot, +0.0 in the vacant ones"""
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    tr = sc.Slots(env)
    env.select_arena(1)
    tr.add(tr.hs[0], method="random", n=11)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    for t in range(3):
        sc.random_step(env, rs)
        h = tr.hs[0]
        reward, status = env.get_reward_slots(h)
        _rs, slot_row = sc.read_host(env, h)
        assert (slot_row < 0).any()
        assert not reward[slot_row < 0].view(np.uint32).any()
        assert not status[slot_row < 0].any()
        lc.check_reward(env, h)


def test_restored_arenas_show_their_snapshot_slots(emu):
    env = arc.make_duel(emu, 3, n=6, _num_arenas=4)
    tr = sc.Slots(env)
    env.select_arena(2)
    tr.add(tr.hs[1], method="random", n=3)
    env.select_arena(-1)
    pool = tr.snapshot()
    rs = np.random.RandomState(9)
    for t in range(4):
        sc.random_step(env, rs)
    tr.restore(pool, [2, -1, 0, 2])
    sc.check(tr, "after the restore")
    for h in tr.hs:
        lc.check_reward(env, h)
        lc.check_mask(env, h)
        _rr, slot_row = sc.read_host(env, h)
        _r, status = env.get_reward_slots(h)
        np.testing.assert_array_equal(status[0] > 0, slot_row[0] >= 0)
        np.testing.assert_array_equal(status[0], status[3])                      # both from snapshot arena 2


def test_host_buffers_count_exactly_their_bytes(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    sc.Slots(env)
    sc.random_step(env, np.random.RandomState(0), cull=False)
    for h in env.get_handles():
        S = env.get_slot_space(h)
        na = env.get_action_space(h)[0]
        reward = np.empty((3, S), np.float32)
        status = np.empty((3, S), np.uint8)
        for r, s, nbytes in ((reward, status, 15 * S), (reward, None, 12 * S), (None, status, 3 * S)):
            before = env.get_io_stats()
            assert lc.call_reward(env, h, r, s) == 0
            after = env.get_io_stats()
            assert after["d2h"] - before["d2h"] == nbytes and after["h2d"] == before["h2d"]
        mask = np.empty((3, S, na), np.uint8)
        before = env.get_io_stats()["d2h"]
        assert lc.call_mask(env, h, mask) == 0
        assert env.get_io_stats()["d2h"] - before == 3 * S * na
        act = lc.slot_actions(env, h, np.random.RandomState(1))
        before = env.get_io_stats()
        assert lc.call_set(env, h, act) == 0
        after = env.get_io_stats()
        assert after["h2d"] - before["h2d"] == 12 * S and after["d2h"] == before["d2h"]


# ---------------------------------------------------------------- mask
def test_mask_sentinels_past_every_output_stay(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    tr = sc.Slots(env)
    env.select_arena(0)
    tr.add(tr.hs[1], method="random", n=5)
    env.select_arena(-1)
    rs = np.random.RandomState(3)
    for t in range(3):
        sc.random_step(env, rs, cull=t != 1)
        for h in tr.hs:
            S, na = env.get_slot_space(h), env.get_action_space(h)[0]
            mask = np.full(3 * S * na + 64, 0xA5, np.uint8)
            reward = np.full(3 * S + 16, -7.0, np.float32)
            status = np.full(3 * S + 64, 0xA5, np.uint8)
            assert lc.call_mask(env, h, mask) == 0 and lc.call_reward(env, h, reward, status) == 0
            assert (mask[3 * S * na:] == 0xA5).all() and (status[3 * S:] == 0xA5).all() and (reward[3 * S:] == -7).all()
            lc.check_mask(env, h, mask[:3 * S * na].reshape(3, S, na), "step %d" % t)
            lc.check_reward(env, h, (reward[:3 * S].reshape(3, S), status[:3 * S].reshape(3, S)), "step %d" % t)


def test_an_empty_slot_space(emu):
    """S == 0: set_action_slots only registers the group's action (NULL allowed), the outputs are empty"""
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    env.reset()
    h0, h1 = env.get_handles()
    env.add_agents(h0, method="random", n=9)
    assert env.get_slot_space(h1) == 0
    assert lc.call_set(env, h1, None) == 0
    snap = env.snapshot_arenas()
    assert env._lib.magent_b200_restore_arenas(env.game, snap, None, 0) == -1       # actions are set for the step
    env.set_action_slots(h1, np.zeros((2, 0), np.int32))
    r, s = env.get_reward_slots(h1)
    assert r.shape == (2, 0) and s.shape == (2, 0)
    assert env.get_action_mask_slots(h1).shape == (2, 0, env.get_action_space(h1)[0])
    env.set_action_slots(h0, lc.slot_actions(env, h0, np.random.RandomState(0)))
    env.step()
    lc.check_outputs(env)


# ---------------------------------------------------------------- refusals
def test_refusals_write_nothing_and_register_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=2)
    sc.Slots(env)
    snap = env.snapshot_arenas()
    L = env._lib
    big = np.full(1 << 16, 0x5A, np.uint8)
    act = np.zeros((2, 20), np.int32)
    before = env.get_io_stats()
    for g in (-1, 2, 9):
        assert L.magent_b200_set_action_slots(env.game, g, act.ctypes.data) == -1
        assert b"invalid group handle" in L.magent_b200_last_error()
        assert L.magent_b200_get_reward_slots(env.game, g, big.ctypes.data, big.ctypes.data) == -1
        assert b"invalid group handle" in L.magent_b200_last_error()
        assert L.magent_b200_get_action_mask_slots(env.game, g, big.ctypes.data) == -1
        assert b"invalid group handle" in L.magent_b200_last_error()
    assert L.magent_b200_set_action_slots(env.game, 0, None) == -1
    assert b"needs an action buffer" in L.magent_b200_last_error()
    assert L.magent_b200_get_reward_slots(env.game, 0, None, None) == -1
    assert b"needs a reward or a status buffer" in L.magent_b200_last_error()
    assert L.magent_b200_get_action_mask_slots(env.game, 0, None) == -1
    assert b"needs a mask buffer" in L.magent_b200_last_error()
    assert (big == 0x5A).all() and env.get_io_stats() == before
    assert L.magent_b200_restore_arenas(env.game, snap, None, 0) == 0               # no action order was left behind
    with pytest.raises(ValueError):
        env.set_action_slots(env.get_handles()[0], np.zeros((2, 19), np.int32))
    with pytest.raises(ValueError):
        env.set_action_slots(env.get_handles()[0], np.zeros((2, 20), np.int64))
    assert L.magent_b200_restore_arenas(env.game, snap, None, 0) == 0
    env.set_action_slots(env.get_handles()[0], act)
    assert L.magent_b200_restore_arenas(env.game, snap, None, 0) == -1
    assert b"while actions are set" in L.magent_b200_last_error()


def test_a_backend_without_the_kernels_refuses_the_calls(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    h = env.get_handles()[0]
    assert env.get_slot_space(h) == 20
    L = env._lib
    big = np.full(1 << 16, 0x5A, np.uint8)
    before = env.get_io_stats()
    assert L.magent_b200_set_action_slots(env.game, 0, big.ctypes.data) == -1
    assert b"no slot-ordered action kernel" in L.magent_b200_last_error()
    assert L.magent_b200_get_reward_slots(env.game, 0, big.ctypes.data, None) == -1
    assert b"no slot-ordered reward kernel" in L.magent_b200_last_error()
    assert L.magent_b200_get_action_mask_slots(env.game, 0, big.ctypes.data) == -1
    assert b"no slot-ordered action-mask kernel" in L.magent_b200_last_error()
    with pytest.raises(RuntimeError, match="no slot-ordered reward kernel"):
        env.get_reward_slots(h)
    assert (big == 0x5A).all() and env.get_io_stats() == before
    sc.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernels
@pytest.mark.parametrize("kernel", ["set_action_slots_kernel", "reward_slots_kernel", "action_mask_slots_kernel"])
def test_kernels_have_no_stack_or_spills(kernel):
    import re
    from magent_b200 import build as b
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    log = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")
    b.build(force=not os.path.exists(log))
    found = re.findall(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads" % kernel, open(log).read())
    assert found, kernel + " not in the ptxas report"
    for m in found:
        assert tuple(int(v) for v in m[1:]) == (0, 0, 0), "%s: %s" % (m[0], m[1:])
