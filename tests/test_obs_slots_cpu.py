"""The slot-ordered observation (magent_b200_get_observation_slots) on the CPU.

The test-only host emulation (tests/emu/obs_slots_emu.cc) composes every occupied slot's record with the pieces the
row-ordered emulation uses and zeros the vacant ones, over the engine's own slot table and counts.  These tests pin the
engine's side of the call (shapes, the slot space, staging and copy-back, the byte count, refusals) to the restatement of
tests/obs_slots_common.py: the emulation's row-ordered observation gathered through get_slots, compared as bits."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import obs_slots_common as oc
import parity_common as pc
import slots_common as sc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SRC_DIR = os.path.join(pc.REPO, "magent_b200", "csrc")


def _emu_lib(name, emu_files):
    path = os.path.join(pc.REPO, "tests", "_emu", name)
    emu_srcs = [os.path.join(EMU_DIR, f) for f in emu_files]
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(path) or os.path.getmtime(path) < newest:
        os.makedirs(os.path.dirname(path), exist_ok=True)
        srcs = [os.path.join(SRC_DIR, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", path], check=True, capture_output=True)
    return path


@pytest.fixture(scope="module")
def emu():
    """the host emulation with its restore, slots and slot-ordered observation loops"""
    return _emu_lib("libmagent_emu_obs_slots.so",
                    ["backend_emu.cc", "arena_restore_emu.cc", "slots_emu.cc", "obs_slots_emu.cc"])


@pytest.fixture(scope="module")
def slots_only_emu():
    """an emulation with the slots loop but without the slot-ordered observation"""
    return _emu_lib("libmagent_emu_slots_no_obs.so", ["backend_emu.cc", "arena_restore_emu.cc", "slots_emu.cc"])


# ---------------------------------------------------------------- every game mode
@pytest.mark.parametrize("half", [0, 1], ids=["f32", "f16"])
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_equals_the_gathered_rows_in_every_game_mode(emu, name, half):
    """every step, between the step and its clear_dead (dead agents keep their slots) and after it; then agents added
    into one arena mid-episode, which leaves the other arenas' new slots vacant"""
    env = arc.SCENARIOS[name](emu, 5, _num_arenas=3)
    tr = sc.Slots(env)
    tally = []
    read = oc.slots_reader(half, tally=tally)
    sc.play_and_check(tr, 4, 3, read)
    sc.add_somewhere(tr, 1, seed=6)
    sc.play_and_check(tr, 2, 4, read)
    assert sum(tally) > 0


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


@pytest.mark.parametrize("half", [0, 1], ids=["f32", "f16"])
def test_under_the_irregular_and_batch_fuzz_callers(emu, half):
    """random configs (5-8 groups, long and turning bodies, a group that stays empty), four arenas, skipped clear_dead,
    adds into every arena or one"""
    tally = []
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed, _num_arenas=4)
        sc.play_irregular(sc.Slots(env), 5, seed, oc.slots_reader(half, tally=tally))
    assert sum(tally) > 0


def test_restores_move_records_between_slots(emu):
    """cross-arena, subset and self restores from a snapshot taken after a mid-episode add"""
    env = arc.make_duel(emu, 3, n=6, _num_arenas=4)
    tr = sc.Slots(env)
    pool = tr.snapshot()
    rs = np.random.RandomState(4)
    for t in range(10):
        sc.random_step(env, rs)
        if t == 1:
            env.select_arena(2)
            tr.add(tr.hs[1], method="random", n=3)
            env.select_arena(-1)
        if t in (3, 6):
            tr.restore(pool, [-1, 2, -1, 0])
        if t == 8:
            tr.restore(pool, [3, 3, 3, 3])
        sc.check(tr, "step %d" % t, oc.slots_reader(t % 2))


# ---------------------------------------------------------------- ragged batches, empty groups, extinct enemies
def test_ragged_batch_with_an_empty_group(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=4)
    tr = sc.Slots(env)
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        tr.add(tr.hs[0], method="random", n=extra)
    env.select_arena(-1)
    for half in (0, 1):
        sc.play_and_check(tr, 3, 1, oc.slots_reader(half))
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # group 1 stays empty: S = 0
    h0, h1 = lone.get_handles()
    for half in (0, 1):
        oc.check(lone, h0, half)
    v, f = lone.get_observation_slots(h1)
    assert v.shape == (2, 0) + lone.view_space[1] and f.shape == (2, 0) + lone.feature_space[1]


def test_an_extinct_enemy_next_to_vacant_slots(emu):
    """arena 0 has no agent of group 1: its minimap channels of group 1 are the reference's NaN, in the occupied slots
    only.  Arena 1 has more agents of group 0, so arena 0 has vacant slots, which stay +0.0 (the gather recipe of
    INTEGRATION.md would put NaN there: vacant slots gather row 0 and NaN * 0 is NaN)"""
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=16, _lib=emu, _num_arenas=2)
    env.set_seed(3)
    env.reset()
    h0, h1 = env.get_handles()
    env.select_arena(0)
    env.add_agents(h0, method="random", n=5)
    env.select_arena(1)
    env.add_agents(h0, method="random", n=9)
    env.add_agents(h1, method="random", n=6)
    env.select_arena(-1)
    tr = sc.Slots(env)
    assert env.get_slot_space(h0) == 9
    for half in (0, 1):
        assert oc.check(env, h0, half) == 14
        rc, v, f = oc.call_host(env, h0, half)
        assert np.isnan(v[0, :5]).any() and not np.isnan(v[1]).any()
        assert not v[0, 5:].view(np.uint16 if half else np.uint32).any()
        _row_slot, slot_row = sc.read_host(env, h0)
        rv, _rf = oc.row_observation(env, h0, half)
        recipe = rv[slot_row.clip(min=0)] * (slot_row >= 0)[..., None, None, None]
        assert np.isnan(recipe[0, 5:]).reshape(4, -1).any(-1).all()
    sc.play_and_check(tr, 2, 5, oc.slots_reader(0))


# ---------------------------------------------------------------- byte counting, refusals
def test_host_buffers_count_exactly_their_bytes(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    sc.Slots(env)
    h = env.get_handles()[1]
    g = env._hv(h)
    S = env.get_slot_space(h)
    for half in (0, 1):
        before = env.get_io_stats()["d2h"]
        rc, _v, _f = oc.call_host(env, h, half)
        assert rc == 0
        per = (int(np.prod(env.view_space[g])) + int(np.prod(env.feature_space[g]))) * (2 if half else 4)
        assert env.get_io_stats()["d2h"] - before == 3 * S * per


def test_refusals_write_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=2)
    sc.Slots(env)
    L = env._lib
    view = np.full(1 << 20, 7, np.uint8)
    feat = np.full(1 << 16, 7, np.uint8)
    bufs = (ctypes.c_void_p * 2)(view.ctypes.data, feat.ctypes.data)
    before = env.get_io_stats()["d2h"]
    for g in (-1, 2, 9):
        assert L.magent_b200_get_observation_slots(env.game, g, bufs, 0) == -1
        assert b"invalid group handle" in L.magent_b200_last_error()
    for half in (-1, 2, 16):
        assert L.magent_b200_get_observation_slots(env.game, 0, bufs, half) == -1
        assert b"half must be 0 or 1" in L.magent_b200_last_error()
    for p in ((None, feat.ctypes.data), (view.ctypes.data, None)):
        assert L.magent_b200_get_observation_slots(env.game, 0, (ctypes.c_void_p * 2)(*p), 0) == -1
        assert b"needs a view and a feature buffer" in L.magent_b200_last_error()
    assert (view == 7).all() and (feat == 7).all()
    assert env.get_io_stats()["d2h"] == before
    oc.check(env, env.get_handles()[0], 0)


def test_a_backend_without_the_kernel_refuses_the_call(slots_only_emu):
    env = pc.make_battle(slots_only_emu, 16, 20, 4)
    h = env.get_handles()[0]
    assert env.get_slot_space(h) == 20
    sc.read_host(env, h)                              # the slots loop itself is there
    with pytest.raises(RuntimeError, match="no slot-ordered observation kernel"):
        env.get_observation_slots(h)
    view = np.full(1 << 20, 7, np.uint8)
    feat = np.full(1 << 16, 7, np.uint8)
    bufs = (ctypes.c_void_p * 2)(view.ctypes.data, feat.ctypes.data)
    assert env._lib.magent_b200_get_observation_slots(env.game, 0, bufs, 1) == -1
    assert (view == 7).all() and (feat == 7).all()
    sc.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernels
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


@pytest.mark.parametrize("kernel", ["obs_slot_headers_kernel", "obs_headers_kernel", "obs_blank_minimap_kernel"])
def test_pre_pass_kernels_have_no_stack_or_spills(kernel):
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    found = re.findall(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads" % kernel, open(LOG).read())
    assert found, kernel + " not in the ptxas report"
    for m in found:
        assert tuple(int(v) for v in m[1:]) == (0, 0, 0), "%s: %s" % (m[0], m[1:])
