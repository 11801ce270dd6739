"""The slot-ordered mean action and neighbours (magent_b200_get_mean_action_slots, _get_neighbours_slots) on the CPU.

The test-only host emulation (tests/emu/nbr_slots_emu.cc) states the two launches single-threaded over nbr_phases.h and
slot_phases.h.  These tests pin the engine's side of the calls (staging and copy-back, the byte counts, refusals) and the
definitions: every output equals the row-ordered call gathered through get_slots, with every listed neighbour's row
translated to its flat slot (tests/nbr_slots_common.py), in every game mode, under the fuzz configs, across culls,
mid-episode additions and host-src restores."""
import os
import re
import subprocess

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import nbr_slots_common as ns
import parity_common as pc
import slots_common as sc


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SRC_DIR = os.path.join(pc.REPO, "magent_b200", "csrc")
NBR_SLOTS_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_nbr_slots.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation with every per-feature loop, the slot-ordered mean action and neighbours included"""
    emu_srcs = [os.path.join(EMU_DIR, f) for f in sorted(os.listdir(EMU_DIR)) if f.endswith("_emu.cc")]
    assert os.path.join(EMU_DIR, "nbr_slots_emu.cc") in emu_srcs
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(NBR_SLOTS_EMU_LIB) or os.path.getmtime(NBR_SLOTS_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(NBR_SLOTS_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(SRC_DIR, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", NBR_SLOTS_EMU_LIB], check=True,
                       capture_output=True)
    return NBR_SLOTS_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the plain emulation (tests/emu/build.sh): no slot kernels at all"""
    subprocess.run(["bash", os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


def without_rel_and_count(env, k, what=""):
    """the raw calls with rel and count NULL (and with count alone) equal the full call's parts"""
    A = env.num_arenas
    for h, o in ns.pairs(env):
        S = env.get_slot_space(h)
        if S == 0:
            continue
        na = env.get_action_space(o)[0]
        mean = np.full((A, S, na), -5.0, np.float32)
        assert ns.call_mean(env, h, o, mean, None) == 0
        ns.check_mean(env, h, o, (mean, None), what)
        idx = np.full((A, S, k), -5, np.int32)
        assert ns.call_neighbours(env, h, o, k, idx, None, None) == 0
        ns.check_neighbours(env, h, o, k, (idx, None, None), what)
        count = np.full((A, S), -5, np.int32)
        assert ns.call_neighbours(env, h, o, k, idx, None, count) == 0
        ns.check_neighbours(env, h, o, k, (idx, None, count), what)


# ---------------------------------------------------------------- against the restatement
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_every_game_mode(emu, name):
    """every (group, of) pair and k in {1, 3, 32} after every step and cull, then after agents are added into one arena"""
    env = arc.SCENARIOS[name](emu, 5, _num_arenas=3)
    tr = sc.Slots(env)
    rs = np.random.RandomState(3)
    listed = 0
    for t in range(4):
        sc.random_step(env, rs, cull=False)
        listed += ns.check_all(env, what="%s step %d before clear_dead" % (name, t))
        env.clear_dead()
        listed += ns.check_all(env, what="%s step %d" % (name, t))
    without_rel_and_count(env, 3, name)
    sc.add_somewhere(tr, 1, seed=6)
    listed += ns.check_all(env, what="%s after adding into arena 1" % name)
    sc.random_step(env, rs)
    listed += ns.check_all(env, what="%s after the last step" % name)
    assert listed > 0


MANY_GROUP_SEEDS = [70001, 70003, 70005, 70006]


@pytest.mark.parametrize("seed", MANY_GROUP_SEEDS + [2, 6, 13, 1004, 100002])
def test_fuzz_configs(emu, seed):
    """the fuzz configs (70000-seeds: 5-8 groups) under the irregular caller: skipped culls, agents added mid-episode
    into every arena or one"""
    env = fz.make_env(emu, seed, _num_arenas=3)
    if seed in MANY_GROUP_SEEDS:
        assert 5 <= len(env.get_handles()) <= 8
    rs = np.random.RandomState(seed ^ 0x3b5)
    H, W, _C = env.get_state_space()
    ks = (1, 3, 32) if len(env.get_handles()) <= 4 else (3, 32)
    for t in range(4):
        sc.random_step(env, rs, cull=rs.rand() < 0.65)
        ns.check_all(env, ks, "seed %d step %d" % (seed, t))
        if rs.rand() < 0.5:
            arena = int(rs.randint(-1, 3))
            g = int(rs.randint(0, len(env.get_handles())))
            pos = [[int(rs.randint(1, W - 1)), int(rs.randint(1, H - 1)), int(rs.randint(0, 4))] for _ in range(6)]
            env.select_arena(arena)
            env.add_agents(env.get_handles()[g], method="custom", pos=pos)
            env.select_arena(-1)
            ns.check_all(env, ks, "seed %d step %d after adding into arena %d" % (seed, t, arena))


@pytest.mark.parametrize("keep_rng", [False, True])
def test_host_src_restores(emu, keep_rng):
    """restores with a host src, the done flags (NULL src) and every arena from itself, between steps"""
    env = arc.make_duel(emu, 3, n=6, _num_arenas=4)
    pool = env.snapshot_arenas()
    rs = np.random.RandomState(4)
    plan = {1: [-1, 2, -1, 0], 3: None, 4: [0, 1, 2, 3], 5: [3, 3, -1, 1]}
    for t in range(6):
        sc.random_step(env, rs)
        if t in plan:
            env.restore_arenas(pool, None if plan[t] is None else np.asarray(plan[t], np.int32), keep_rng=keep_rng)
            ns.check_all(env, what="step %d after restoring %s" % (t, plan[t]))


def test_vacant_slots_and_episode_stable_indices(emu):
    """culls open vacant slots (zero mean rows, -1 neighbour rows); an index taken one step earlier names, after the
    next cull, the same agent or a vacant slot, never another agent"""
    env = pc.make_battle(emu, 16, 50, 1, _num_arenas=2)
    rs = np.random.RandomState(0)
    hs = env.get_handles()
    vacant = stale = 0

    def owners(o):
        """the agent id in every flat slot of group o, -1 where vacant"""
        row_slot, _sr = sc.read_host(env, o)
        owner = np.full(env.num_arenas * env.get_slot_space(o), -1, np.int64)
        owner[row_slot] = env.get_agent_id(o)
        return owner

    before = {}
    for t in range(10):
        for h in hs:                                # actions drawn from the legal ones: dense enough that agents die
            mask = env.get_action_mask(h).view(np.uint8)
            env.set_action(h, (rs.rand(*mask.shape) * mask).argmax(-1).astype(np.int32))
        env.step()
        env.clear_dead()
        for h in hs:
            _rs, slot_row = sc.read_host(env, h)
            mean, count = env.get_mean_action_slots(h)
            idx, rel, cnt = env.get_neighbours_slots(h, 8)
            vac = slot_row < 0
            vacant += int(vac.sum())
            assert not mean[vac].view(np.uint32).any() and not count[vac].any()
            assert (idx[vac] == -1).all() and (rel[vac] == -1).all() and not cnt[vac].any()
        for h in hs:
            for o in hs:
                owner = owners(o)
                key = env._hv(h), env._hv(o)
                if key in before:
                    idx0, owner0 = before[key]
                    used = idx0[idx0 >= 0]
                    assert ((owner[used] == owner0[used]) | (owner[used] == -1)).all(), "step %d" % t
                    stale += int((owner[used] == -1).sum())
                before[key] = (env.get_neighbours_slots(h, 8, o)[0].copy(), owner)
        ns.check_all(env, (8,), "step %d" % t)
    assert vacant > 0 and stale > 0


def test_host_buffers_count_exactly_their_bytes(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    sc.Slots(env)
    sc.random_step(env, np.random.RandomState(0), cull=False)
    for h, o in ns.pairs(env):
        S, na = env.get_slot_space(h), env.get_action_space(o)[0]
        mean = np.empty((3, S, na), np.float32)
        count = np.empty((3, S), np.int32)
        for c, nbytes in ((count, 12 * S * na + 12 * S), (None, 12 * S * na)):
            before = env.get_io_stats()
            assert ns.call_mean(env, h, o, mean, c) == 0
            after = env.get_io_stats()
            assert after["d2h"] - before["d2h"] == nbytes and after["h2d"] == before["h2d"]
        k = 5
        idx = np.empty((3, S, k), np.int32)
        rel = np.empty((3, S, k, 2), np.int32)
        for r, c, nbytes in ((rel, count, 36 * S * k + 12 * S), (None, count, 12 * S * k + 12 * S),
                             (rel, None, 36 * S * k), (None, None, 12 * S * k)):
            before = env.get_io_stats()
            assert ns.call_neighbours(env, h, o, k, idx, r, c) == 0
            after = env.get_io_stats()
            assert after["d2h"] - before["d2h"] == nbytes and after["h2d"] == before["h2d"]


def test_sentinels_past_every_output_stay(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    tr = sc.Slots(env)
    env.select_arena(0)
    tr.add(tr.hs[1], method="random", n=5)
    env.select_arena(-1)
    rs = np.random.RandomState(3)
    for t in range(3):
        sc.random_step(env, rs, cull=t != 1)
        for h, o in ns.pairs(env):
            S, na, k = env.get_slot_space(h), env.get_action_space(o)[0], 4
            n = 3 * S
            mean = np.full(n * na + 16, -7.0, np.float32)
            mc = np.full(n + 16, -7, np.int32)
            idx = np.full(n * k + 16, -7, np.int32)
            rel = np.full(2 * n * k + 16, -7, np.int32)
            cnt = np.full(n + 16, -7, np.int32)
            assert ns.call_mean(env, h, o, mean, mc) == 0 and ns.call_neighbours(env, h, o, k, idx, rel, cnt) == 0
            for x, m in ((mean, n * na), (mc, n), (idx, n * k), (rel, 2 * n * k), (cnt, n)):
                assert (x[m:] == -7).all()
            what = "step %d" % t
            ns.check_mean(env, h, o, (mean[:n * na].reshape(3, S, na), mc[:n].reshape(3, S)), what)
            ns.check_neighbours(env, h, o, k, (idx[:n * k].reshape(3, S, k), rel[:2 * n * k].reshape(3, S, k, 2),
                                               cnt[:n].reshape(3, S)), what)


def test_an_empty_slot_space(emu):
    """S == 0 writes nothing and returns 0; an empty `of` lists no neighbours"""
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    env.reset()
    h0, h1 = env.get_handles()
    env.add_agents(h0, method="random", n=9)
    assert env.get_slot_space(h1) == 0
    big = np.full(256, 0x5A, np.uint8)
    assert ns.call_mean(env, h1, h0, big, big) == 0
    assert ns.call_neighbours(env, h1, h0, 3, big, big, big) == 0
    assert (big == 0x5A).all()
    m, c = env.get_mean_action_slots(h1, h0)
    assert m.shape == (2, 0, env.get_action_space(h0)[0]) and c.shape == (2, 0)
    assert env.get_neighbours_slots(h1, 3)[0].shape == (2, 0, 3)
    idx, rel, cnt = env.get_neighbours_slots(h0, 3, h1)
    assert (idx == -1).all() and (rel == -1).all() and not cnt.any()
    ns.check_all(env, (3,))


# ---------------------------------------------------------------- refusals
def test_refusals_write_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=2)
    sc.Slots(env)
    L = env._lib
    big = np.full(1 << 16, 0x5A, np.uint8)
    p = big.ctypes.data
    before = env.get_io_stats()
    for g, o, what in ((-1, 0, b"invalid group handle"), (2, 0, b"invalid group handle"),
                       (0, -1, b"invalid group handle"), (0, 2, b"invalid group handle")):
        assert L.magent_b200_get_mean_action_slots(env.game, g, o, p, p) == -1
        assert what in L.magent_b200_last_error()
        assert L.magent_b200_get_neighbours_slots(env.game, g, o, 3, p, p, p) == -1
        assert what in L.magent_b200_last_error()
    for k in (0, 33, -2):
        assert L.magent_b200_get_neighbours_slots(env.game, 0, 1, k, p, p, p) == -1
        assert b"outside [1, 32]" in L.magent_b200_last_error()
    assert L.magent_b200_get_mean_action_slots(env.game, 0, 0, None, p) == -1
    assert b"needs a mean buffer" in L.magent_b200_last_error()
    assert L.magent_b200_get_neighbours_slots(env.game, 0, 0, 3, None, p, p) == -1
    assert b"needs an idx buffer" in L.magent_b200_last_error()
    assert (big == 0x5A).all() and env.get_io_stats() == before
    h = env.get_handles()[0]
    for k in (0, 33):
        with pytest.raises(ValueError):
            env.get_neighbours_slots(h, k)
    ns.check_all(env, (3,))


def test_a_view_too_large_for_the_key_is_refused(emu):
    """a view whose neighbour key would not fit an int is refused as get_neighbours refuses it; the mean action serves"""
    from magent_b200 import gridworld as gw
    from magent_b200.builtin.config.battle import SMALL
    import magent_b200 as magent
    cfg = gw.Config()
    cfg.set({"map_width": 12, "map_height": 12})
    t = cfg.register_agent_type("far", dict(SMALL, view_range=gw.CircleRange(140)))
    cfg.add_group(t)
    env = magent.GridWorld(cfg, _lib=emu)
    env.reset()
    h = env.get_handles()[0]
    env.add_agents(h, method="random", n=3)
    L = env._lib
    big = np.full(4096, 0x5A, np.uint8)
    assert L.magent_b200_get_neighbours(env.game, 0, 0, 3, big.ctypes.data, None, None) == -1
    assert L.magent_b200_get_neighbours_slots(env.game, 0, 0, 3, big.ctypes.data, None, None) == -1
    assert b"too large to order its cells by an int key" in L.magent_b200_last_error()
    assert (big == 0x5A).all()
    ns.check_mean(env, h, h)


def test_a_backend_without_the_kernels_refuses_the_calls(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    h = env.get_handles()[0]
    assert env.get_slot_space(h) == 20
    L = env._lib
    big = np.full(1 << 16, 0x5A, np.uint8)
    before = env.get_io_stats()
    assert L.magent_b200_get_mean_action_slots(env.game, 0, 1, big.ctypes.data, None) == -1
    assert b"no slot-ordered mean-action kernel" in L.magent_b200_last_error()
    assert L.magent_b200_get_neighbours_slots(env.game, 0, 1, 3, big.ctypes.data, None, None) == -1
    assert b"no slot-ordered neighbours kernel" in L.magent_b200_last_error()
    with pytest.raises(RuntimeError, match="no slot-ordered neighbours kernel"):
        env.get_neighbours_slots(h, 3)
    assert (big == 0x5A).all() and env.get_io_stats() == before
    sc.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernels
@pytest.mark.parametrize("kernel", ["mean_action_slots_kernel", "neighbours_slots_kernel"])
def test_kernels_have_no_stack_or_spills(kernel):
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
