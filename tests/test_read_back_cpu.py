"""The per-agent read-backs into host memory (engine.cc Engine::read_back) on the CPU.

get_reward, get_info's id/pos/alive/hp, get_action_mask, get_mean_action, get_neighbours and get_slots share one host
path: the wanted outputs are packed into one staging block, copied back, and counted in the d2h figure of
get_io_stats.  One emulation library with every per-feature loop of tests/emu serves all of them.  Each read-back must
count exactly the bytes it hands back, with its optional outputs present and absent; a group without rows must return
at once, write nothing and count nothing; and the outputs must still equal the restatements of tests/*_common.py."""
import os
import subprocess

import numpy as np
import pytest

import action_mask_common as am
import mean_action_common as ma
import neighbours_common as nc
import parity_common as pc
import slots_common as sc
from magent_b200 import gridworld as gw
from magent_b200.builtin.config.battle import SMALL


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
ALL_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_all.so")
SENTINEL = 0xA5
SLACK = 64              # sentinel bytes after every buffer: nothing may be written there


@pytest.fixture(scope="module")
def emu():
    """the host emulation with every per-feature loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in sorted(os.listdir(EMU_DIR)) if f.endswith("_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(ALL_EMU_LIB) or os.path.getmtime(ALL_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(ALL_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", ALL_EMU_LIB], check=True, capture_output=True)
    return ALL_EMU_LIB


def checker():
    return pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB


# every read-back and which of its parts may be left out (NULL); the first combination has every part
OPTIONAL = {
    "mean_action": [(1, 1), (1, 0)],
    "neighbours": [(1, 1, 1), (1, 0, 0), (1, 1, 0), (1, 0, 1)],
    "slots": [(1, 1), (1, 0), (0, 1)],
}


def read_backs(env, g, of, k):
    """every host read-back of group g: name -> (bytes of each part, call(pointers) -> return code).  The sizes are
    those of the ABI (include/magent_b200_ext.h)."""
    L, game = env._lib, env.game
    n, na, na_of = env.get_num(g), env.get_action_space(g)[0], env.get_action_space(of)[0]
    bound, S = env.get_num_bound(g), env.get_slot_space(g)

    def info(key):
        return lambda p: L.env_get_info(game, g, key, p[0])
    return {
        "reward": ([n * 4], lambda p: L.env_get_reward(game, g, p[0])),
        "id": ([n * 4], info(b"id")),
        "pos": ([n * 8], info(b"pos")),
        "alive": ([n], info(b"alive")),
        "hp": ([n * 4], info(b"hp")),
        "action_mask": ([n * na], lambda p: L.magent_b200_get_action_mask(game, g, p[0])),
        "mean_action": ([n * na_of * 4, n * 4], lambda p: L.magent_b200_get_mean_action(game, g, of, *p)),
        "neighbours": ([n * k * 4, 2 * n * k * 4, n * 4], lambda p: L.magent_b200_get_neighbours(game, g, of, k, *p)),
        "slots": ([bound * 4, env.num_arenas * S * 4], lambda p: L.magent_b200_get_slots(game, g, *p)),
    }


def read_back(env, sizes, call, wanted):
    """call one read-back into sentinel-filled host buffers; returns (return code, d2h bytes counted, buffers: None
    for a part left out)"""
    bufs = [np.full(size + SLACK, SENTINEL, np.uint8) if w else None for size, w in zip(sizes, wanted)]
    before = env.get_io_stats()["d2h"]
    rc = call([None if b is None else b.ctypes.data for b in bufs])
    return rc, env.get_io_stats()["d2h"] - before, bufs


def each_read_back(env, g, of, k):
    for name, (sizes, call) in read_backs(env, g, of, k).items():
        for wanted in OPTIONAL.get(name, [(1,) * len(sizes)]):
            yield name, sizes, call, wanted


def play(env, steps, seed):
    rs = np.random.RandomState(seed)
    for _ in range(steps):
        sc.random_step(env, rs)


def settle(env):
    """wait for the counts, so that the d2h figure of the next read-back is its own"""
    for h in env.get_handles():
        env.get_num(h)


# ---------------------------------------------------------------- what each read-back counts
@pytest.mark.parametrize("arenas", [1, 3])
def test_every_host_read_back_counts_exactly_its_bytes(emu, arenas):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=arenas)
    play(env, 3, 1)
    settle(env)
    hs = env.get_handles()
    checked = 0
    for g, of in ((0, 1), (1, 1)):
        assert env.get_num(hs[g]) > 0
        for name, sizes, call, wanted in each_read_back(env, g, of, k=5):
            rc, d2h, bufs = read_back(env, sizes, call, wanted)
            what = "%s of group %d, parts %s" % (name, g, wanted)
            assert rc == 0, what
            assert d2h == sum(s for s, w in zip(sizes, wanted) if w), "%s: %d bytes counted, want %s" % (
                what, d2h, [s for s, w in zip(sizes, wanted) if w])
            for size, b in zip(sizes, bufs):
                if b is not None:
                    assert (b[size:] == SENTINEL).all(), what + ": written past its end"
                    assert size == 0 or (b[:size] != SENTINEL).any(), what + ": nothing written"
            checked += 1
    assert checked == 2 * 15


# ---------------------------------------------------------------- a group without rows
def starving_config(size):
    """two armies; the second starves to death in its first step (hp 1, step_recover -2): a group without rows whose
    slot space is not 0"""
    cfg = gw.Config()
    cfg.set({"map_width": size, "map_height": size})
    ranges = dict(view_range=gw.CircleRange(4), attack_range=gw.CircleRange(1.5))
    small = cfg.register_agent_type("small", dict(SMALL, **ranges))
    frail = cfg.register_agent_type("frail", dict(SMALL, hp=1, step_recover=-2, **ranges))
    cfg.add_group(small)
    cfg.add_group(frail)
    return cfg


def never_placed(emu):
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    env.reset()
    env.add_agents(env.get_handles()[0], method="random", n=9)
    return env


def starved(emu):
    import magent_b200 as magent
    env = magent.GridWorld(starving_config(14), _lib=emu, _num_arenas=2)
    env.set_seed(3)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=8)
    play(env, 1, 2)
    return env


@pytest.mark.parametrize("make", [never_placed, starved])
def test_a_group_without_rows_reads_back_nothing(emu, make):
    """every row-ordered output returns at once, untouched and uncounted; slot_row is A * S words whatever the rows"""
    env = make(emu)
    hs = env.get_handles()
    settle(env)
    assert env.get_num(hs[1]) == 0 and env.get_num(hs[0]) > 0
    assert env.get_num_bound(hs[1]) == 0
    S = env.get_slot_space(hs[1])
    assert S == (8 if make is starved else 0)
    for of in (0, 1):
        for name, sizes, call, wanted in each_read_back(env, 1, of, k=4):
            rc, d2h, bufs = read_back(env, sizes, call, wanted)
            what = "%s of the empty group over %d, parts %s" % (name, of, wanted)
            assert rc == 0, what
            slot_row = bufs[1] if name == "slots" else None
            assert d2h == (env.num_arenas * S * 4 if slot_row is not None else 0), "%s: %d bytes counted" % (what, d2h)
            for b in bufs:
                if b is not None and b is not slot_row:
                    assert (b == SENTINEL).all(), what + ": written"
            if slot_row is not None:
                words = slot_row[:env.num_arenas * S * 4].view(np.int32)
                assert (words == -1).all() and (slot_row[env.num_arenas * S * 4:] == SENTINEL).all(), what


# ---------------------------------------------------------------- the values
def test_the_outputs_equal_the_restatements(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    tr = sc.Slots(env)
    play(env, 3, 5)
    am.check_masks(env)
    assert ma.check_means(env, pairs=[(0, 1)]) > 0
    assert nc.check_rows(env, 5, pairs=[(1, 0)]) > 0
    assert sc.check(tr) > 0
    # hp against the global state's hp / max_hp plane at every agent's cell
    state = env.get_global_state()
    hp = np.empty(env.get_num(env.get_handles()[0]), np.float32)
    h0 = env.get_handles()[0]
    env._info(h0, b"hp", hp)
    arena = np.repeat(np.arange(env.num_arenas), env.get_arena_nums(h0))
    pos = env.get_pos(h0)
    np.testing.assert_allclose(state[arena, pos[:, 1], pos[:, 0], 2], hp / SMALL["hp"], rtol=1e-6)


def test_reward_id_pos_alive_equal_the_reference(emu):
    def make(lib):
        return pc.make_battle(lib, 16, 20, 4)
    pc.compare_traces(pc.run_trace(make(emu), 4, 7), pc.run_trace(make(checker()), 4, 7), "emulation vs reference")
