"""The built-in scripted opponents (magent_b200_rule_actions, _get_rule_actions, _get_rule_actions_slots) on the CPU.

The test-only host emulation (tests/emu/rule_actions_emu.cc) decides every agent with the function the CUDA kernels use
(rule_phases.h rule_action).  Here it is checked against the plain numpy restatement of tests/rule_actions_common.py in
every game mode and under the fuzz configs, for both policies and every (group, target) pair, target == group included."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import action_mask_common as am
import arena_restore_common as arc
import fuzz_common as fz
import parity_common as pc
import rule_actions_common as rc
from magent_b200 import build as b

EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SRC_DIR = os.path.join(pc.REPO, "magent_b200", "csrc")
RULE_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_rule.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation with every emulated loop: the restatement reads walls and food through the global state, and
    the slot variant needs the slot loops"""
    emu_srcs = [os.path.join(EMU_DIR, f) for f in sorted(os.listdir(EMU_DIR)) if f.endswith("_emu.cc")]
    assert os.path.join(EMU_DIR, "rule_actions_emu.cc") in emu_srcs
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(RULE_EMU_LIB) or os.path.getmtime(RULE_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(RULE_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(SRC_DIR, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", RULE_EMU_LIB], check=True,
                       capture_output=True)
    return RULE_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the default emulation library, which has no rule loops"""
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    if not os.path.exists(pc.EMU_LIB) or os.path.getmtime(pc.EMU_LIB) < newest:
        subprocess.run([os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


GAMES = dict(arc.SCENARIOS, sector=lambda lib, seed, **kw: pc.make_sector(lib, 30, seed, **kw))


def read_variants(env, h, t, policy, seed):
    """the row call, checked against the slot call (through get_slots) and the in-place call (read back through the
    feature one-hot)"""
    rows = env.get_rule_actions(h, t, rc.POLICIES[policy], seed).copy()
    slots = env.get_rule_actions_slots(h, t, rc.POLICIES[policy], seed).copy()
    row_slot, slot_row = env.get_slots(h)
    np.testing.assert_array_equal(slots.reshape(-1)[row_slot], rows)
    assert (slots[slot_row < 0] == -1).all()
    env.set_rule_actions(h, t, rc.POLICIES[policy], seed)
    np.testing.assert_array_equal(am.last_actions(env, h)[env.get_alive(h)], rows[env.get_alive(h)])
    return rows


@pytest.mark.parametrize("name", sorted(GAMES))
def test_rule_actions_equal_the_restatement_in_every_game_mode(emu, name, tmp_path):
    env = GAMES[name](emu, 5)
    steps = rc.play_and_check(env, 8, 3, tmp_path, uncull_every=3)
    print(name, "agents decided by none / attack / approach / fallback:", steps.tolist())
    assert steps[rc.APPROACH] > 0, steps


@pytest.mark.parametrize("name", ["battle", "turn", "arrange", "food", "sector"])
def test_row_slot_and_in_place_variants_agree(emu, name, tmp_path):
    env = GAMES[name](emu, 2)
    rc.play_and_check(env, 4, 7, tmp_path, read=read_variants)


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


def test_rule_actions_equal_the_restatement_under_the_fuzz_configs(emu, tmp_path):
    """random configs: many groups, long and turning bodies, sector views, absorbers, empty groups"""
    total = np.zeros(4, np.int64)
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed)
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        G = len(env.get_handles())
        pairs = [(g, t, p) for g in range(G) for t in {0, g, (g + 1) % G} for p in (rc.RUSH, rc.FLEE)]
        total += rc.play_and_check(env, 5, seed, d, uncull_every=3, pairs=pairs)
    assert (total[1:] > 0).all(), total


def test_the_restatement_rejects_a_wrong_choice(emu):
    env = pc.make_battle(emu, 20, 40, 5)
    for _ in range(3):
        am.random_step(env, np.random.RandomState(1))
    state = rc.State(env)
    want, step = state.expected(0, 1, rc.RUSH, 9)
    i = int(np.flatnonzero(step == rc.APPROACH)[0])

    def bad(e, h, t, p, s):
        got = rc.read_rows(e, h, t, p, s)
        got[i] = (got[i] + 1) % env.get_action_space(h)[0]
        return got
    with pytest.raises(AssertionError):
        rc.check(state, [(0, 1, rc.RUSH)], 9, read=bad)
    rc.check(state, [(0, 1, rc.RUSH)], 9)


def test_rule_calls_leave_the_random_draws_alone(emu):
    """neither call counts as a random_legal_actions call: the next draw is the one it would have been without them"""
    def draws(rule_calls):
        env = pc.make_battle(emu, 20, 40, 5)
        h, t = env.get_handles()
        for _ in range(rule_calls):
            env.get_rule_actions(h, t, "rush", 3)
            env.set_rule_actions(h, t, "flee", 3)
        env.set_random_legal_actions(h, 4)
        return am.last_actions(env, h)
    np.testing.assert_array_equal(draws(0), draws(2))


# ---------------------------------------------------------------- the Python classes
def test_random_actor_draws_as_the_reference_does(emu):
    """the reference's RandomActor: np.random.randint(n_action, size=num, dtype=np.int32) from numpy's global state"""
    from magent.builtin.rule_model import RandomActor
    env = pc.make_battle(emu, 20, 40, 5)
    h = env.get_handles()[0]
    obs = env.get_observation(h)
    np.random.seed(123)
    got = RandomActor(env, h).infer_action(obs, env.get_agent_id(h))
    np.random.seed(123)
    want = np.random.randint(env.get_action_space(h)[0], size=len(obs[0]), dtype=np.int32)
    assert got.dtype == np.int32
    np.testing.assert_array_equal(got, want)


def test_rush_and_flee_actors_return_the_device_choice(emu):
    from magent_b200.builtin.rule_model import FleeActor, RushActor
    env = pc.make_pursuit(emu, 24, 2)
    pred, prey = env.get_handles()
    rush, flee = RushActor(env, pred, prey, seed=4), FleeActor(env, prey, pred, seed=4)
    for _ in range(3):
        a, b_ = rush.infer_action(None), flee.infer_action(env.get_observation(prey))
        np.testing.assert_array_equal(a, env.get_rule_actions(pred, prey, "rush", 4))
        np.testing.assert_array_equal(b_, env.get_rule_actions(prey, pred, "flee", 4))
        env.set_action(pred, a)
        env.set_action(prey, b_)
        env.step()
        env.clear_dead()


# ---------------------------------------------------------------- refusals
def test_bad_handles_and_policies_are_refused_and_change_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4)
    h, t = env.get_handles()
    before = env.get_rule_actions(h, t).copy()
    buf = np.full(4096, 7, dtype=np.int32)
    L = env._lib
    for g, tt, p in ((-1, 1, 0), (2, 1, 0), (99, 1, 0), (0, -1, 0), (0, 2, 0), (0, 1, -1), (0, 1, 2)):
        for rcode in (L.magent_b200_rule_actions(env.game, g, tt, p, 1),
                      L.magent_b200_get_rule_actions(env.game, g, tt, p, 1, buf.ctypes.data),
                      L.magent_b200_get_rule_actions_slots(env.game, g, tt, p, 1, buf.ctypes.data)):
            assert rcode == -1
            assert L.magent_b200_last_error()
    assert (buf == 7).all()
    for bad in (dict(target=ctypes.c_int(5)), dict(policy=3), dict(policy=-1)):
        kw = dict(target=t, policy="rush")
        kw.update(bad)
        with pytest.raises(RuntimeError):
            env.set_rule_actions(h, kw["target"], kw["policy"])
        with pytest.raises(RuntimeError):
            env.get_rule_actions(h, kw["target"], kw["policy"])
        with pytest.raises(RuntimeError):
            env.get_rule_actions_slots(h, kw["target"], kw["policy"])
    with pytest.raises(RuntimeError, match="invalid group handle"):
        env.set_rule_actions(ctypes.c_int(7), t)
    with pytest.raises(ValueError):
        env.set_rule_actions(h, t, "charge")
    np.testing.assert_array_equal(env.get_rule_actions(h, t), before)
    env.step()                                                    # nobody was marked as having acted
    assert env.get_counters()[0] == 0


def test_a_backend_without_the_rule_loops_refuses_the_calls(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    h, t = env.get_handles()
    with pytest.raises(RuntimeError, match="no rule-action kernel"):
        env.set_rule_actions(h, t)
    with pytest.raises(RuntimeError, match="no rule-action kernel"):
        env.get_rule_actions(h, t)
    with pytest.raises(RuntimeError, match="no slot-ordered rule-action kernel"):
        env.get_rule_actions_slots(h, t)
    am.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernels
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


@pytest.mark.parametrize("kernel", ["rule_actions_kernel", "rule_actions_slots_kernel"])
def test_rule_kernels_have_no_stack_or_spills(kernel):
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    m = re.search(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, open(LOG).read())
    assert m, kernel + " not in the ptxas report"
    assert tuple(int(v) for v in m.groups()[1:]) == (0, 0, 0), "%s: %s" % (kernel, m.groups()[1:])
