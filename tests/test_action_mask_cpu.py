"""The legal-action mask and the legal draws (magent_b200_get_action_mask, magent_b200_random_legal_actions) on the CPU.

The test-only host emulation (tests/emu/) decides every (agent, action) with the function the CUDA kernels use
(mask_phases.h action_legal).  Here it is checked against the outcome of the compiled reference (or the oracle's C
restatement where that is absent) playing single actions, and against the plain numpy restatement of
tests/action_mask_common.py in every game mode and under the fuzz configs."""
import os
import re
import subprocess

import numpy as np
import pytest

import action_mask_common as am
import arena_restore_common as arc
import fuzz_common as fz
import parity_common as pc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
MASK_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_mask.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation plus its global-state loop (the restatement reads walls and food from it) and its mask loops"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "global_state_emu.cc", "action_mask_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(MASK_EMU_LIB) or os.path.getmtime(MASK_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(MASK_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", MASK_EMU_LIB], check=True, capture_output=True)
    return MASK_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the default emulation library, which has no mask loops"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    if not os.path.exists(pc.EMU_LIB) or os.path.getmtime(pc.EMU_LIB) < newest:
        subprocess.run([os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


def checker():
    return pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB


# ---------------------------------------------------------------- the definition, pinned to the reference's outcomes
def centre_action(t):
    return t.moves.index((0, 0))


def replay(make, lib, history):
    env = make(lib)
    for acts in history:
        for h, a in zip(env.get_handles(), acts):
            env.set_action(h, a)
        env.step()
        env.clear_dead()
    return env


def outcome(env, types, g, i, k, tmpdir):
    """everyone plays the centre move, agent i of group g plays k: what the engine library `env` then shows"""
    hs = env.get_handles()
    for gg, h in enumerate(hs):
        act = np.full(env.get_num(h), centre_action(types[gg]), dtype=np.int32)
        if gg == g:
            act[i] = k
        env.set_action(h, act)
    env.step()
    out = dict(pos=[env.get_pos(h).copy() for h in hs], alive=[env.get_alive(h).copy() for h in hs],
               views=[env.get_observation(h)[0].copy() for h in hs], reward=[env.get_reward(h).copy() for h in hs])
    if tmpdir is not None:
        env.set_render_dir(tmpdir)
        out["dirs"] = am.frame_headings(env, tmpdir)
    return out


OUTCOME_GAMES = {
    "battle": lambda lib: pc.make_battle(lib, 12, 14, 3),
    "pursuit": lambda lib: pc.make_pursuit(lib, 24, 2),
    "gather": lambda lib: pc.make_gather(lib, 14, 1, 6, 24),
    "forest": lambda lib: pc.make_builtin(lib, "forest", 14, 3, 14, 7),
    "double_attack": lambda lib: pc.make_builtin(lib, "double_attack", 14, 3, 14, 7),
    "multi4": lambda lib: pc.make_multi4(lib, 14, 8, 7),
    "arrange": lambda lib: pc.make_arrange(lib, 14, 12, 10, 16),
}


@pytest.mark.parametrize("name", sorted(OUTCOME_GAMES))
def test_mask_equals_what_the_reference_does_with_single_actions(emu, name):
    """Replay a small game to step t in a fresh reference instance, let one agent play action k while everyone else
    stands still, and read what happened: the agent's position changed (or k is the centre move), it vanished into an
    absorber, or somebody's view (an hp, a death) or somebody else's reward (a weaponless hit that a rule pays for) changed
    against the replay in which it stands still too.  That
    verdict must be the emulation's bit for every agent and action.  (food_mode and turn_mode outcomes are not all visible
    through the reference's getters -- a bite of food, a heading; those modes are pinned through the restatement.)"""
    make, ref_lib = OUTCOME_GAMES[name], checker()
    eng = make(emu)
    types = [am.GroupType(eng, g) for g in range(len(eng.get_handles()))]
    tracker = am.AbsorbTracker(eng)
    rs = np.random.RandomState(11)
    history, checked = [], 0
    for t in range(5):
        tracker.update()
        if t in (0, 2, 4):
            masks = [eng.get_action_mask(h).copy() for h in eng.get_handles()]
            base = outcome(replay(make, ref_lib, history), types, 0, 0, centre_action(types[0]), None)
            for g, h in enumerate(eng.get_handles()):
                ab = tracker.absorbed(g, h)
                for i in range(eng.get_num(h)):
                    for k in range(types[g].n_action):
                        got = outcome(replay(make, ref_lib, history), types, g, i, k, None)
                        if k < types[g].n_move:
                            if ab is not None and ab[i]:
                                want = False                     # its move is skipped: nothing to observe
                                assert (got["pos"][g][i] == base["pos"][g][i]).all()
                            else:
                                want = (k == centre_action(types[g]) or (got["pos"][g][i] != base["pos"][g][i]).any()
                                        or not got["alive"][g][i])
                        else:
                            got["reward"][g][i] = base["reward"][g][i]       # its own: attack_penalty either way
                            want = any((a != b).any() for key in ("alive", "views", "reward")
                                       for a, b in zip(got[key], base[key]))
                        assert bool(masks[g][i, k]) == bool(want), "%s step %d group %d agent %d action %d: mask %d" % (
                            name, t, g, i, k, masks[g][i, k])
                        checked += 1
        acts = [rs.randint(0, eng.get_action_space(h)[0], size=eng.get_num(h)).astype(np.int32) for h in eng.get_handles()]
        history.append(acts)
        for h, a in zip(eng.get_handles(), acts):
            eng.set_action(h, a)
        eng.step()
        eng.clear_dead()
    assert checked > 300
    print("outcomes read from", os.path.relpath(ref_lib, pc.REPO), "-", checked, "single actions")


# ---------------------------------------------------------------- emulation against the restatement
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_mask_equals_the_restatement_in_every_game_mode(emu, name, tmp_path):
    env = arc.SCENARIOS[name](emu, 5)
    bits, ones = am.play_and_check(env, 10, 3, tmp_path, uncull_every=3)
    assert 0 < ones < bits
    for h in env.get_handles():                                   # a live agent that has not absorbed can stand still
        m, alive = env.get_action_mask(h), env.get_alive(h)
        if not am.GroupType(env, env._hv(h)).can_absorb:
            assert m[alive].any(axis=1).all()


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


def test_mask_equals_the_restatement_under_the_fuzz_configs(emu, tmp_path):
    """random configs: many groups, large-map bands, sector ranges, long bodies, absorbers, empty groups, fills"""
    wide = turn = absorb = empty = 0
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed)
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        am.play_and_check(env, 8, seed, d, uncull_every=4)
        types = [am.GroupType(env, g) for g in range(len(env.get_handles()))]
        wide += any(t.n_action > 32 for t in types)
        turn += types[0].turn_mode
        absorb += any(t.can_absorb for t in types)
        empty += any(env.get_num(h) == 0 for h in env.get_handles())
    assert wide and turn and absorb and empty, (wide, turn, absorb, empty)


def test_chaotic_caller_and_arena_batch_with_selected_adds(emu):
    """a batch of arenas, agents added to single arenas between steps, groups that skip set_action, steps without
    clear_dead"""
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=3)
    rs = np.random.RandomState(9)
    hs = env.get_handles()
    for t in range(12):
        am.check_masks(env, what="step %d" % t)
        if t % 4 == 1:
            env.select_arena(t % 3)
            env.add_agents(hs[t % 2], method="random", n=5)
            env.select_arena(-1)
            am.check_masks(env, what="step %d after add_agents" % t)
        for h in hs:
            if rs.rand() < 0.7:
                env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
        env.step()
        if rs.rand() < 0.6:
            env.clear_dead()


def test_the_restatement_rejects_corrupted_masks(emu):
    env = pc.make_pursuit(emu, 16, 2)
    hs = env.get_handles()
    want = am.expected_masks(env)
    types = [am.GroupType(env, g) for g in range(len(hs))]
    # a move into a wall that the mask allows
    g = 1
    blocked = np.argwhere(~want[g][:, :types[g].n_move])
    assert len(blocked)
    bad = want[g].copy()
    bad[tuple(blocked[0])] = True
    with pytest.raises(AssertionError):
        am.check_masks(env, read=lambda e, h, bad=bad, g=g: bad if e._hv(h) == g else e.get_action_mask(h))
    # a flipped attack bit
    bad = want[0].copy()
    bad[0, types[0].attack_base] ^= True
    with pytest.raises(AssertionError):
        am.check_masks(env, read=lambda e, h, bad=bad: bad if e._hv(h) == 0 else e.get_action_mask(h))
    # a live agent's row zeroed
    bad = want[0].copy()
    bad[1] = False
    with pytest.raises(AssertionError):
        am.check_masks(env, read=lambda e, h, bad=bad: bad if e._hv(h) == 0 else e.get_action_mask(h))
    am.check_masks(env)


# ---------------------------------------------------------------- legal draws
@pytest.mark.parametrize("name", ["battle", "gather", "turn", "arrange", "food"])
def test_legal_draws_are_legal_and_follow_the_documented_function(emu, name):
    env = arc.SCENARIOS[name](emu, 2)
    hs = env.get_handles()
    calls = 0
    for t in range(8):
        masks = [env.get_action_mask(h).copy() for h in hs]
        for g, h in enumerate(hs):
            env.set_random_legal_actions(h, 77 + t)
            calls += 1
            acts = am.last_actions(env, h)
            np.testing.assert_array_equal(acts, am.restate_draws(masks[g], 77 + t, calls, t))
            rows = masks[g].any(axis=1)
            assert masks[g][np.flatnonzero(rows), acts[rows]].all()
            assert (acts[~rows] == 0).all()
        env.step()
        if t % 3 != 2:                                            # some steps keep their dead: they must not be acted
            env.clear_dead()
    counters = env.get_counters()
    assert counters[0] > 0


def test_legal_draws_are_uniform_over_a_fixed_legal_set():
    """the draw function over 2 * 10^5 ordinals and a 7-action legal set: chi-square against uniform (6 degrees of
    freedom; 22.5 is the 0.1 % point)"""
    mask = np.zeros((200000, 21), dtype=bool)
    legal = [0, 3, 4, 9, 13, 17, 20]
    mask[:, legal] = True
    acts = am.restate_draws(mask, 5, 1, 3)
    counts = np.array([(acts == k).sum() for k in legal], dtype=np.float64)
    assert counts.sum() == len(mask)
    chi2 = ((counts - len(mask) / 7.0) ** 2 / (len(mask) / 7.0)).sum()
    assert chi2 < 22.5, (chi2, counts)


def test_legal_draws_make_a_denser_fight_than_uniform_draws(emu):
    def hits(legal):
        env = pc.make_battle(emu, 30, 120, 3)
        for t in range(25):
            for h in env.get_handles():
                (env.set_random_legal_actions if legal else env.set_random_actions)(h, t)
            env.step()
            env.clear_dead()
        return env.get_counters()[2]
    assert hits(True) > 1.5 * hits(False)


# ---------------------------------------------------------------- refusals
def test_bad_group_handles_are_refused_and_change_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4)
    h = env.get_handles()[0]
    before = env.get_action_mask(h).copy()
    buf = np.zeros(4096, dtype=np.uint8)
    for bad in (-1, 2, 99):
        assert env._lib.magent_b200_get_action_mask(env.game, bad, buf.ctypes.data) == -1
        assert b"invalid group handle" in env._lib.magent_b200_last_error()
        assert env._lib.magent_b200_random_legal_actions(env.game, bad, 1) == -1
        assert b"invalid group handle" in env._lib.magent_b200_last_error()
    assert not buf.any()
    np.testing.assert_array_equal(env.get_action_mask(h), before)
    env.step()                                                    # nobody was marked as having acted
    assert env.get_counters()[0] == 0


def test_a_backend_without_the_mask_loops_refuses_both_calls(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    h = env.get_handles()[0]
    with pytest.raises(RuntimeError, match="no action-mask kernel"):
        env.get_action_mask(h)
    with pytest.raises(RuntimeError, match="no legal-action sampler"):
        env.set_random_legal_actions(h, 1)
    am.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernels
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


@pytest.mark.parametrize("kernel", ["action_mask_kernel", "random_legal_actions_kernel"])
def test_mask_kernels_have_no_stack_or_spills(kernel):
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    m = re.search(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, open(LOG).read())
    assert m, kernel + " not in the ptxas report"
    assert tuple(int(v) for v in m.groups()[1:]) == (0, 0, 0), "%s: %s" % (kernel, m.groups()[1:])
