"""The built-in scripted opponents computed by the CUDA kernels (rule_actions_kernel, rule_actions_slots_kernel), on the
GPU: against the numpy restatement of tests/rule_actions_common.py in every game mode and under the fuzz configs, the
row, slot and in-place variants through host and device pointers, after clear_dead, a device-src restore_arenas and
add_agents, inside a recorded CUDA graph, a rush-driven game against the oracle, and a fixed-seed sanity battle."""
import os

import numpy as np
import pytest

import action_mask_common as am
import arena_restore_common as arc
import fuzz_common as fz
import parity_common as pc
import rule_actions_common as rc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

GAMES = dict(arc.SCENARIOS, sector=lambda lib, seed, **kw: pc.make_sector(lib, 30, seed, **kw))


def every_variant(env, h, t, policy, seed):
    """the host row call, checked against the torch row call, the host and torch slot calls and the in-place call"""
    p = rc.POLICIES[policy]
    rows = env.get_rule_actions(h, t, p, seed).copy()
    np.testing.assert_array_equal(env.get_rule_actions_torch(h, t, p, seed).cpu().numpy(), rows)
    slots = env.get_rule_actions_slots(h, t, p, seed).copy()
    np.testing.assert_array_equal(env.get_rule_actions_slots_torch(h, t, p, seed).cpu().numpy(), slots)
    row_slot, slot_row = env.get_slots(h)
    np.testing.assert_array_equal(slots.reshape(-1)[row_slot], rows)
    assert (slots[slot_row < 0] == -1).all()
    env.set_rule_actions(h, t, p, seed)
    alive = env.get_alive(h)
    np.testing.assert_array_equal(am.last_actions(env, h)[alive], rows[alive])
    return rows


@pytest.mark.parametrize("name", sorted(GAMES))
def test_cuda_rule_actions_equal_the_restatement_in_every_game_mode(name, tmp_path):
    env = GAMES[name](pc.CUDA_LIB, 5)
    steps = rc.play_and_check(env, 8, 3, tmp_path, uncull_every=3, read=every_variant)
    assert steps[rc.APPROACH] > 0, steps


def test_cuda_rule_actions_under_the_fuzz_configs(tmp_path):
    total = np.zeros(4, np.int64)
    for seed in [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]:
        env = fz.make_env(pc.CUDA_LIB, seed)
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        G = len(env.get_handles())
        pairs = [(g, t, p) for g in range(G) for t in {0, g, (g + 1) % G} for p in (rc.RUSH, rc.FLEE)]
        total += rc.play_and_check(env, 5, seed, d, uncull_every=3, pairs=pairs)
    assert (total[1:] > 0).all(), total


def test_after_clear_dead_device_restore_and_add_agents():
    env = pc.make_battle(pc.CUDA_LIB, 20, 40, 6, _num_arenas=3)
    hs = env.get_handles()
    pairs = rc.all_pairs(env)
    snap = env.snapshot_arenas()
    rs = np.random.RandomState(4)
    steps = 0
    for t in range(9):
        am.random_step(env, rs)                                   # with clear_dead
        steps += 1
        what = "step %d" % t
        if t % 3 == 1:                                            # before the in-place call sets this step's actions
            env.restore_arenas(snap, arc.as_src([2, -1, 0], "device"))
            what += " after restore"
        if t % 3 == 2:
            env.select_arena(t % 3)
            env.add_agents(hs[t % 2], method="random", n=5)
            env.select_arena(-1)
            what += " after add_agents"
        rc.check(rc.State(env, call=1, steps=steps), pairs, t, every_variant, what)


def test_a_recorded_two_step_graph_decides_afresh_every_step():
    """set_rule_actions for both armies and get_rule_actions_torch into fixed tensors, two steps with clear_dead in one
    graph; every replay's decisions equal the restatement on an un-captured twin's state before each step"""
    import torch
    env, twin = (pc.make_battle(pc.CUDA_LIB, 24, 60, 8, _num_arenas=2) for _ in range(2))
    hs, ths = env.get_handles(), twin.get_handles()
    bound = env.get_num_bound(hs[0])
    got = [torch.full((bound,), -7, dtype=torch.int32, device="cuda") for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")

    def one(k):
        env.get_rule_actions_torch(hs[0], hs[1], "rush", 11, out=got[k])
        env.set_rule_actions(hs[0], hs[1], "rush", 11)
        env.set_rule_actions(hs[1], hs[0], "flee", 11)
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()

    def twin_step(steps):
        state = rc.State(twin, call=1, steps=steps)
        want, _ = state.expected(0, 1, rc.RUSH, 11)
        twin.set_rule_actions(ths[0], ths[1], "rush", 11)
        twin.set_rule_actions(ths[1], ths[0], "flee", 11)
        twin.step()
        twin.clear_dead()
        return want

    one(0)
    one(1)
    twin_step(0)
    twin_step(1)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    steps, seen = 2, []
    for _ in range(5):
        env.launch_graph(gid, 1)
        want = [twin_step(steps), twin_step(steps + 1)]
        steps += 2
        torch.cuda.synchronize()
        for k in range(2):
            np.testing.assert_array_equal(got[k][:len(want[k])].cpu().numpy(), want[k])
        seen.append(want[0])
    for h, th in zip(hs, ths):
        np.testing.assert_array_equal(env.get_pos(h), twin.get_pos(th))
    assert any(not np.array_equal(seen[0][:20], s[:20]) for s in seen[1:])


def checker():
    return next((p for p in (pc.REF_LIB, pc.PORT_LIB) if os.path.exists(p)), None)


def test_a_rush_driven_game_stays_bit_exact_with_the_oracle():
    ref_lib = checker()
    if ref_lib is None:
        pytest.skip("no oracle library built")
    env, ref = pc.make_battle(pc.CUDA_LIB, 30, 120, 2), pc.make_battle(ref_lib, 30, 120, 2)
    hs, rhs = env.get_handles(), ref.get_handles()
    for t in range(25):
        acts = [env.get_rule_actions(hs[0], hs[1], "rush", t).copy(), env.get_rule_actions(hs[1], hs[0], "flee", t).copy()]
        for h, rh, a in zip(hs, rhs, acts):
            env.set_action(h, a)
            ref.set_action(rh, a)
        env.step()
        ref.step()
        for h, rh in zip(hs, rhs):
            np.testing.assert_array_equal(env.get_pos(h), ref.get_pos(rh), "step %d" % t)
            np.testing.assert_array_equal(env.get_alive(h), ref.get_alive(rh), "step %d" % t)
            np.testing.assert_array_equal(env.get_reward(h).view(np.uint32), ref.get_reward(rh).view(np.uint32))
            np.testing.assert_array_equal(env.get_observation(h)[0], ref.get_observation(rh)[0], "step %d" % t)
        env.clear_dead()
        ref.clear_dead()


def sanity_battle(lib):
    """rush (group 0) against random legal actions (group 1) on eight small arenas, 30 steps: each side's losses"""
    env = pc.make_battle(lib, 20, 40, 1, _num_arenas=8)
    hs = env.get_handles()
    lost = [0, 0]
    for t in range(30):
        env.set_rule_actions(hs[0], hs[1], "rush", t)
        env.set_random_legal_actions(hs[1], t)
        env.step()
        for g, h in enumerate(hs):
            lost[g] += int((~env.get_alive(h)).sum())
        env.clear_dead()
    return lost


# the outcome of sanity_battle, deterministic given the seeds: rush wipes out all 8 x 40 random players and loses nobody
SANITY_LOST = [0, 320]


def test_rush_beats_random_legal_actions():
    lost = sanity_battle(pc.CUDA_LIB)
    assert lost[1] > 2 * lost[0], lost
    assert lost == SANITY_LOST, lost
