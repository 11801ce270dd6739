"""The legal-action mask and the legal draws computed by the CUDA kernels (action_mask_kernel,
random_legal_actions_kernel), on the GPU: against the numpy restatement of tests/action_mask_common.py in every game
mode and under fuzz configs, host pointer against device pointer, ragged batches, a whole-grid arena and battle at its
full size against a PyTorch restatement, odd output tensors, a recorded CUDA graph, and the draws themselves."""
import numpy as np
import pytest

import action_mask_common as am
import arena_restore_common as arc
import fullsize_common as fs
import fuzz_common as fz
import parity_common as pc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


def host_and_device(env, h):
    host = env.get_action_mask(h).copy()
    np.testing.assert_array_equal(env.get_action_mask_torch(h).cpu().numpy(), host)
    return host


def battle_masks_torch(env, size):
    """the mask of both armies of a battle batch (1 x 1 bodies, speed 2, attack radius 1.5, no walls inside), restated
    with torch on the device from positions alone"""
    import torch
    dev = torch.device("cuda")
    hs = env.get_handles()
    types = [am.GroupType(env, g) for g in range(2)]
    nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
    pos = [torch.as_tensor(env.get_pos(h), device=dev).long() for h in hs]
    ar = [fs.arena_index(n, dev) for n in nums]
    owner = torch.full((len(nums[0]), size, size), -1, dtype=torch.int64, device=dev)
    for g in range(2):
        owner[ar[g], pos[g][:, 1], pos[g][:, 0]] = g
    out = []
    for g in range(2):
        t = types[g]
        m = torch.zeros((pos[g].shape[0], t.n_action), dtype=torch.bool, device=dev)
        x, y = pos[g][:, 0], pos[g][:, 1]
        for k, (dx, dy) in enumerate(t.moves + t.attacks):
            tx, ty = x + dx, y + dy
            if k < t.n_move:
                inb = (tx >= 0) & (ty >= 0) & (tx + 1 < size) & (ty + 1 < size)
                o = owner[ar[g], ty.clamp(0, size - 1), tx.clamp(0, size - 1)]
                border = (tx == 0) | (ty == 0)                      # the border wall (the far sides fail the board test)
                m[:, k] = inb & ~border & ((o == -1) | ((dx == 0) & (dy == 0)))
            else:
                inb = (tx >= 0) & (ty >= 0) & (tx < size) & (ty < size)
                o = owner[ar[g], ty.clamp(0, size - 1), tx.clamp(0, size - 1)]
                m[:, k] = inb & (o == 1 - g)
        out.append(m)
    return out


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_mask_equals_the_restatement_in_every_game_mode(name, tmp_path):
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5)
    bits, ones = am.play_and_check(env, 10, 3, tmp_path, uncull_every=3, read=host_and_device)
    assert 0 < ones < bits


def test_cuda_mask_under_fuzz_configs(tmp_path):
    for seed in (2, 5, 8, 13, 14, 41, 1004, 70001, 100002):
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        am.play_and_check(fz.make_env(pc.CUDA_LIB, seed), 6, seed, d, uncull_every=3, read=host_and_device)


def test_ragged_batch_with_an_empty_group():
    env = pc.make_battle(pc.CUDA_LIB, 16, 20, 4, _num_arenas=4)
    hs = env.get_handles()
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        env.add_agents(hs[0], method="random", n=extra)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    for t in range(6):
        am.check_masks(env, what="step %d" % t, read=host_and_device)
        am.random_step(env, rs)
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=pc.CUDA_LIB, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # group 1 stays empty
    masks = am.check_masks(lone, read=host_and_device)
    assert masks[1].shape == (0, 21) and not masks[0][:, 13:].any()


def test_whole_grid_arena_and_battle_at_full_size():
    """one arena of 2 x 20000 agents (more than the CTA-per-arena step holds) and bench.py's 512 arenas of 2 x 1000,
    against the torch restatement, under uniform and under legal draws"""
    import torch
    for arenas, size, n, steps in ((1, 400, 20000, 3), (512, 200, 1000, 4)):
        env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=arenas)
        hs = env.get_handles()
        for t in range(steps):
            want = battle_masks_torch(env, size)
            for g, h in enumerate(hs):
                got = env.get_action_mask_torch(h)
                assert got.dtype == torch.bool and got.shape == want[g].shape
                assert bool((got == want[g]).all()), "%d arenas step %d group %d: %d wrong bits" % (
                    arenas, t, g, int((got != want[g]).sum()))
                assert bool(got[:, 6].all())                           # the centre move
            for h in hs:
                (env.set_random_legal_actions if t % 2 else env.set_random_actions)(h, t)
            env.step()
            env.clear_dead()
        del env


def test_unaligned_and_over_long_outputs_keep_their_guard_bytes():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    h = env.get_handles()[1]
    want = env.get_action_mask(h).copy()
    n, na = want.shape
    for lead in (1, 5, 16, 23):
        big = torch.full((lead + (n + 9) * na + 40,), 7, dtype=torch.uint8, device="cuda")
        out = big[lead:lead + (n + 9) * na].view(n + 9, na)               # longer than the group, not 16-byte aligned
        got = env.get_action_mask_torch(h, out=out)
        assert got.shape == (n, na) and got.dtype == torch.bool
        np.testing.assert_array_equal(got.cpu().numpy(), want)
        assert bool((big[:lead] == 7).all()) and bool((big[lead + n * na:] == 7).all()), "bytes outside the rows were written"
    # refusals: wrong device, dtype, width, too few rows
    for bad in (torch.zeros((n, na), dtype=torch.uint8), torch.zeros((n, na), dtype=torch.int32, device="cuda"),
                torch.zeros((n, na + 1), dtype=torch.uint8, device="cuda"),
                torch.zeros((n - 1, na), dtype=torch.uint8, device="cuda"),
                torch.zeros((n, 2 * na), dtype=torch.uint8, device="cuda")[:, :na]):
        with pytest.raises(ValueError):
            env.get_action_mask_torch(h, out=bad)
    np.testing.assert_array_equal(env.get_action_mask(h), want)


def test_mask_and_restore_inside_a_replayed_cuda_graph():
    """two steps recorded with a restore of two arenas (a device src) and the mask of both groups into fixed tensors sized by
    num_bound, replayed 20 times with refilled actions, against an un-captured twin making the same calls"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env, twin = (arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4) for _ in range(2))
    hs = env.get_handles()
    snap, tsnap = env.snapshot_arenas(), twin.snapshot_arenas()
    bound = [env.get_num_bound(h) for h in hs]
    assert bound == [env.get_num(h) for h in hs]
    na = env.get_action_space(hs[0])[0]
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)]
    masks = [[torch.zeros((n, na), dtype=torch.uint8, device="cuda") for n in bound] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    src = np.array([1, -1, 3, -1], dtype=np.int32)
    d_src = torch.from_numpy(src).cuda()

    def one(k):
        for h, a in zip(hs, acts[k]):
            L.env_set_action(env.game, env._hv(h), a.data_ptr())
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()
        env.restore_arenas(snap, d_src)
        for h, m in zip(hs, masks[k]):
            env.get_action_mask_torch(h, out=m)

    rs = np.random.RandomState(7)

    def draw():
        a = [[rs.randint(0, na, size=n).astype(np.int32) for n in bound] for _ in range(2)]
        for k in range(2):
            for g in range(2):
                acts[k][g].copy_(torch.from_numpy(a[k][g]))
        return a

    def twin_pair(a):
        out = []
        for k in range(2):
            for h, x in zip(twin.get_handles(), a[k]):
                twin.set_action(h, np.ascontiguousarray(x[:twin.get_num(h)]))
            twin.step()
            twin.clear_dead()
            twin.restore_arenas(tsnap, src)
            out.append([twin.get_action_mask(h).copy() for h in twin.get_handles()])
        return out

    a = draw()
    one(0)
    one(1)
    want = twin_pair(a)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    for _ in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for g in range(2):
                n = len(want[k][g])
                np.testing.assert_array_equal(masks[k][g][:n].cpu().numpy().astype(bool), want[k][g])
    nums = twin.get_arena_nums(twin.get_handles()[0])
    assert nums[0] == 8 and nums[2] == 8 and nums[1] + nums[3] < 16, "arenas 0 and 2 restart every step, 1 and 3 fight on"


def test_legal_draws_on_the_device():
    """every action set is legal under the mask taken just before; the restated draw reproduces the kernel exactly; the
    same seed, call and step give the same actions on a twin; dead agents get action 0"""
    env, twin = (pc.make_battle(pc.CUDA_LIB, 24, 120, 6, _num_arenas=3) for _ in range(2))
    hs = env.get_handles()
    calls = 0
    for t in range(10):
        for g, h in enumerate(hs):
            mask = env.get_action_mask(h).copy()
            env.set_random_legal_actions(h, 40 + t)
            twin.set_random_legal_actions(twin.get_handles()[g], 40 + t)
            calls += 1
            acts = am.last_actions(env, h)
            np.testing.assert_array_equal(acts, am.restate_draws(mask, 40 + t, calls, t))
            np.testing.assert_array_equal(acts, am.last_actions(twin, twin.get_handles()[g]))
            rows = mask.any(axis=1)
            assert mask[np.flatnonzero(rows), acts[rows]].all() and (acts[~rows] == 0).all()
        env.step()
        twin.step()
        if t % 3 != 2:
            env.clear_dead()
            twin.clear_dead()
    assert env.get_counters()[3] > 0


def test_replayed_graph_draws_fresh_legal_actions():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 30, 200, 3, _num_arenas=2)
    hs = env.get_handles()
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")

    def pair():
        for k in range(2):
            for h in hs:
                env.set_random_legal_actions(h, 5)
            env.step_device_done(done.data_ptr() + 4 * k)
            env.clear_dead()

    pair()
    gid = env.capture_graph(pair)
    seen = []
    for _ in range(3):
        env.launch_graph(gid, 1)
        seen.append(am.last_actions(env, hs[0])[:150].copy())
    assert not np.array_equal(seen[0], seen[1]) and not np.array_equal(seen[1], seen[2])


def test_legal_draws_are_uniform_and_a_legal_soak_holds_the_invariants():
    """battle at full size driven by legal draws only: uniformity of the draw over the agents that share the most common
    legal set (chi-square, 0.1 % point), then 40 steps with the state invariants after every step and kills in a good share of the
    arenas"""
    import torch
    A, size, n = 512, 200, 1000
    env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=A)
    hs = env.get_handles()
    mask = env.get_action_mask_torch(hs[0])
    env.set_random_legal_actions(hs[0], 9)
    acts = torch.as_tensor(am.last_actions(env, hs[0]), device="cuda").long()
    free = mask[:, :13].all(dim=1) & ~mask[:, 13:].any(dim=1)              # every move legal, nothing to attack
    assert int(free.sum()) >= 100000
    counts = torch.bincount(acts[free], minlength=21).double().cpu().numpy()
    assert counts[13:].sum() == 0
    exp = counts.sum() / 13.0
    chi2 = ((counts[:13] - exp) ** 2 / exp).sum()
    assert chi2 < 32.9, (chi2, counts)                                     # 12 degrees of freedom
    env.set_random_legal_actions(hs[1], 9)
    env.step()
    env.clear_dead()
    nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
    start = [x.copy() for x in nums]
    prev = None
    for t in range(40):
        pos = [env.get_pos(h).copy() for h in hs]
        ids = [env.get_agent_id(h).copy() for h in hs]
        fs.check_state(pos, ids, nums, size, size, prev=prev, speed=2)
        for h in hs:
            env.set_random_legal_actions(h, 1000 + t)
        env.step()
        env.clear_dead()
        prev = (ids, pos, nums)
        nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
    lost = (start[0] - nums[0]) + (start[1] - nums[1])
    # 2 x 1000 agents placed at random on 200 x 200 cells meet rarely: about half the arenas see a kill in 40 steps
    assert (lost > 0).mean() > 0.25, "arenas without a kill: %d" % int((lost == 0).sum())
