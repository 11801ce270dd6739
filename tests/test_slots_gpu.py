"""The stable agent slots computed by the CUDA kernels (slots_kernel, restore_slots_kernel), on the GPU: against the
restatement of tests/slots_common.py in every game mode, under the fuzz configs and across device-src restores, host
pointers against device pointers, battle at its full size, a recorded CUDA graph with restores, and the INTEGRATION.md
recipe run literally against a twin driven row by row."""
import ctypes

import numpy as np
import pytest

import arena_restore_common as arc
import fullsize_common as fs
import fuzz_common as fz
import parity_common as pc
import slots_common as sc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


def host_and_device(env, h):
    """the host-pointer maps, after checking them bit for bit against the device-pointer maps, each buffer alone, and
    a row_slot longer than num_bound (only num_bound entries are written)"""
    import torch
    row_slot, slot_row = sc.read_host(env, h)
    bound = env.get_num_bound(h)
    dr, dm = env.get_slots_torch(h)
    assert tuple(dr.shape) == (bound,) and tuple(dm.shape) == slot_row.shape
    n = len(row_slot)
    np.testing.assert_array_equal(dr[:n].cpu().numpy(), row_slot)
    assert bool((dr[n:] == -1).all())
    np.testing.assert_array_equal(dm.cpu().numpy(), slot_row)
    long_rows = torch.full((bound + 7,), -5, dtype=torch.int32, device="cuda")
    got_r, got_m = env.get_slots_torch(h, out=(long_rows, None))
    assert got_m is None
    np.testing.assert_array_equal(got_r[:bound].cpu().numpy(), dr.cpu().numpy())
    assert bool((long_rows[bound:] == -5).all())
    only_m = torch.full(slot_row.shape, -5, dtype=torch.int32, device="cuda")
    got_r, got_m = env.get_slots_torch(h, out=(None, only_m))
    assert got_r is None
    np.testing.assert_array_equal(only_m.cpu().numpy(), slot_row)
    return row_slot, slot_row


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_slots_equal_the_restatement_in_every_game_mode(name):
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5, _num_arenas=3)
    tr = sc.Slots(env)
    n = sc.play_and_check(tr, 5, 3, read=host_and_device)
    sc.add_somewhere(tr, 1, seed=6)
    pool = tr.snapshot()
    n += sc.play_and_check(tr, 2, 4, read=host_and_device)
    tr.restore(pool, [2, -1, 1], src_kind="device")
    n += sc.play_and_check(tr, 2, 5, read=host_and_device)
    assert n > 0


def test_cuda_slots_under_fuzz_configs():
    for seed in (2, 5, 6, 8, 13, 14, 41, 1004, 70001, 70005, 100002):
        tr = sc.Slots(fz.make_env(pc.CUDA_LIB, seed, _num_arenas=4))
        sc.play_irregular(tr, 6, seed, read=host_and_device)


def test_cuda_slots_across_device_restores():
    env = arc.make_duel(pc.CUDA_LIB, 3, n=6, _num_arenas=4)
    tr = sc.Slots(env)
    pool = tr.snapshot()
    rs = np.random.RandomState(2)
    for t in range(30):
        sc.random_step(env, rs)
        if t == 1:
            sc.add_somewhere(tr, 2, seed=t)
            late = tr.snapshot()
        if t in (2, 5):
            tr.restore(pool, [-1, 2, -1, 0], src_kind="device")
        if t == 3:
            tr.restore(late, [2, 2, -1, -1], keep_rng=True, src_kind="device")
        if t >= 6:
            tr.restore(pool, None)
        sc.check(tr, "step %d" % t, read=host_and_device)
    tr.free(late)
    sc.check(tr, "after free_snapshot", read=host_and_device)


def test_mixed_pointers_and_bad_outputs_are_refused():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    hs = env.get_handles()
    h = hs[1]
    want = sc.read_host(env, h)
    bound, S = env.get_num_bound(h), env.get_slot_space(h)
    dr = torch.full((bound,), -9, dtype=torch.int32, device="cuda")
    dm = torch.full((3, S), -9, dtype=torch.int32, device="cuda")
    hr = np.full(bound, -9, dtype=np.int32)
    hm = np.full((3, S), -9, dtype=np.int32)
    L = env._lib
    dp = lambda t: ctypes.c_void_p(t.data_ptr())                                         # noqa: E731
    for args in ((dp(dr), hm.ctypes.data), (hr.ctypes.data, dp(dm))):
        assert L.magent_b200_get_slots(env.game, 1, *args) == -1
        assert b"must both be host memory or both CUDA device memory" in L.magent_b200_last_error()
    for g in (-1, 2):
        assert L.magent_b200_get_slots(env.game, g, dp(dr), dp(dm)) == -1
    assert L.magent_b200_get_slots(env.game, 1, None, None) == -1
    torch.cuda.synchronize()
    assert (hr == -9).all() and (hm == -9).all()
    assert bool((dr == -9).all()) and bool((dm == -9).all())
    bad_outs = [
        (torch.zeros((bound,), dtype=torch.int32), dm),                                   # host tensor
        (torch.zeros((bound,), dtype=torch.int64, device="cuda"), dm),                    # dtype
        (dr, torch.zeros((3, S), dtype=torch.float32, device="cuda")),
        (torch.zeros((bound - 1,), dtype=torch.int32, device="cuda"), dm),                # too few rows
        (dr, torch.zeros((3, S + 1), dtype=torch.int32, device="cuda")),                  # not (A, S)
        (dr, torch.zeros((3, 2 * S), dtype=torch.int32, device="cuda")[:, :S]),           # not contiguous
        (None, None),
        dr,
    ]
    for bad in bad_outs:
        with pytest.raises(ValueError):
            env.get_slots_torch(h, out=bad)
    got_r, got_m = env.get_slots_torch(h, out=(dr, dm))
    np.testing.assert_array_equal(got_r.cpu().numpy(), want[0])
    np.testing.assert_array_equal(got_m.cpu().numpy(), want[1])


def check_device_invariants(env, h, row_slot, slot_row, ids, what):
    """slot_row inverts row_slot, the tail is -1, rows sit in their arena's block, every occupied slot is a live row,
    and inside every arena the ids increase with the slots"""
    import torch
    n = ids.shape[0]
    S = slot_row.shape[1]
    arena = fs.arena_index(env.get_arena_nums(h).astype(np.int64), row_slot.device)
    assert bool((row_slot[n:] == -1).all()), what + ": tail"
    rs = row_slot[:n].long()
    assert bool((rs >= 0).all()) and bool((rs // S == arena).all()), what + ": arena blocks"
    assert torch.equal(slot_row.view(-1)[rs], torch.arange(n, device=rs.device, dtype=torch.int32)), what + ": inverse"
    assert int((slot_row >= 0).sum()) == n, what + ": vacant slots"
    order = torch.argsort(arena.long() * (1 << 32) + ids.long())
    a_s, s_s = arena[order], (rs % S)[order]
    same = a_s[1:] == a_s[:-1]
    assert bool((s_s[1:] > s_s[:-1])[same].all()), what + ": ids do not increase with the slots"


def test_battle_at_full_size_with_device_restores():
    """bench.py's 512 arenas of 2 x 1000: 30 device-resident steps with random legal actions and clear_dead, a tenth of
    the arenas restored from a device src every 10 steps; the invariants against the ids read back"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=512)
    hs = env.get_handles()
    A = 512
    pool = env.snapshot_arenas()
    assert [env.get_slot_space(h) for h in hs] == [1000, 1000]
    rs = np.random.RandomState(3)
    done = torch.zeros((1,), dtype=torch.int32, device="cuda")
    for t in range(30):
        for g, h in enumerate(hs):
            env.set_random_legal_actions(h, 100 * t + g)
        env.step_device_done(done.data_ptr())
        env.clear_dead()
        if t % 10 == 9:
            src = np.full(A, -1, dtype=np.int32)
            pick = rs.choice(A, size=A // 10, replace=False)
            src[pick] = rs.randint(0, A, size=len(pick))
            env.restore_arenas(pool, torch.from_numpy(src).cuda())
        outs = [env.get_slots_torch(h) for h in hs]
        for g, h in enumerate(hs):
            ids = torch.as_tensor(env.get_agent_id(h), device="cuda")
            check_device_invariants(env, h, outs[g][0], outs[g][1], ids, "step %d group %d" % (t, g))
    assert env.get_num(hs[0]) < A * 1000 and [env.get_slot_space(h) for h in hs] == [1000, 1000]


def test_slots_and_restore_inside_a_replayed_cuda_graph():
    """two steps recorded with a restore of two arenas (a device src) and both groups' maps into fixed tensors, the rows
    sized by num_bound and one longer, replayed 20 times with refilled actions, against an un-captured twin making the
    same calls with host buffers"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env, twin = (arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4) for _ in range(2))
    hs = env.get_handles()
    snap, tsnap = env.snapshot_arenas(), twin.snapshot_arenas()
    bound = [env.get_num_bound(h) for h in hs]
    S = [env.get_slot_space(h) for h in hs]
    na = env.get_action_space(hs[0])[0]
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)]
    outs = [[(torch.zeros((bound[g] + 5 * g,), dtype=torch.int32, device="cuda"),
              torch.zeros((4, S[g]), dtype=torch.int32, device="cuda")) for g in range(2)] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    src = np.array([1, -1, 3, -1], dtype=np.int32)
    d_src = torch.from_numpy(src).cuda()

    def one(k):
        for h, a in zip(hs, acts[k]):
            L.env_set_action(env.game, env._hv(h), a.data_ptr())
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()
        env.restore_arenas(snap, d_src)
        for g in range(2):
            env.get_slots_torch(hs[g], out=outs[k][g])

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
            ths = twin.get_handles()
            for h, x in zip(ths, a[k]):
                twin.set_action(h, np.ascontiguousarray(x[:twin.get_num(h)]))
            twin.step()
            twin.clear_dead()
            twin.restore_arenas(tsnap, src)
            out.append([sc.read_host(twin, ths[g]) for g in range(2)])
        return out

    a = draw()
    one(0)
    one(1)
    twin_pair(a)
    for k in range(2):
        for g in range(2):
            outs[k][g][0].fill_(-3)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    compared = 0
    for _ in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for g, (wr, wm) in enumerate(want[k]):
                got_r, got_m = outs[k][g]
                n = len(wr)
                np.testing.assert_array_equal(got_r[:n].cpu().numpy(), wr)
                assert bool((got_r[n:bound[g]] == -1).all()), "the tail up to num_bound"
                assert bool((got_r[bound[g]:] == -3).all()), "written beyond num_bound"
                np.testing.assert_array_equal(got_m.cpu().numpy(), wm)
                compared += n
    assert compared > 0


def test_the_integration_recipe_against_a_twin_driven_row_by_row():
    """INTEGRATION.md §4 literally: observations scattered into [A, S] with slot_row, random actions drawn per slot and
    gathered back into a num_bound-long row buffer with row_slot, passed to env_set_action as a device pointer.  The twin
    gets the same actions row by row as a host array of exactly get_num rows: both must play the same game, so the
    device set_action reads no row past the device-side count even when num_bound is larger."""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    # one-hit duels on a small map: agents die every step, so num_bound (held at the placement counts by the
    # snapshot) soon exceeds the count
    env, twin = (arc.make_duel(pc.CUDA_LIB, 5, n=8, _num_arenas=3) for _ in range(2))
    hs, ths = env.get_handles(), twin.get_handles()
    env.snapshot_arenas()
    twin.snapshot_arenas()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    longer = 0
    for t in range(10):
        for g, (h, th) in enumerate(zip(hs, ths)):
            row_slot, slot_row = env.get_slots_torch(h)
            A, S = slot_row.shape
            n = env.get_num(h)
            if n:
                obs = env.get_observation_torch(h)[0]
                obs_s = obs[slot_row.clamp(min=0).view(-1)] * (slot_row >= 0).view(-1, 1, 1, 1)
                occ = (slot_row >= 0).view(-1)
                assert torch.equal(obs_s[occ], obs[slot_row.view(-1)[occ].long()]), "step %d group %d" % (t, g)
                assert not bool(obs_s[~occ].any()), "step %d group %d" % (t, g)
            act_s = torch.randint(0, env.get_action_space(h)[0], (A, S), dtype=torch.int32, device="cuda",
                                  generator=gen)
            act_rows = act_s.view(-1)[row_slot.clamp(min=0)]
            assert act_rows.shape[0] == env.get_num_bound(h)
            longer += act_rows.shape[0] > n
            L.env_set_action(env.game, env._hv(h), act_rows.data_ptr())
            twin.set_action(th, np.ascontiguousarray(act_rows[:n].cpu().numpy()))
        env.step()
        twin.step()
        for h, th in zip(hs, ths):
            np.testing.assert_array_equal(env.get_reward(h), twin.get_reward(th), err_msg="step %d" % t)
            np.testing.assert_array_equal(env.get_alive(h), twin.get_alive(th), err_msg="step %d" % t)
        env.clear_dead()
        twin.clear_dead()
        for h, th in zip(hs, ths):
            np.testing.assert_array_equal(env.get_pos(h), twin.get_pos(th), err_msg="step %d" % t)
            np.testing.assert_array_equal(env.get_agent_id(h), twin.get_agent_id(th), err_msg="step %d" % t)
    assert longer > 0, "num_bound never exceeded the count: the row buffer's tail was not exercised"
