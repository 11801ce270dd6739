"""The mean neighbour action computed by the CUDA kernel (mean_action_kernel), on the GPU: against the numpy restatement
of tests/mean_action_common.py in every game mode and under fuzz configs, host pointers against device pointers, ragged
batches, a whole-grid arena and battle at its full size against a PyTorch restatement, odd output tensors, mixed
pointers, and a recorded CUDA graph."""
import ctypes

import numpy as np
import pytest

import arena_restore_common as arc
import fullsize_common as fs
import fuzz_common as fz
import global_state_common as gs
import mean_action_common as ma
import parity_common as pc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


def host_and_device(env, h, of):
    """the host-pointer rows, after checking them bit for bit against the device-pointer rows"""
    m, c = (x.copy() for x in env.get_mean_action(h, of))
    dm, dc = env.get_mean_action_torch(h, of)
    np.testing.assert_array_equal(ma._bits(dm.cpu().numpy()), ma._bits(m))
    np.testing.assert_array_equal(dc.cpu().numpy(), c)
    return m, c


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_mean_action_equals_the_restatement_in_every_game_mode(name, tmp_path):
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5)
    assert ma.play_and_check(env, 8, 3, tmp_path, uncull_every=3, read=host_and_device) > 0


def test_cuda_mean_action_under_fuzz_configs(tmp_path):
    for seed in (2, 5, 8, 13, 14, 41, 1004, 70001, 70005, 100002):
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        ma.play_and_check(fz.make_env(pc.CUDA_LIB, seed), 5, seed, d, uncull_every=3, read=host_and_device)


def test_ragged_batch_with_an_empty_group():
    env = pc.make_battle(pc.CUDA_LIB, 16, 20, 4, _num_arenas=4)
    hs = env.get_handles()
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        env.add_agents(hs[0], method="random", n=extra)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    import action_mask_common as am
    for t in range(6):
        ma.check_means(env, what="step %d" % t, read=host_and_device)
        am.random_step(env, rs)
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=pc.CUDA_LIB, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # group 1 stays empty
    ma.check_means(lone, read=host_and_device)
    m, c = lone.get_mean_action_torch(lone.get_handles()[1], lone.get_handles()[0])
    assert tuple(m.shape) == (0, 21) and tuple(c.shape) == (0,)


def battle_means_torch(env, size, acts):
    """(mean, count) of every (group, of) pair of a battle batch (1 x 1 bodies, no walls inside), restated with torch
    on the device: the owner grid gathered at the view's in-range offsets, then a bincount.  acts: per group the int64
    CUDA tensor of the actions the agents hold."""
    import torch
    dev = torch.device("cuda")
    hs = env.get_handles()
    nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
    pos = [torch.as_tensor(env.get_pos(h), device=dev).long() for h in hs]
    ar = [fs.arena_index(n, dev) for n in nums]
    A = len(nums[0])
    out = {}
    for of in range(2):
        owner = torch.full((A, size, size), -1, dtype=torch.int64, device=dev)
        owner[ar[of], pos[of][:, 1], pos[of][:, 0]] = torch.arange(pos[of].shape[0], device=dev)
        na = env.get_action_space(hs[of])[0]
        for g in range(2):
            mask, x1, y1, w, l = gs.view_geometry(env, g)
            vy, vx = np.nonzero(mask)
            n = pos[g].shape[0]
            bins = torch.zeros((n, na + 1), dtype=torch.int32, device=dev)
            count = torch.zeros((n,), dtype=torch.int32, device=dev)
            me = torch.arange(n, device=dev)
            x, y = pos[g][:, 0], pos[g][:, 1]
            for dx, dy in zip(w // 2 + x1 + vx, l // 2 + y1 + vy):
                tx, ty = x + int(dx), y + int(dy)
                inb = (tx >= 0) & (ty >= 0) & (tx < size) & (ty < size)
                o = owner[ar[g], ty.clamp(0, size - 1), tx.clamp(0, size - 1)]
                hit = inb & (o >= 0)
                if of == g:
                    hit &= o != me
                count += hit.int()
                k = acts[of][o.clamp(min=0)]
                k = torch.where(hit & (k >= 0) & (k < na), k, torch.full_like(k, na))
                bins.scatter_add_(1, k.unsqueeze(1), hit.int().unsqueeze(1))
            num = bins[:, :na].float()
            den = count.float().unsqueeze(1).expand_as(num).contiguous()
            mean = torch.where(den > 0, num / den.clamp(min=1.0), torch.zeros_like(num))
            out[(g, of)] = (mean, count)
    return out


def test_whole_grid_arena_and_battle_at_full_size():
    """one arena of 2 x 20000 agents (more than the CTA-per-arena step holds) and bench.py's 512 arenas of 2 x 1000,
    against the torch restatement, right after set_action (the actions are known on the device) with some ids out of
    range"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    for arenas, size, n, steps in ((1, 400, 20000, 3), (512, 200, 1000, 3)):
        env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=arenas)
        hs = env.get_handles()
        gen = torch.Generator(device="cuda")
        gen.manual_seed(7)
        counted = 0
        for t in range(steps):
            acts = []
            for h in hs:
                a = torch.randint(-1, 22, (env.get_num(h),), device="cuda", generator=gen, dtype=torch.int32)
                L.env_set_action(env.game, env._hv(h), ctypes.c_void_p(a.data_ptr()))
                acts.append(a.long())
            want = battle_means_torch(env, size, acts)
            for (g, of), (wm, wc) in want.items():
                got_m, got_c = env.get_mean_action_torch(hs[g], hs[of])
                assert got_m.dtype == torch.float32 and got_m.shape == wm.shape and got_c.dtype == torch.int32
                assert bool((got_c == wc).all()), "%d arenas step %d %d over %d: %d wrong counts" % (
                    arenas, t, g, of, int((got_c != wc).sum()))
                bad = got_m.view(torch.int32) != wm.view(torch.int32)
                assert not bool(bad.any()), "%d arenas step %d %d over %d: %d wrong means" % (
                    arenas, t, g, of, int(bad.sum()))
                counted += int(wc.sum())
            env.step()
            env.clear_dead()
        assert counted > 0
        del env


def test_unaligned_and_over_long_outputs_and_refusals():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    hs = env.get_handles()
    h, of = hs[1], hs[0]
    want_m, want_c = (x.copy() for x in env.get_mean_action(h, of))
    n, na = want_m.shape
    for lead in (1, 3):
        big = torch.full((lead + (n + 9) * na + 40,), 7.5, dtype=torch.float32, device="cuda")
        cbig = torch.full((lead + n + 9 + 40,), -3, dtype=torch.int32, device="cuda")
        out = (big[lead:lead + (n + 9) * na].view(n + 9, na), cbig[lead:lead + n + 9])
        m, c = env.get_mean_action_torch(h, of, out=out)
        assert tuple(m.shape) == (n, na) and tuple(c.shape) == (n,)
        np.testing.assert_array_equal(ma._bits(m.cpu().numpy()), ma._bits(want_m))
        np.testing.assert_array_equal(c.cpu().numpy(), want_c)
        assert bool((big[:lead] == 7.5).all()) and bool((big[lead + n * na:] == 7.5).all()), "floats outside the rows"
        assert bool((cbig[:lead] == -3).all()) and bool((cbig[lead + n:] == -3).all()), "counts outside the rows"
    good_m = torch.zeros((n, na), dtype=torch.float32, device="cuda")
    good_c = torch.zeros((n,), dtype=torch.int32, device="cuda")
    bad_outs = [
        (torch.zeros((n, na), dtype=torch.float32), good_c),                       # host tensor
        (torch.zeros((n, na), dtype=torch.float64, device="cuda"), good_c),        # dtype
        (good_m, torch.zeros((n,), dtype=torch.int64, device="cuda")),
        (torch.zeros((n, na + 1), dtype=torch.float32, device="cuda"), good_c),    # width
        (torch.zeros((n - 1, na), dtype=torch.float32, device="cuda"), good_c),    # too few rows
        (good_m, torch.zeros((n - 1,), dtype=torch.int32, device="cuda")),
        (torch.zeros((n, 2 * na), dtype=torch.float32, device="cuda")[:, :na], good_c),   # not contiguous
        (good_m, torch.zeros((n, 2), dtype=torch.int32, device="cuda")),
        good_m,                                                                     # not a pair
    ]
    for bad in bad_outs:
        with pytest.raises(ValueError):
            env.get_mean_action_torch(h, of, out=bad)
    # one host and one device buffer: refused, nothing written
    host_c = np.full(n, -9, dtype=np.int32)
    rc = env._lib.magent_b200_get_mean_action(env.game, 1, 0, ctypes.c_void_p(good_m.data_ptr()), host_c.ctypes.data)
    assert rc == -1 and b"must both be host memory or both CUDA device memory" in env._lib.magent_b200_last_error()
    host_m = np.zeros((n, na), dtype=np.float32)
    rc = env._lib.magent_b200_get_mean_action(env.game, 1, 0, host_m.ctypes.data, ctypes.c_void_p(good_c.data_ptr()))
    assert rc == -1
    torch.cuda.synchronize()
    assert (host_c == -9).all() and not host_m.any() and not bool(good_m.any()) and not bool(good_c.any())
    # bad handles through the device path
    for g, o in ((2, 0), (0, 5), (-1, 1)):
        assert env._lib.magent_b200_get_mean_action(env.game, g, o, ctypes.c_void_p(good_m.data_ptr()),
                                                    ctypes.c_void_p(good_c.data_ptr())) == -1
    # count may be NULL with a device mean
    assert env._lib.magent_b200_get_mean_action(env.game, 1, 0, ctypes.c_void_p(good_m.data_ptr()), None) == 0
    np.testing.assert_array_equal(ma._bits(good_m.cpu().numpy()), ma._bits(want_m))


def test_mean_action_and_restore_inside_a_replayed_cuda_graph():
    """two steps recorded with a restore of two arenas (a device src) and the rows of every (group, of) pair into fixed
    tensors sized by num_bound, replayed 20 times with refilled actions, against an un-captured twin making the same
    calls"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env, twin = (arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4) for _ in range(2))
    hs = env.get_handles()
    snap, tsnap = env.snapshot_arenas(), twin.snapshot_arenas()
    bound = [env.get_num_bound(h) for h in hs]
    assert bound == [env.get_num(h) for h in hs]
    na = env.get_action_space(hs[0])[0]
    pairs = [(0, 0), (0, 1), (1, 0), (1, 1)]
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)]
    outs = [[(torch.zeros((bound[g], na), dtype=torch.float32, device="cuda"),
              torch.zeros((bound[g],), dtype=torch.int32, device="cuda")) for g, _o in pairs] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    src = np.array([1, -1, 3, -1], dtype=np.int32)
    d_src = torch.from_numpy(src).cuda()

    def one(k):
        for h, a in zip(hs, acts[k]):
            L.env_set_action(env.game, env._hv(h), a.data_ptr())
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()
        env.restore_arenas(snap, d_src)
        for (g, o), out in zip(pairs, outs[k]):
            env.get_mean_action_torch(hs[g], hs[o], out=out)

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
            out.append([tuple(x.copy() for x in twin.get_mean_action(ths[g], ths[o])) for g, o in pairs])
        return out

    a = draw()
    one(0)
    one(1)
    twin_pair(a)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    counted = 0
    for _ in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for p, (wm, wc) in enumerate(want[k]):
                n = len(wc)
                m, c = outs[k][p]
                np.testing.assert_array_equal(c[:n].cpu().numpy(), wc)
                np.testing.assert_array_equal(ma._bits(m[:n].cpu().numpy()), ma._bits(wm))
                counted += int(wc.sum())
    assert counted > 0
