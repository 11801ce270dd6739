"""The nearest visible neighbours computed by the CUDA kernel (neighbours_kernel), on the GPU: against the numpy
restatement of tests/neighbours_common.py in every game mode and under fuzz configs, host pointers against device
pointers, with and without count (the early exit), a whole-grid arena and battle at its full size against a PyTorch
restatement, odd output tensors, mixed pointers, and a recorded CUDA graph."""
import ctypes

import numpy as np
import pytest

import arena_restore_common as arc
import fullsize_common as fs
import fuzz_common as fz
import global_state_common as gs
import neighbours_common as nb
import parity_common as pc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


def host_and_device(env, h, of, k):
    """the host-pointer rows, after checking them bit for bit against the device-pointer rows, and against the device
    rows without count (the kernel then stops at the k-th neighbour) and without rel and count"""
    import torch
    idx, rel, c = (x.copy() for x in env.get_neighbours(h, k, of))
    di, dr, dc = env.get_neighbours_torch(h, k, of)
    np.testing.assert_array_equal(di.cpu().numpy(), idx)
    np.testing.assert_array_equal(dr.cpu().numpy(), rel)
    np.testing.assert_array_equal(dc.cpu().numpy(), c)
    bound = env.get_num_bound(h)
    only_i = torch.full((bound, k), -7, dtype=torch.int32, device="cuda")
    only_r = torch.full((bound, k, 2), -7, dtype=torch.int32, device="cuda")
    oi, orel, oc = env.get_neighbours_torch(h, k, of, out=(only_i, only_r, None))
    assert oc is None
    np.testing.assert_array_equal(oi.cpu().numpy(), idx)
    np.testing.assert_array_equal(orel.cpu().numpy(), rel)
    only_i.fill_(-7)
    oi, orel, oc = env.get_neighbours_torch(h, k, of, out=(only_i, None, None))
    assert orel is None and oc is None
    np.testing.assert_array_equal(oi.cpu().numpy(), idx)
    return idx, rel, c


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_neighbours_equal_the_restatement_in_every_game_mode(name, tmp_path):
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5)
    assert nb.play_and_check(env, 6, 3, (1, 3, 32), tmp_path, uncull_every=3, read=host_and_device) > 0


def test_cuda_neighbours_under_fuzz_configs(tmp_path):
    for seed in (2, 5, 8, 13, 14, 41, 1004, 70001, 70005, 100002):
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        nb.play_and_check(fz.make_env(pc.CUDA_LIB, seed), 4, seed, (3, 32), d, uncull_every=3, read=host_and_device)


def test_ragged_batch_with_an_empty_group():
    env = pc.make_battle(pc.CUDA_LIB, 16, 20, 4, _num_arenas=4)
    hs = env.get_handles()
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        env.add_agents(hs[0], method="random", n=extra)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    import action_mask_common as am
    for t in range(5):
        nb.check_rows(env, 5, what="step %d" % t, read=host_and_device)
        am.random_step(env, rs)
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=pc.CUDA_LIB, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # group 1 stays empty
    nb.check_rows(lone, 4, read=host_and_device)
    i, r, c = lone.get_neighbours_torch(lone.get_handles()[1], 4, lone.get_handles()[0])
    assert tuple(i.shape) == (0, 4) and tuple(r.shape) == (0, 4, 2) and tuple(c.shape) == (0,)


def battle_neighbours_torch(env, size, k):
    """(idx, rel, count) of every (group, of) pair of a battle batch (1 x 1 bodies, no walls inside), restated with
    torch on the device: the view's in-range offsets walked in key order over an owner grid, with a running hit rank per
    observer, scattered where the rank is below k"""
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
        for g in range(2):
            mask, x1, y1, w, l = gs.view_geometry(env, g)
            assert (w, l) == (1, 1)
            vh, vw = mask.shape
            vy, vx = np.nonzero(mask)
            dx, dy = x1 + vx, y1 + vy
            order = np.argsort((dx * dx + dy * dy) * (vh * vw) + vy * vw + vx, kind="stable")
            n = pos[g].shape[0]
            idx = torch.full((n, k), -1, dtype=torch.int32, device=dev)
            rel = torch.full((n, k, 2), -1, dtype=torch.int32, device=dev)
            rank = torch.zeros((n,), dtype=torch.int64, device=dev)
            me = torch.arange(n, device=dev)
            x, y = pos[g][:, 0], pos[g][:, 1]
            for q in order:
                tx, ty = x + int(dx[q]), y + int(dy[q])
                inb = (tx >= 0) & (ty >= 0) & (tx < size) & (ty < size)
                o = owner[ar[g], ty.clamp(0, size - 1), tx.clamp(0, size - 1)]
                hit = inb & (o >= 0)
                if of == g:
                    hit &= o != me
                sel = torch.nonzero(hit & (rank < k)).squeeze(1)
                idx[sel, rank[sel]] = o[sel].int()
                rel[sel, rank[sel], 0] = int(vy[q])
                rel[sel, rank[sel], 1] = int(vx[q])
                rank += hit.long()
            out[(g, of)] = (idx, rel, rank.int())
    return out


def test_whole_grid_arena_and_battle_at_full_size():
    """one arena of 2 x 20000 agents (more than the CTA-per-arena step holds) and bench.py's 512 arenas of 2 x 1000,
    against the torch restatement, after a few steps"""
    import torch
    for arenas, size, n in ((1, 400, 20000), (512, 200, 1000)):
        env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=arenas)
        hs = env.get_handles()
        listed = 0
        for t in range(3):
            for k in (3, 32):
                want = battle_neighbours_torch(env, size, k)
                for (g, of), (wi, wr, wc) in want.items():
                    gi, gr, gc = env.get_neighbours_torch(hs[g], k, hs[of])
                    assert gi.dtype == torch.int32 and gi.shape == wi.shape and gr.shape == wr.shape
                    for got, w, what in ((gi, wi, "idx"), (gr, wr, "rel"), (gc, wc, "count")):
                        bad = (got != w).reshape(got.shape[0], -1).any(dim=1)
                        assert not bool(bad.any()), "%d arenas step %d k=%d %d over %d: %d wrong %s rows" % (
                            arenas, t, k, g, of, int(bad.sum()), what)
                    early = torch.empty((env.get_num_bound(hs[g]), k), dtype=torch.int32, device="cuda")
                    assert torch.equal(env.get_neighbours_torch(hs[g], k, hs[of], out=(early, None, None))[0], wi)
                    listed += int((wi >= 0).sum())
            for h in hs:
                env.set_random_actions(h, t)
            env.step()
            env.clear_dead()
        assert listed > 0
        del env


def test_unaligned_and_over_long_outputs_and_refusals():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    hs = env.get_handles()
    h, of = hs[1], hs[0]
    k = 5
    want = [x.copy() for x in env.get_neighbours(h, k, of)]
    n = len(want[2])
    for lead in (1, 3):
        bi = torch.full((lead + (n + 9) * k + 40,), -3, dtype=torch.int32, device="cuda")
        br = torch.full((lead + (n + 9) * k * 2 + 40,), -5, dtype=torch.int32, device="cuda")
        bc = torch.full((lead + n + 9 + 40,), -9, dtype=torch.int32, device="cuda")
        out = (bi[lead:lead + (n + 9) * k].view(n + 9, k), br[lead:lead + (n + 9) * k * 2].view(n + 9, k, 2),
               bc[lead:lead + n + 9])
        got = env.get_neighbours_torch(h, k, of, out=out)
        assert tuple(got[0].shape) == (n, k) and tuple(got[1].shape) == (n, k, 2) and tuple(got[2].shape) == (n,)
        for x, y in zip(got, want):
            np.testing.assert_array_equal(x.cpu().numpy(), y)
        assert bool((bi[:lead] == -3).all()) and bool((bi[lead + n * k:] == -3).all()), "idx outside the rows"
        assert bool((br[:lead] == -5).all()) and bool((br[lead + n * k * 2:] == -5).all()), "rel outside the rows"
        assert bool((bc[:lead] == -9).all()) and bool((bc[lead + n:] == -9).all()), "counts outside the rows"
    gi = torch.zeros((n, k), dtype=torch.int32, device="cuda")
    gr = torch.zeros((n, k, 2), dtype=torch.int32, device="cuda")
    gc = torch.zeros((n,), dtype=torch.int32, device="cuda")
    bad_outs = [
        (torch.zeros((n, k), dtype=torch.int32), gr, gc),                               # host tensor
        (torch.zeros((n, k), dtype=torch.int64, device="cuda"), gr, gc),                # dtype
        (gi, torch.zeros((n, k, 2), dtype=torch.float32, device="cuda"), gc),
        (gi, gr, torch.zeros((n,), dtype=torch.int64, device="cuda")),
        (torch.zeros((n, k + 1), dtype=torch.int32, device="cuda"), gr, gc),            # width
        (gi, torch.zeros((n, k, 3), dtype=torch.int32, device="cuda"), gc),
        (torch.zeros((n - 1, k), dtype=torch.int32, device="cuda"), gr, gc),            # too few rows
        (gi, torch.zeros((n - 1, k, 2), dtype=torch.int32, device="cuda"), gc),
        (gi, gr, torch.zeros((n - 1,), dtype=torch.int32, device="cuda")),
        (torch.zeros((n, 2 * k), dtype=torch.int32, device="cuda")[:, :k], gr, gc),     # not contiguous
        (gi, gr, torch.zeros((n, 2), dtype=torch.int32, device="cuda")),
        (None, gr, gc),                                                                 # idx is needed
        (gi, gr),                                                                       # not a triple
        gi,
    ]
    for bad in bad_outs:
        with pytest.raises(ValueError):
            env.get_neighbours_torch(h, k, of, out=bad)
    for bad_k in (0, 33):
        with pytest.raises(ValueError):
            env.get_neighbours_torch(h, bad_k, of)
    # host and device buffers mixed: refused, nothing written
    L = env._lib
    host_i = np.full((n, k), -9, dtype=np.int32)
    host_c = np.full(n, -9, dtype=np.int32)
    dp = lambda t: ctypes.c_void_p(t.data_ptr())                                         # noqa: E731
    for args in ((dp(gi), dp(gr), host_c.ctypes.data), (host_i.ctypes.data, dp(gr), None),
                 (host_i.ctypes.data, None, dp(gc))):
        assert L.magent_b200_get_neighbours(env.game, 1, 0, k, *args) == -1
        assert b"must all be host memory or all CUDA device memory" in L.magent_b200_last_error()
    # bad handles and k through the device path
    for g, o, kk in ((2, 0, k), (0, 5, k), (-1, 1, k), (1, 0, 0), (1, 0, 33)):
        assert L.magent_b200_get_neighbours(env.game, g, o, kk, dp(gi), dp(gr), dp(gc)) == -1
    torch.cuda.synchronize()
    assert (host_i == -9).all() and (host_c == -9).all()
    assert not bool(gi.any()) and not bool(gr.any()) and not bool(gc.any())
    # rel and count may be NULL with a device idx
    assert L.magent_b200_get_neighbours(env.game, 1, 0, k, dp(gi), None, None) == 0
    np.testing.assert_array_equal(gi.cpu().numpy(), want[0])


def test_neighbours_and_restore_inside_a_replayed_cuda_graph():
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
    K = 4
    pairs = [(0, 0), (0, 1), (1, 0), (1, 1)]
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)]
    outs = [[(torch.zeros((bound[g], K), dtype=torch.int32, device="cuda"),
              torch.zeros((bound[g], K, 2), dtype=torch.int32, device="cuda"),
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
            env.get_neighbours_torch(hs[g], K, hs[o], out=out)

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
            out.append([tuple(x.copy() for x in twin.get_neighbours(ths[g], K, ths[o])) for g, o in pairs])
        return out

    a = draw()
    one(0)
    one(1)
    twin_pair(a)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    listed = 0
    for _ in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for p, w in enumerate(want[k]):
                n = len(w[2])
                for got, x in zip(outs[k][p], w):
                    np.testing.assert_array_equal(got[:n].cpu().numpy(), x)
                listed += int((w[0] >= 0).sum())
    assert listed > 0
