"""The slot-ordered mean action and neighbours (magent_b200_get_mean_action_slots, _get_neighbours_slots) on the GPU.

Every output must equal the row-ordered call gathered through get_slots, with every listed neighbour's row translated
to its flat slot (tests/nbr_slots_common.py): in every game mode and the fuzz configs, through host and device pointers,
after device-src and NULL-src restores, at battle512's full size, on a one-arena large map and inside a replayed CUDA
graph.  The calls must not perturb the engine: the slot-loop twin of tests/slot_loop_common.py still holds with them
interleaved."""
import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import nbr_slots_common as ns
import parity_common as pc
import slot_loop_common as lc
import slots_common as sc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def host_and_device(env, ks=(1, 3, 32), what=""):
    """every (group, of) pair: the host outputs against the restatement, the device outputs (full, and without rel and
    count) bit for bit equal to them"""
    listed = 0
    for h, o in ns.pairs(env):
        w = "%s group %d of %d" % (what, env._hv(h), env._hv(o))
        hm, hc = (x.copy() for x in env.get_mean_action_slots(h, o))
        ns.check_mean(env, h, o, (hm, hc), w)
        dm, dc = env.get_mean_action_slots_torch(h, o)
        assert np.array_equal(dm.cpu().numpy().view(np.uint32), hm.view(np.uint32)), w + ": device mean"
        assert np.array_equal(dc.cpu().numpy(), hc), w + ": device mean count"
        for k in ks:
            hi, hr, hn = (x.copy() for x in env.get_neighbours_slots(h, k, o))
            listed += ns.check_neighbours(env, h, o, k, (hi, hr, hn), "%s k %d" % (w, k))
            di, dr, dn = env.get_neighbours_slots_torch(h, k, o)
            assert np.array_equal(di.cpu().numpy(), hi) and np.array_equal(dr.cpu().numpy(), hr), w + ": device idx/rel"
            assert np.array_equal(dn.cpu().numpy(), hn), w + ": device count"
            import torch
            only = torch.empty_like(di)
            env.get_neighbours_slots_torch(h, k, o, out=(only, None, None))
            assert np.array_equal(only.cpu().numpy(), hi), w + ": device idx without rel and count"
    return listed


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_every_game_mode_through_host_and_device_pointers(name):
    """steps, culls, a device-src restore and a NULL-src restore"""
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5, _num_arenas=3)
    tr = sc.Slots(env)
    pool = env.snapshot_arenas()
    rs = np.random.RandomState(2)
    listed = 0
    for t in range(5):
        sc.random_step(env, rs, cull=False)
        listed += host_and_device(env, what="%s step %d before clear_dead" % (name, t))
        env.clear_dead()
        if t == 1:
            env.restore_arenas(pool, arc.as_src([2, -1, 1], "device"))
        elif t == 3:
            env.restore_arenas(pool)
        listed += host_and_device(env, what="%s step %d" % (name, t))
    sc.add_somewhere(tr, 1, seed=6)
    listed += host_and_device(env, what="%s after adding into arena 1" % name)
    assert listed > 0


def test_fuzz_configs():
    for seed in (2, 6, 13, 41, 1004, 70001, 70005, 100002):
        env = fz.make_env(pc.CUDA_LIB, seed, _num_arenas=4)
        rs = np.random.RandomState(seed)
        ks = (1, 3, 32) if len(env.get_handles()) <= 4 else (3, 32)
        for t in range(3):
            sc.random_step(env, rs, cull=rs.rand() < 0.65)
            host_and_device(env, ks, "seed %d step %d" % (seed, t))


def test_the_calls_do_not_perturb_the_slot_loop_twin():
    """the slot-driven twin of the slot-ordered step loop, with both calls (host and device, every pair) interleaved on
    its slot engine only: the two engines stay bit for bit alike"""
    import torch

    def set_device(env, h, act):
        env.set_action_slots(h, torch.from_numpy(act).cuda())

    for name in ("battle", "turn", "multi4"):
        tw = lc.Twin(lambda lib: arc.SCENARIOS[name](lib, 5, _num_arenas=3), pc.CUDA_LIB, set_device)
        rs = np.random.RandomState(9)
        for t in range(5):
            tw.act(rs)
            for h, o in ns.pairs(tw.s):
                tw.s.get_mean_action_slots_torch(h, o)
                tw.s.get_neighbours_slots(h, 4, o)
            tw.both(lambda e: e.step())
            for h, o in ns.pairs(tw.s):
                tw.s.get_mean_action_slots(h, o)
                tw.s.get_neighbours_slots_torch(h, 32, o)
            tw.check("%s step %d" % (name, t))
            tw.both(lambda e: e.clear_dead())
            tw.check("%s step %d after clear_dead" % (name, t))


def test_mixed_pointers_and_bad_outputs_are_refused():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    h, o = env.get_handles()
    S, na, k = env.get_slot_space(h), env.get_action_space(o)[0], 4
    L = env._lib
    dm = torch.full((3, S, na), -9.0, device="cuda")
    hc = np.full((3, S), 7, np.int32)
    hm = np.full((3, S, na), -9.0, np.float32)
    dc = torch.full((3, S), 7, dtype=torch.int32, device="cuda")
    for p in ((dm.data_ptr(), hc.ctypes.data), (hm.ctypes.data, dc.data_ptr())):
        assert L.magent_b200_get_mean_action_slots(env.game, 0, 1, *p) == -1
        assert b"must both be host memory or both CUDA device memory" in L.magent_b200_last_error()
    di = torch.full((3, S, k), 7, dtype=torch.int32, device="cuda")
    hi = np.full((3, S, k), 7, np.int32)
    hr = np.full((3, S, k, 2), 7, np.int32)
    for p in ((di.data_ptr(), hr.ctypes.data, None), (hi.ctypes.data, None, dc.data_ptr())):
        assert L.magent_b200_get_neighbours_slots(env.game, 0, 1, k, *p) == -1
        assert b"must all be host memory or all CUDA device memory" in L.magent_b200_last_error()
    torch.cuda.synchronize()
    assert (hm == -9).all() and (hc == 7).all() and bool((dm == -9).all()) and bool((dc == 7).all())
    assert (hi == 7).all() and (hr == 7).all() and bool((di == 7).all())
    for bad in ((dm, None, None), dm, (dm[:, :-1].contiguous(), dc), (dm.double(), dc), (dm, dc.long()),
                (dm.cpu(), dc), (torch.zeros((3, S, na + 1), device="cuda"), dc)):
        with pytest.raises(ValueError):
            env.get_mean_action_slots_torch(h, o, out=bad)
    for bad in ((di, None), (di[:, :, :-1].contiguous(), None, None), (di.long(), None, None),
                (di, torch.zeros((3, S, k, 3), dtype=torch.int32, device="cuda"), None),
                (di, None, dc[:, ::2])):
        with pytest.raises(ValueError):
            env.get_neighbours_slots_torch(h, k, o, out=bad)
    m, c = env.get_mean_action_slots_torch(h, o, out=(dm, None))
    assert c is None
    ns.check_mean(env, h, o, (m.cpu().numpy(), None))
    i, r, n = env.get_neighbours_slots_torch(h, k, o, out=(di, None, dc))
    assert r is None
    ns.check_neighbours(env, h, o, k, (i.cpu().numpy(), None, n.cpu().numpy()))


# ---------------------------------------------------------------- full size
def gathered_on_device(env, h, o, k):
    """the restatement with torch on the device: (mean, count, idx, rel, ncount) in slot order"""
    import torch
    _rs, slot_row = env.get_slots_torch(h)
    row_slot_of, _sr = env.get_slots_torch(o)
    occ = slot_row >= 0
    rows = slot_row.clamp(min=0).long()
    m, c = env.get_mean_action_torch(h, o)
    i, r, n = env.get_neighbours_torch(h, k, o)
    zero = torch.zeros((), dtype=torch.int32, device="cuda")
    mean = torch.where(occ[..., None], m.view(torch.int32)[rows], zero)
    count = torch.where(occ, c[rows], zero)
    ir = i[rows]
    idx = torch.where(occ[..., None] & (ir >= 0), row_slot_of[ir.clamp(min=0).long()], zero - 1)
    rel = torch.where(occ[..., None, None], r[rows], zero - 1)
    ncount = torch.where(occ, n[rows], zero)
    return mean, count, idx, rel, ncount


def check_on_device(env, h, o, k, what):
    import torch
    mean, count = env.get_mean_action_slots_torch(h, o)
    idx, rel, ncount = env.get_neighbours_slots_torch(h, k, o)
    want = gathered_on_device(env, h, o, k)
    for name, got, w in zip(("mean", "count", "idx", "rel", "ncount"),
                            (mean.view(torch.int32), count, idx, rel, ncount), want):
        assert torch.equal(got, w), "%s: %s differs" % (what, name)
    return int((idx >= 0).sum())


def test_battle512_at_full_size():
    """bench.py's 512 arenas of 2 x 1000: group 0 over its own group and the enemy, k = 32, with culls and NULL-src
    restores of the finished arenas"""
    env = pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=512)
    pool = env.snapshot_arenas()
    h, e = env.get_handles()
    listed = 0
    for t in range(6):
        for g in env.get_handles():
            env.set_random_legal_actions(g, t)
        env.step()
        if t % 2:
            env.clear_dead()
            env.restore_arenas(pool)
        for o in (h, e):
            listed += check_on_device(env, h, o, 32, "step %d of %d" % (t, env._hv(o)))
    assert listed > 0


def test_one_arena_large_map():
    """one arena, many CTAs over its slots; a few culls open vacant slots"""
    env = pc.make_battle(pc.CUDA_LIB, 300, 9000, 7)
    h, e = env.get_handles()
    assert env.get_slot_space(h) >= 9000
    for t in range(4):
        for g in env.get_handles():
            env.set_random_legal_actions(g, t)
        env.step()
        env.clear_dead()
        for o in (h, e):
            check_on_device(env, h, o, 32, "step %d of %d" % (t, env._hv(o)))
            check_on_device(env, e, o, 3, "step %d enemy of %d" % (t, env._hv(o)))
    ns.check_all(env, (3,), "host pointers")


# ---------------------------------------------------------------- CUDA graphs
def test_inside_a_replayed_cuda_graph():
    """two steps of the slot-native loop recorded with device buffers (NULL-src restores), whose last recorded calls
    are the two slot calls, replayed 10 times with refilled actions: after each replay, what the calls wrote equals the
    restatement taken at that state"""
    import torch
    env = arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4)
    hs = env.get_handles()
    snap = env.snapshot_arenas()
    A, k = 4, 5
    S = [env.get_slot_space(h) for h in hs]
    na = [env.get_action_space(h)[0] for h in hs]
    acts = [[torch.zeros((A, S[g]), dtype=torch.int32, device="cuda") for g in range(2)] for _ in range(2)]
    means = [env.get_mean_action_slots_torch(hs[g], hs[1 - g]) for g in range(2)]
    nbrs = [env.get_neighbours_slots_torch(hs[g], k, hs[g]) for g in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")

    def one(s):
        for g, h in enumerate(hs):
            env.set_action_slots(h, acts[s][g])
        env.step_device_done(done.data_ptr() + 4 * s)
        env.clear_dead()
        env.restore_arenas(snap)

    def reads():
        for g, h in enumerate(hs):
            env.get_mean_action_slots_torch(h, hs[1 - g], out=means[g])
            env.get_neighbours_slots_torch(h, k, h, out=nbrs[g])

    rs = np.random.RandomState(7)

    def draw():
        for s in range(2):
            for g in range(2):
                acts[s][g].copy_(torch.from_numpy(rs.randint(0, na[g], size=(A, S[g])).astype(np.int32)))

    draw()
    one(0)
    one(1)
    reads()
    for x in means + nbrs:
        for y in x:
            y.fill_(-3)
    gid = env.capture_graph(lambda: (one(0), one(1), reads()))
    listed = 0
    for r in range(10):
        draw()
        env.launch_graph(gid, 1)
        torch.cuda.synchronize()
        for g, h in enumerate(hs):
            what = "replay %d group %d" % (r, g)
            ns.check_mean(env, h, hs[1 - g], tuple(x.cpu().numpy() for x in means[g]), what)
            listed += ns.check_neighbours(env, h, hs[g], k, tuple(x.cpu().numpy() for x in nbrs[g]), what)
    assert listed > 0
