"""The slot-ordered step loop (magent_b200_set_action_slots, _get_reward_slots, _get_action_mask_slots) on the GPU.

An engine driven through set_action_slots with CUDA tensors (vacant slots full of garbage) must stay bit for bit the twin
of one driven through set_action in rows, and the reward, status and mask must equal the row-ordered outputs gathered
through get_slots (tests/slot_loop_common.py): in every game mode and the fuzz configs, through host and device
pointers, into unaligned and over-long outputs, across device-src and NULL-src restores, at battle512's full size, and
inside a replayed CUDA graph whose second step acts after the cull of its first."""
import ctypes

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import obs_slots_common as oc
import parity_common as pc
import slot_loop_common as lc
import slots_common as sc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def set_device(env, h, act):
    import torch
    env.set_action_slots(h, torch.from_numpy(act).cuda())


def host_and_device(env, tally=None, what=""):
    """every group's host-pointer outputs against the restatements, and the device-pointer outputs against them"""
    for h in env.get_handles():
        hr, hs = (x.copy() for x in env.get_reward_slots(h))
        hm = env.get_action_mask_slots(h).copy()
        n = lc.check_reward(env, h, (hr, hs), what)
        lc.check_mask(env, h, hm, what)
        dr, ds = env.get_reward_slots_torch(h)
        dm = env.get_action_mask_slots_torch(h)
        assert np.array_equal(dr.cpu().numpy().view(np.uint32), hr.view(np.uint32)), what + ": device rewards"
        assert np.array_equal(ds.cpu().numpy(), hs), what + ": device status"
        assert np.array_equal(dm.cpu().numpy(), hm), what + ": device mask"
        if tally is not None:
            tally.append(n)


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_twin_in_every_game_mode(name):
    """device actions, then host actions after a device-src restore and a NULL-src restore"""
    tw = lc.Twin(lambda lib: arc.SCENARIOS[name](lib, 5, _num_arenas=3), pc.CUDA_LIB, set_device)
    pools = tw.both(lambda e: e.snapshot_arenas())
    rs = np.random.RandomState(2)
    tally = []
    for t in range(6):
        tw.set_slots = set_device if t < 3 else lc.set_host
        tw.step(rs, t, cull=False)
        host_and_device(tw.s, tally, "%s step %d" % (name, t))
        tw.both(lambda e: e.clear_dead())
        tw.check("step %d after clear_dead" % t)
        if t in (1, 4):
            src = arc.as_src([2, -1, 1], "device") if t == 1 else None
            for e, p in zip((tw.s, tw.r), pools):
                e.restore_arenas(p, src)
            tw.check("step %d after a restore" % t)
            host_and_device(tw.s, tally, "%s step %d after a restore" % (name, t))
    assert sum(tally) > 0


def test_cuda_twin_under_fuzz_configs():
    for seed in (2, 6, 13, 41, 1004, 70001, 70005, 100002):
        tw = lc.Twin(lambda lib: fz.make_env(lib, seed, _num_arenas=4), pc.CUDA_LIB, set_device)
        rs = np.random.RandomState(seed)
        for t in range(4):
            tw.step(rs, t, cull=rs.rand() < 0.65, order=list(rs.permutation(len(tw.hs))), mix=True)
            host_and_device(tw.s, what="seed %d step %d" % (seed, t))


def test_unaligned_and_over_long_outputs():
    """reward, status and mask one element past an aligned start inside longer device buffers (and aligned): equal to
    the restatement, the sentinels around them untouched"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 24, 50, 7, _num_arenas=3)
    tr = sc.Slots(env)
    env.select_arena(1)
    tr.add(tr.hs[0], method="random", n=9)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    L = env._lib
    for t in range(4):
        sc.random_step(env, rs, cull=t % 2 == 1)
        for h in tr.hs:
            g = env._hv(h)
            S, na = env.get_slot_space(h), env.get_action_space(h)[0]
            n = 3 * S
            for off in (0, 1, 3):
                rw = torch.full((n + 16 + 37,), -7.0, device="cuda")
                st = torch.full((n + 16 + 37,), 0xA5, dtype=torch.uint8, device="cuda")
                mk = torch.full((n * na + 16 + 37,), 0xA5, dtype=torch.uint8, device="cuda")
                assert L.magent_b200_get_reward_slots(env.game, g, rw[off:].data_ptr(), st[off:].data_ptr()) == 0
                assert L.magent_b200_get_action_mask_slots(env.game, g, mk[off:].data_ptr()) == 0
                torch.cuda.synchronize()
                rw, st, mk = rw.cpu().numpy(), st.cpu().numpy(), mk.cpu().numpy()
                assert (rw[:off] == -7).all() and (rw[off + n:] == -7).all()
                assert (st[:off] == 0xA5).all() and (st[off + n:] == 0xA5).all()
                assert (mk[:off] == 0xA5).all() and (mk[off + n * na:] == 0xA5).all()
                what = "step %d group %d offset %d" % (t, g, off)
                lc.check_reward(env, h, (rw[off:off + n].reshape(3, S), st[off:off + n].reshape(3, S)), what)
                lc.check_mask(env, h, mk[off:off + n * na].reshape(3, S, na), what)


def test_mixed_pointers_and_bad_arguments_are_refused():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    snap = env.snapshot_arenas()
    h = env.get_handles()[1]
    S, na = env.get_slot_space(h), env.get_action_space(h)[0]
    L = env._lib
    dr = torch.full((3, S), -9.0, device="cuda")
    hs_ = np.full((3, S), 7, np.uint8)
    hr = np.full((3, S), -9.0, np.float32)
    ds = torch.full((3, S), 7, dtype=torch.uint8, device="cuda")
    for p in ((dr.data_ptr(), hs_.ctypes.data), (hr.ctypes.data, ds.data_ptr())):
        assert L.magent_b200_get_reward_slots(env.game, 1, *p) == -1
        assert b"must both be host memory or both CUDA device memory" in L.magent_b200_last_error()
    torch.cuda.synchronize()
    assert (hr == -9).all() and (hs_ == 7).all() and bool((dr == -9).all()) and bool((ds == 7).all())
    for bad in ((dr, None, None), (None, None), (dr[:, :-1].contiguous(), ds), (dr.double(), ds), (dr, ds.int()),
                (dr.cpu(), ds), dr):
        with pytest.raises(ValueError):
            env.get_reward_slots_torch(h, out=bad)
    for bad in (torch.zeros((3, S, na), dtype=torch.int32, device="cuda"), torch.zeros((3, S, na + 1), device="cuda"),
                torch.zeros((3, S, 2 * na), dtype=torch.uint8, device="cuda")[..., ::2]):
        with pytest.raises(ValueError):
            env.get_action_mask_slots_torch(h, out=bad)
    for bad in (torch.zeros((3, S), dtype=torch.int64, device="cuda"), torch.zeros((3, S + 1), dtype=torch.int32,
                                                                                      device="cuda")):
        with pytest.raises(ValueError):
            env.set_action_slots(h, bad)
    assert L.magent_b200_restore_arenas(env.game, snap, None, 0) == 0           # the refusals set no action order
    rw, st = env.get_reward_slots_torch(h, out=(dr, None))
    assert st is None
    lc.check_reward(env, h, (rw.cpu().numpy(), env.get_reward_slots(h)[1]))
    m = env.get_action_mask_slots_torch(h, out=torch.empty((3, S, na), dtype=torch.bool, device="cuda"))
    lc.check_mask(env, h, m.cpu().numpy())


# ---------------------------------------------------------------- battle512 at full size
def test_battle512_slot_native_loop_against_a_row_driven_twin():
    """bench.py's 512 arenas of 2 x 1000: 20 steps of the slot-native loop (observation, mask, actions drawn from the
    mask, set_action_slots, step, reward and status, clear_dead, restore_arenas(pool)) against a twin driven through the
    row-ordered calls and the gathers of the slot recipe, every output compared on the device"""
    import torch
    A = 512
    env, twin = (pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=A) for _ in range(2))
    hs = env.get_handles()
    pools = env.snapshot_arenas(), twin.snapshot_arenas()
    L = env._lib
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    i32 = torch.int32
    vacant = dead = 0

    def gathered(rows, slot_row):
        occ = (slot_row >= 0).view(slot_row.shape + (1,) * (rows.dim() - 1))
        return torch.where(occ, rows[slot_row.clamp(min=0).long()], torch.zeros((), dtype=rows.dtype, device="cuda"))

    for t in range(20):
        for g, h in enumerate(hs):
            gv, gf = env.get_observation_slots_torch(h)
            _rs, slot_row = twin.get_slots_torch(h)
            wv, wf = twin.get_observation_torch(h)
            assert torch.equal(gv.view(i32), gathered(wv.view(i32), slot_row)), "step %d group %d views" % (t, g)
            assert torch.equal(gf.view(i32), gathered(wf.view(i32), slot_row)), "step %d group %d features" % (t, g)
            del gv, gf, wv, wf
            mask = env.get_action_mask_slots_torch(h)
            assert torch.equal(mask, gathered(twin.get_action_mask_torch(h), slot_row)), "step %d group %d mask" % (t, g)
            act = (torch.rand(mask.shape, device="cuda", generator=gen) * mask).argmax(-1).to(i32)
            act[slot_row < 0] = -12345
            env.set_action_slots(h, act)
            row_slot, _sr = twin.get_slots_torch(h)
            rows = act.view(-1)[row_slot.clamp(min=0).long()].contiguous()
            L.env_set_action(twin.game, twin._hv(h), rows.data_ptr())
            vacant += int((slot_row < 0).sum())
        env.step_device_done(done.data_ptr())
        twin.step_device_done(done.data_ptr() + 4)
        for g, h in enumerate(hs):
            rw, st = env.get_reward_slots_torch(h)
            _rs, slot_row = twin.get_slots_torch(h)
            n = twin.get_num(h)
            twr = torch.from_numpy(twin.get_reward(h)).cuda()
            alive = torch.from_numpy(twin.get_alive(h).view(np.uint8)).cuda()
            assert torch.equal(rw.view(i32), gathered(twr.view(i32), slot_row)), "step %d group %d rewards" % (t, g)
            want_st = gathered(2 - alive, slot_row) if n else torch.zeros_like(st)
            assert torch.equal(st, want_st), "step %d group %d status" % (t, g)
            dead += int((st == 2).sum())
        for e, p in zip((env, twin), pools):
            e.clear_dead()
            e.restore_arenas(p)
        assert torch.equal(done[0], done[1])
        if t % 5 == 4:
            for g, h in enumerate(hs):
                for get in ("get_agent_id", "get_pos", "get_alive"):
                    assert np.array_equal(getattr(env, get)(h), getattr(twin, get)(h)), "step %d %s" % (t, get)
    assert vacant > 0 and dead > 0


# ---------------------------------------------------------------- CUDA graphs
def test_two_slot_native_steps_inside_a_replayed_cuda_graph():
    """two steps of the whole slot-native loop recorded with device buffers (a different action buffer per step, NULL-src
    restores, observations and masks), replayed 20 times with refilled per-slot actions, against an un-captured twin
    given the same per-slot actions in rows as it goes: the second step's actions land on the right agents after the
    cull inside the replay"""
    import torch
    env, twin = (arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4) for _ in range(2))
    hs, ths = env.get_handles(), twin.get_handles()
    snap, tsnap = env.snapshot_arenas(), twin.snapshot_arenas()
    A = 4
    S = [env.get_slot_space(h) for h in hs]
    na = [env.get_action_space(h)[0] for h in hs]
    acts = [[torch.zeros((A, S[g]), dtype=torch.int32, device="cuda") for g in range(2)] for _ in range(2)]
    rews = [[env.get_reward_slots_torch(hs[g]) for g in range(2)] for _ in range(2)]
    obs = [[env.get_observation_slots_torch(hs[g]) for g in range(2)] for _ in range(2)]
    masks = [[env.get_action_mask_slots_torch(hs[g]) for g in range(2)] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")

    def one(k):
        for g, h in enumerate(hs):
            env.set_action_slots(h, acts[k][g])
        env.step_device_done(done.data_ptr() + 4 * k)
        for g, h in enumerate(hs):
            env.get_reward_slots_torch(h, out=rews[k][g])
        env.clear_dead()
        env.restore_arenas(snap)
        for g, h in enumerate(hs):
            env.get_observation_slots_torch(h, out=obs[k][g])
            env.get_action_mask_slots_torch(h, out=masks[k][g])

    rs = np.random.RandomState(7)

    def draw():
        a = [[rs.randint(0, na[g], size=(A, S[g])).astype(np.int32) for g in range(2)] for _ in range(2)]
        for k in range(2):
            for g in range(2):
                acts[k][g].copy_(torch.from_numpy(a[k][g]))
        return a

    def twin_pair(a):
        out = []
        for k in range(2):
            for g, h in enumerate(ths):
                twin.set_action(h, lc.rows_of(twin, h, a[k][g]))
            twin.step()
            rw = [lc.expected_reward(twin, h)[:2] for h in ths]
            twin.clear_dead()
            twin.restore_arenas(tsnap)
            out.append([(rw[g], oc.expected(twin, h, 0)[:2], lc.expected_mask(twin, h)) for g, h in enumerate(ths)])
        return out

    a = draw()
    one(0)
    one(1)
    twin_pair(a)
    for k in range(2):
        for g in range(2):
            for x in rews[k][g] + obs[k][g]:
                x.fill_(-3)
            masks[k][g].fill_(True)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    occupied = 0
    for r in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for g, ((wr, ws), (wv, wf), wm) in enumerate(want[k]):
                what = "replay %d step %d group %d" % (r, k, g)
                assert np.array_equal(rews[k][g][0].cpu().numpy().view(np.uint32), wr.view(np.uint32)), what + " rewards"
                assert np.array_equal(rews[k][g][1].cpu().numpy(), ws), what + " status"
                assert np.array_equal(obs[k][g][0].cpu().numpy().view(np.uint32), wv.view(np.uint32)), what + " views"
                assert np.array_equal(obs[k][g][1].cpu().numpy().view(np.uint32), wf.view(np.uint32)), what + " features"
                assert np.array_equal(masks[k][g].cpu().numpy().view(np.uint8), wm), what + " mask"
                occupied += int((ws > 0).sum())
    assert occupied > 0
    for get in ("get_agent_id", "get_pos", "get_alive"):
        for h, th in zip(hs, ths):
            assert np.array_equal(getattr(env, get)(h), getattr(twin, get)(th)), get
