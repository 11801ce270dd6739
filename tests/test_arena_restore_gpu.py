"""The reset pool (snapshot_arenas / restore_arenas) with the CUDA restore kernel, on the GPU.

  * the scenarios of tests/test_arena_restore_cpu.py, with src passed as a host array, as a CUDA tensor and as NULL
    (the done flags);
  * battle at its full size (512 arenas of 2 x 1000 agents): a random tenth of the arenas restored from a CUDA tensor
    after 30 device-resident steps, checked against the snapshot and against reference twins;
  * out-of-range device sources, a restore into arenas large enough for the whole-grid step kernels, and the restore
    recorded into a CUDA graph together with two steps, replayed against an un-captured twin engine."""
import ctypes
import os

import numpy as np
import pytest

import arena_restore_common as ar
import fullsize_common as fs
import parity_common as pc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


@pytest.mark.parametrize("src_kind", ["host", "device"])
@pytest.mark.parametrize("name", sorted(ar.SCENARIOS))
def test_restart_equals_a_fresh_episode(name, src_kind):
    assert ar.play_restarts(ar.SCENARIOS[name], pc.CUDA_LIB, checker_lib(), src_kind=src_kind) >= 8


def test_done_arenas_restart_on_their_own():
    n = ar.play_restarts(ar.make_duel, pc.CUDA_LIB, checker_lib(), steps=60, seed=3, plan={t: None for t in range(60)},
                         arenas=8)
    assert n >= 3, "no arena finished: the scenario no longer exercises the done-driven restore"


@pytest.mark.parametrize("name", ["battle", "pursuit", "turn"])
def test_keep_rng_continues_the_arenas_own_stream(name):
    assert ar.play_restarts(ar.SCENARIOS[name], pc.CUDA_LIB, checker_lib(), src_kind="device", keep_rng=True) >= 8


@pytest.mark.parametrize("name", ["battle", "food", "arrange"])
def test_mid_episode_snapshot_replays_identically(name):
    ar.mid_episode_replay(ar.SCENARIOS[name], pc.CUDA_LIB, src_kind="device")


def test_add_agents_after_a_device_restore_continues_the_ids():
    L = ar.Lockstep(ar.make_duel, pc.CUDA_LIB, checker_lib(), 4, 9)
    pool = L.snapshot()
    for _ in range(12):
        L.step()
    assert L.restore(pool, [1, -1, 3, 0], "device") == 3
    L.check(" (after the restore)")
    L.eng.add_agents(L.eng.get_handles()[0], method="random", n=3)
    for ref in L.refs:
        ref.add_agents(ref.get_handles()[0], method="random", n=3)
    for _ in range(3):
        L.check()
        L.step()


def test_restore_after_capacity_growth():
    L = ar.Lockstep(ar.SCENARIOS["battle"], pc.CUDA_LIB, checker_lib(), 4, 11)
    L.step()
    pool = L.snapshot()
    L.step()
    L.eng.add_agents(L.eng.get_handles()[0], method="random", n=60)
    for ref in L.refs:
        ref.add_agents(ref.get_handles()[0], method="random", n=60)
    L.step()
    assert L.restore(pool, [2, -1, 0, 1], "device") == 3
    for _ in range(4):
        L.check()
        L.step()


def test_device_src_out_of_range_is_ignored():
    plan = {1: [-5, 4, 100, 1], 3: [7, -1, 2, -(1 << 30)]}
    assert ar.play_restarts(ar.SCENARIOS["battle"], pc.CUDA_LIB, checker_lib(), steps=6, plan=plan, src_kind="device") == 2


def _hp(env, h):
    n = env.get_num(h)
    buf = np.empty((n,), dtype=np.float32)
    env._lib.env_get_info(env.game, env._hv(h), b"hp", buf.ctypes.data)
    return buf


def _per_arena(env):
    """per group: (arena offsets, pos, ids, hp) of the whole batch"""
    out = []
    for h in env.get_handles():
        off = np.concatenate([[0], np.cumsum(env.get_arena_nums(h))])
        out.append((off, env.get_pos(h).copy(), env.get_agent_id(h).copy(), _hp(env, h)))
    return out


def test_battle_512_arenas_of_2x1000():
    """bench.py's default workload: snapshot after placement, 30 device-resident steps with device actions, then a
    random tenth of the arenas (0, 255 and 511 among them) restored from a CUDA tensor"""
    import torch
    A, size, n, seed = 512, 200, 1000, 100
    env = pc.make_battle(pc.CUDA_LIB, size, n, seed, _num_arenas=A)
    hs, L = env.get_handles(), env._lib
    pool = env.snapshot_arenas()
    snap_state = env.get_global_state_torch()
    snap = _per_arena(env)
    bound = [env.get_num_bound(h) for h in hs]
    assert bound == [A * n, A * n]
    acts = [torch.empty((b,), dtype=torch.int32, device="cuda") for b in bound]
    done = torch.zeros((1,), dtype=torch.int32, device="cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    for _ in range(30):
        for h, x in zip(hs, acts):
            x.random_(0, 21, generator=gen)
            L.env_set_action(env.game, env._hv(h), ctypes.c_void_p(x.data_ptr()))
        env.step_device_done(done.data_ptr())
        env.clear_dead()
    rs = np.random.RandomState(1)
    chosen = sorted(set(rs.choice(A, A // 10, replace=False).tolist()) | {0, 255, 511})
    src = np.full((A,), -1, dtype=np.int32)
    src[chosen] = rs.randint(0, A, size=len(chosen))
    before = env.get_global_state_torch()
    env.restore_arenas(pool, torch.from_numpy(src).cuda())
    after = env.get_global_state_torch()
    keep = torch.from_numpy(src < 0).cuda()
    fs.assert_bits_equal(after[keep], before[keep], "arenas that were not restored")
    idx = torch.from_numpy(src[chosen]).long().cuda()
    fs.assert_bits_equal(after[torch.tensor(chosen).cuda()], snap_state[idx], "restored arenas vs the snapshot")
    now = _per_arena(env)
    for g in range(2):
        off0, pos0, id0, hp0 = snap[g]
        off1, pos1, id1, hp1 = now[g]
        for a in chosen:
            s = src[a]
            for what, x0, x1 in (("pos", pos0, pos1), ("ids", id0, id1), ("hp", hp0, hp1)):
                np.testing.assert_array_equal(x1[off1[a]:off1[a + 1]], x0[off0[s]:off0[s + 1]],
                                              err_msg="group %d arena %d (from %d) %s" % (g, a, s, what))
    # arenas 0, 255 and 511 play on against reference twins of their source arenas
    twins = {a: pc.make_battle(checker_lib(), size, n, seed + int(src[a])) for a in (0, 255, 511)}
    for t in range(4):
        nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
        offs = [np.concatenate([[0], np.cumsum(x)]) for x in nums]
        views = [env.get_observation_torch(h) for h in hs]
        ids, pos = [env.get_agent_id(h) for h in hs], [env.get_pos(h) for h in hs]
        for a, ref in twins.items():
            for g, rh in enumerate(ref.get_handles()):
                sl = slice(offs[g][a], offs[g][a + 1])
                m = "step %d arena %d group %d" % (t, a, g)
                assert nums[g][a] == ref.get_num(rh), m
                np.testing.assert_array_equal(ids[g][sl], ref.get_agent_id(rh), err_msg=m + " ids")
                np.testing.assert_array_equal(pos[g][sl], ref.get_pos(rh), err_msg=m + " pos")
                rv, rf = ref.get_observation(rh)
                np.testing.assert_array_equal(views[g][0][sl].cpu().numpy().view(np.uint32), rv.view(np.uint32),
                                              err_msg=m + " views")
                np.testing.assert_array_equal(views[g][1][sl].cpu().numpy().view(np.uint32), rf.view(np.uint32),
                                              err_msg=m + " features")
        del views
        for g, h in enumerate(hs):
            act = rs.randint(0, 21, size=int(offs[g][-1])).astype(np.int32)
            env.set_action(h, act)
            for a, ref in twins.items():
                ref.set_action(ref.get_handles()[g], np.ascontiguousarray(act[offs[g][a]:offs[g][a + 1]]))
        env.step()
        rew = [env.get_reward(h) for h in hs]
        for a, ref in twins.items():
            ref.step()
            for g, rh in enumerate(ref.get_handles()):
                np.testing.assert_allclose(rew[g][offs[g][a]:offs[g][a + 1]], ref.get_reward(rh), rtol=0,
                                           atol=pc.REWARD_TOL, err_msg="step %d arena %d group %d reward" % (t, a, g))
            ref.clear_dead()
        env.clear_dead()


def test_restore_into_whole_grid_arenas():
    """2 arenas of 2 x 20000 agents (above the 32768 agents per arena where the whole grid teams up on one arena),
    restored to counts above the current ones, then stepped against the references"""
    make = lambda lib, seed, **kw: pc.make_battle(lib, 300, 20000, seed, **kw)
    L = ar.Lockstep(make, pc.CUDA_LIB, checker_lib(), 2, 21)
    pool = L.snapshot()
    for _ in range(8):
        L.step()
    low = [L.eng.get_arena_nums(h).copy() for h in L.eng.get_handles()]
    assert min(int(x.min()) for x in low) < 20000, "agents are supposed to die"
    assert L.restore(pool, [1, 0], "device") == 2
    for h in L.eng.get_handles():
        np.testing.assert_array_equal(L.eng.get_arena_nums(h), [20000, 20000])
    for _ in range(2):
        L.check()
        L.step()
    L.check()


def test_restore_recorded_into_a_cuda_graph():
    """gather, 64 arenas: two steps, get_arena_done_torch and restore_arenas(pool, device src) recorded into one graph,
    its device buffers sized by get_num_bound; replayed 20 times with refilled actions and sources against an
    un-captured twin engine fed the same actions and sources, output for output"""
    import torch
    A = 64
    make = lambda lib: pc.make_gather(lib, 40, 4, 20, 60, _num_arenas=A)
    env, twin = make(pc.CUDA_LIB), make(pc.CUDA_LIB)
    L = env._lib
    pool, tpool = env.snapshot_arenas(), twin.snapshot_arenas()
    hs = env.get_handles()
    bound = [env.get_num_bound(h) for h in hs]
    acts = [[torch.zeros((b,), dtype=torch.int32, device="cuda") for b in bound] for _ in range(2)]
    rews = [[torch.zeros((b,), dtype=torch.float32, device="cuda") for b in bound] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    arena_done = torch.zeros((A,), dtype=torch.int32, device="cuda")
    src = torch.full((A,), -1, dtype=torch.int32, device="cuda")

    def seq():
        for k in range(2):
            for h, a in zip(hs, acts[k]):
                L.env_set_action(env.game, env._hv(h), ctypes.c_void_p(a.data_ptr()))
            env.step_device_done(done.data_ptr() + 4 * k)
            for h, r in zip(hs, rews[k]):
                L.env_get_reward(env.game, env._hv(h), ctypes.c_void_p(r.data_ptr()))
            env.clear_dead()
        env.get_arena_done_torch(out=arena_done)
        env.restore_arenas(pool, src)

    rs = np.random.RandomState(7)

    def draw():
        a = [[rs.randint(0, env.get_action_space(h)[0], size=b).astype(np.int32) for h, b in zip(hs, bound)]
             for _ in range(2)]
        s = np.full((A,), -1, dtype=np.int32)
        pick = rs.choice(A, 5, replace=False)
        s[pick] = rs.randint(-2, A + 2, size=5)           # some out of range: ignored
        for k in range(2):
            for g in range(2):
                acts[k][g].copy_(torch.from_numpy(a[k][g]))
        src.copy_(torch.from_numpy(s))
        return a, s

    def twin_run(a, s):
        out = []
        for k in range(2):
            for h, x in zip(twin.get_handles(), a[k]):
                twin.set_action(h, np.ascontiguousarray(x[:twin.get_num(h)]))
            twin.step()
            out.append([twin.get_reward(h).copy() for h in twin.get_handles()])
            twin.clear_dead()
        d = twin.get_arena_done().copy()
        twin.restore_arenas(tpool, np.where((s >= 0) & (s < A), s, -1).astype(np.int32))
        return out, d

    a, s = draw()
    seq()                                               # one un-captured round first: every buffer gets its size
    twin_run(a, s)
    gid = env.capture_graph(seq)
    for rep in range(20):
        a, s = draw()
        env.launch_graph(gid, 1)
        want, want_done = twin_run(a, s)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(arena_done.cpu().numpy(), want_done, err_msg="replay %d arena done" % rep)
        for k in range(2):
            for g in range(2):
                n = len(want[k][g])
                np.testing.assert_allclose(rews[k][g][:n].cpu().numpy(), want[k][g], rtol=0, atol=0,
                                           err_msg="replay %d step %d group %d rewards" % (rep, k, g))
        for h, th in zip(hs, twin.get_handles()):
            assert env.get_num(h) == twin.get_num(th) <= env.get_num_bound(h)
            np.testing.assert_array_equal(env.get_arena_nums(h), twin.get_arena_nums(th))
            np.testing.assert_array_equal(env.get_agent_id(h), twin.get_agent_id(th), err_msg="replay %d ids" % rep)
            np.testing.assert_array_equal(env.get_pos(h), twin.get_pos(th), err_msg="replay %d pos" % rep)
    np.testing.assert_array_equal(env.get_arena_rng(), twin.get_arena_rng())
