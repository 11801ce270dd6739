"""The global state (magent_b200_get_global_state) computed by the CUDA kernel, on the GPU.

  * the scenarios of tests/test_global_state_cpu.py in lockstep with the reference, the state read through a host
    buffer and through a device tensor (identical), and in float16 (the float32 state rounded to nearest-even);
  * battle at its full size (512 arenas of 2 x 1000 agents) against a PyTorch restatement, every observer's window
    against its view, and three arenas against independent references;
  * the call recorded into a CUDA graph, and made with device pointers in the middle of a device-resident loop."""
import ctypes
import os

import numpy as np
import pytest

import fullsize_common as fs
import global_state_common as gs
import parity_common as pc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


def read_host_and_device(env):
    """[host float32, device float32]; the float16 state checked against the float32 one on the way"""
    import torch
    host = env.get_global_state().copy()
    dev = env.get_global_state_torch().cpu().numpy()
    half = env.get_global_state_torch(dtype=torch.float16).cpu().numpy()
    np.testing.assert_array_equal(half.view(np.uint16), host.astype(np.float16).view(np.uint16))
    return [host, dev]


SCENARIOS = {
    "battle": lambda lib: pc.make_battle(lib, 30, 120, 3),
    "battle_rect": lambda lib: pc.make_battle_rect(lib),
    "pursuit": lambda lib: pc.make_pursuit(lib),
    "gather": lambda lib: pc.make_gather(lib, 30, 1),
    "food": lambda lib: pc.make_food(lib, 30, 3),
    "sector": lambda lib: pc.make_sector(lib),
    "multi4": lambda lib: pc.make_multi4(lib),
    "arrange": lambda lib: pc.make_arrange(lib),
}


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_state_matches_the_reference_views_and_getters(name):
    gs.play_lockstep(SCENARIOS[name], pc.CUDA_LIB, checker_lib(), 15, 4, read_host_and_device)


def test_state_in_turn_mode(tmp_path):
    gs.play_lockstep(lambda lib: pc.make_turn(lib, 30, 5), pc.CUDA_LIB, checker_lib(), 15, 5, read_host_and_device,
                     str(tmp_path), turn=True)


def test_arena_batch_equals_single_arena_references():
    gs.play_batch_lockstep(lambda lib, seed, **kw: pc.make_battle(lib, 30, 80, seed, **kw), pc.CUDA_LIB, checker_lib(),
                           4, 12, 7, read_host_and_device)


def test_ragged_and_offset_outputs():
    """A*H*W*C not a multiple of the 16-byte vector (the ragged end), written into a tensor that is a view 16 bytes
    into a larger allocation: the bytes around the state stay untouched"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 13, 20, 2, _num_arenas=3)           # 3 * 13 * 13 * 5 = 2535 elements
    want = env.get_global_state().copy()
    for dtype, pad in ((torch.float32, 4), (torch.float16, 8)):
        n = want.size
        big = torch.full((n + 3 * pad,), 7.0, dtype=dtype, device="cuda")
        out = big[pad:pad + n].view(want.shape)
        env.get_global_state_torch(out=out)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(out.cpu().numpy(), want.astype(out.cpu().numpy().dtype))
        rest = torch.cat([big[:pad], big[pad + n:]])
        assert bool((rest == 7.0).all()), "bytes outside the state were written"
    with pytest.raises(ValueError):
        env.get_global_state_torch(out=big[1:1 + want.size].view(want.shape))             # not 16-byte aligned


def test_battle_512_arenas_of_2x1000():
    """bench.py's default workload: the whole batch against a PyTorch restatement (positions from the engine, hp from
    each agent's own view centre), every observer's view window against the state, arenas 0 / 255 / 511 against
    independent references"""
    import torch
    A, size, n, seed, R = 512, 200, 1000, 100, 6
    env = pc.make_battle(pc.CUDA_LIB, size, n, seed, _num_arenas=A)
    samples = {a: pc.make_battle(checker_lib(), size, n, seed + a) for a in (0, 255, 511)}
    hs = env.get_handles()
    dev = torch.device("cuda")
    d = torch.arange(-R, R + 1, device=dev)
    mask = (d.view(-1, 1) ** 2 + d.view(1, -1) ** 2) <= R * R
    rs = np.random.RandomState(17)
    for t in range(3):
        state = env.get_global_state_torch()
        assert state.shape == (A, size, size, 5)
        views = [env.get_observation_torch(h)[0] for h in hs]
        nums = [env.get_arena_nums(h).astype(np.int64) for h in hs]
        pos = [torch.as_tensor(env.get_pos(h), device=dev).long() for h in hs]
        exp = torch.zeros_like(state)
        exp[:, 0, :, 0] = exp[:, size - 1, :, 0] = exp[:, :, 0, 0] = exp[:, :, size - 1, 0] = 1.0
        for g in range(2):
            ar = fs.arena_index(nums[g], dev)
            x, y = pos[g][:, 0], pos[g][:, 1]
            exp[ar, y, x, 1 + 2 * g] = 1.0
            exp[ar, y, x, 2 + 2 * g] = views[g][:, R, R, 2]
        fs.assert_bits_equal(state, exp, "step %d state" % t)
        # every observer's window, gathered out of the state
        sp = torch.zeros((A, size + 2 * R, size + 2 * R, 5), dtype=torch.float32, device=dev)
        sp[:, R:R + size, R:R + size] = state
        for g in range(2):
            ar = fs.arena_index(nums[g], dev)
            order = [g, 1 - g]
            for s in range(0, pos[g].shape[0], 65536):
                e = min(pos[g].shape[0], s + 65536)
                yy = (pos[g][s:e, 1] + R).view(-1, 1, 1) + d.view(1, -1, 1)
                xx = (pos[g][s:e, 0] + R).view(-1, 1, 1) + d.view(1, 1, -1)
                win = torch.where(mask.view(1, 2 * R + 1, 2 * R + 1, 1), sp[ar[s:e].view(-1, 1, 1), yy, xx], 0.0)
                v = views[g][s:e]
                fs.assert_bits_equal(v[..., 0], win[..., 0], "step %d group %d wall" % (t, g))
                for slot, og in enumerate(order):
                    for k in (0, 1):
                        fs.assert_bits_equal(v[..., 1 + 3 * slot + k], win[..., 1 + 2 * og + k],
                                             "step %d group %d view channel %d" % (t, g, 1 + 3 * slot + k))
        host = state.cpu().numpy()
        for a, ref in samples.items():
            gs.check_arena_state(host[a], ref, None, "step %d arena %d" % (t, a))
        del views, sp, exp
        off = [np.concatenate([[0], np.cumsum(nm)]) for nm in nums]
        for g, h in enumerate(hs):
            act = rs.randint(0, 21, size=int(nums[g].sum())).astype(np.int32)
            env.set_action(h, act)
            for a, ref in samples.items():
                ref.set_action(ref.get_handles()[g], np.ascontiguousarray(act[off[g][a]:off[g][a + 1]]))
        env.step()
        for ref in samples.values():
            ref.step()
            ref.clear_dead()
        env.clear_dead()


def test_replayed_cuda_graph_writes_the_state():
    """two steps recorded with get_global_state_torch(out=...) into fixed tensors (float32 and float16), replayed 10
    times with refilled actions, against an un-captured twin engine driven with the same actions"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env = pc.make_battle(pc.CUDA_LIB, 30, 300, 3, _num_arenas=2)
    twin = pc.make_battle(pc.CUDA_LIB, 30, 300, 3, _num_arenas=2)
    hs = env.get_handles()
    n0 = [env.get_num(h) for h in hs]
    shape = (2,) + env.get_state_space()
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in n0] for _ in range(2)]
    s32 = [torch.empty(shape, dtype=torch.float32, device="cuda") for _ in range(2)]
    s16 = [torch.empty(shape, dtype=torch.float16, device="cuda") for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")

    def one(k):
        for h, a in zip(hs, acts[k]):
            L.env_set_action(env.game, env._hv(h), a.data_ptr())
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()
        env.get_global_state_torch(out=s32[k])
        env.get_global_state_torch(out=s16[k])

    rs = np.random.RandomState(7)

    def draw():
        a = [[rs.randint(0, 21, size=n).astype(np.int32) for n in n0] for _ in range(2)]
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
            out.append(twin.get_global_state().copy())
        return out

    a = draw()
    one(0)
    one(1)                                              # one un-captured pair first: every buffer gets its size
    want = twin_pair(a)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    for _ in range(10):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            np.testing.assert_array_equal(s32[k].cpu().numpy().view(np.uint32), want[k].view(np.uint32))
            np.testing.assert_array_equal(s16[k].cpu().numpy().view(np.uint16), want[k].astype(np.float16).view(np.uint16))
    assert twin.get_num(twin.get_handles()[0]) < 600, "agents are supposed to die inside the replays"


def test_device_state_mid_loop_needs_no_counts():
    """get_global_state_torch between device-resident steps: no count read-back, and the state of that moment"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 30, 250, 5)
    ref = pc.make_battle(checker_lib(), 30, 250, 5)
    hs, rhs = env.get_handles(), ref.get_handles()
    L = env._lib
    done = torch.zeros((1,), dtype=torch.int32, device="cuda")
    out = torch.empty((1,) + env.get_state_space(), dtype=torch.float32, device="cuda")
    rs = np.random.RandomState(9)
    for t in range(12):
        acts = [rs.randint(0, 21, size=ref.get_num(h)).astype(np.int32) for h in rhs]
        d_acts = [torch.from_numpy(x).cuda() for x in acts]
        for h, rh, x, dx in zip(hs, rhs, acts, d_acts):
            L.env_set_action(env.game, env._hv(h), ctypes.c_void_p(dx.data_ptr()))
            ref.set_action(rh, x)
        env.step_device_done(done.data_ptr())
        env.clear_dead()
        ref.step()
        ref.clear_dead()
        before = env.get_io_stats()["d2h"]
        env.get_global_state_torch(out=out)
        assert env.get_io_stats()["d2h"] == before, "the state call read something back"
        gs.check_arena_state(out.cpu().numpy()[0], ref, None, "step %d" % t)
