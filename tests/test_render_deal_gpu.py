"""The observation render deals its chunks of tiles per SM through device counters: every CTA claims chunks from the
counter of the SM it runs on and, once that SM's sequence is drained, from the other SMs' counters.  Whatever the grid,
every chunk must be rendered exactly once, and the counters must be back at zero after every launch (a replayed CUDA
graph has no node that clears them).

These tests render the same state under the automatic launch (at these sizes: chunks round-robin over the CTAs), under
forced grids, which always deal when there is more than one round, that leave most SMs without a CTA (1 CTA) or give
SMs more CTAs than fit at once (more CTAs than SMs times the most that any SM can hold), and with one tile per CTA
(grid = tiles: a single round, no counters), and require the results to be equal bit for bit.  A captured graph with a
dealing render is replayed 20 times against an un-captured twin that renders without counters."""
import numpy as np
import pytest

import parity_common as pc

pytestmark = pytest.mark.gpu

ARENAS = 16
STEPS = 3
ONE_TILE_PER_CTA = (1 << 20, 1, 0)       # grid clamped to the tile count: every CTA renders one tile, nothing is dealt


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def observe_all(env, launch):
    env._set_obs_launch(*launch)
    out = []
    for h in env.get_handles():
        v, f = env.get_observation_torch(h)
        out.append((v.cpu().numpy().view(np.uint32), f.cpu().numpy().view(np.uint32), env._get_obs_launch()))
    env._set_obs_launch(0, 0, 0)
    return out


def dealt(report):
    return report["grid"] * report["chunk"] < report["tiles"]


def check_shapes(env, steps):
    """the observations of every group under each launch shape, equal to one tile per CTA, for `steps` steps"""
    for step in range(steps):
        want = observe_all(env, ONE_TILE_PER_CTA)
        for v, f, rep in want:
            assert not dealt(rep) and rep["grid"] == rep["tiles"], rep
        tile_agents = want[0][2]["tile_agents"]
        # more CTAs than any SM count times CTAs per SM can hold at once (at most 64 warps per SM): some SMs take extra
        over = sm_count() * 64 // tile_agents + 7
        shapes = {"automatic": (0, 0, 0), "one CTA": (1, 0, 0), "more CTAs than fit": (over, 1, 0)}
        for name, launch in shapes.items():
            got = observe_all(env, launch)
            for g, ((wv, wf, _), (v, f, rep)) in enumerate(zip(want, got)):
                assert dealt(rep), (name, g, rep)
                if launch[0]:
                    assert rep["grid"] == launch[0], (name, g, rep)
                np.testing.assert_array_equal(v, wv, err_msg="%s: views of group %d, step %d" % (name, g, step))
                np.testing.assert_array_equal(f, wf, err_msg="%s: features of group %d, step %d" % (name, g, step))
        for h in env.get_handles():
            env.set_random_actions(h, 50 + step)
        env.step()
        env.clear_dead()


def test_multi_arena_battle_any_grid():
    env = pc.make_battle(pc.CUDA_LIB, 80, 600, 3, _num_arenas=ARENAS)
    assert min(env.get_num(h) for h in env.get_handles()) // 8 > sm_count() * 8 + 7
    check_shapes(env, STEPS)


def test_gather_batch_any_grid():
    env = pc.make_gather(pc.CUDA_LIB, 80, 4, n_agent=600, n_food=900, _num_arenas=ARENAS)
    check_shapes(env, STEPS)


def test_replayed_graph_resets_the_counters():
    """two steps with the render (64 CTAs, dealt) captured once and replayed 20 times with refilled actions; the twin
    makes the same calls un-captured and renders with one tile per CTA"""
    import ctypes
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env, twin = (pc.make_battle(pc.CUDA_LIB, 80, 600, 9, _num_arenas=12) for _ in range(2))
    env._set_obs_launch(64, 1, 0)
    twin._set_obs_launch(*ONE_TILE_PER_CTA)
    bound = [env.get_num(h) for h in env.get_handles()]
    n_act = env.get_action_space(env.get_handles()[0])[0]
    acts, tacts = ([[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)] for _ in range(2))
    rs = np.random.RandomState(11)

    def draw():
        for k in range(2):
            for g, n in enumerate(bound):
                a = torch.from_numpy(rs.randint(0, n_act, size=n).astype(np.int32))
                acts[k][g].copy_(a)
                tacts[k][g].copy_(a)

    def buffers(e):
        return {e._hv(h): (torch.zeros((e.get_num(h),) + e.get_view_space(h), dtype=torch.float32, device="cuda"),
                           torch.zeros((e.get_num(h),) + e.get_feature_space(h), dtype=torch.float32, device="cuda"))
                for h in e.get_handles()}

    bufs, tbufs = buffers(env), buffers(twin)
    done, tdone = (torch.zeros((1,), dtype=torch.int32, device="cuda") for _ in range(2))

    def dev_step(e, b, d, a):
        for g, (v, f) in b.items():
            L.env_get_observation(e.game, g, (ctypes.c_void_p * 2)(v.data_ptr(), f.data_ptr()))
        for h, x in zip(e.get_handles(), a):
            L.env_set_action(e.game, e._hv(h), x.data_ptr())
        e.step_device_done(d.data_ptr())
        e.clear_dead()

    draw()
    for k in range(2):
        dev_step(env, bufs, done, acts[k])
        dev_step(twin, tbufs, tdone, tacts[k])
    rep = env._get_obs_launch()
    gid = env.capture_graph(lambda: (dev_step(env, bufs, done, acts[0]), dev_step(env, bufs, done, acts[1])))
    for r in range(20):
        draw()
        env.launch_graph(gid, 1)
        dev_step(twin, tbufs, tdone, tacts[0])
        dev_step(twin, tbufs, tdone, tacts[1])
        torch.cuda.synchronize()
        for g in bufs:
            for k in range(2):
                np.testing.assert_array_equal(bufs[g][k].cpu().numpy().view(np.uint32), tbufs[g][k].cpu().numpy().view(np.uint32),
                                              err_msg="replay %d, group %d" % (r, g))
    assert dealt(rep), rep
    assert not dealt(twin._get_obs_launch())
