"""The wrapper's per-agent output methods in torch form on the GPU: the engine calls each one makes, and its results.

The recording proxy of tests/wrapper_outputs_common.py logs every call the wrapper makes to the CUDA engine.  Each
torch method is run with out=None and with caller-owned tensors (optional parts given as None), for a populated group,
a group that never had an agent (S = 0) and `of` set to the other group; its log is held to a literal expectation and
its results to the numpy form.  get_observation_torch must refuse an `out` it cannot hold: the engine writes get_num
records through device pointers."""
import numpy as np
import pytest

import parity_common as pc
from wrapper_outputs_common import NULL, NUM_BOUND, PTR, SLOT_SPACE, Recorder, num

pytestmark = pytest.mark.gpu

A, N, S = 2, 24, 12          # arenas, agents of group 0 over all arenas, its slot space
P = PTR


@pytest.fixture(scope="module")
def env():
    """battle in two arenas: group 0 holds 12 agents per arena, group 1 never had one (S = 0); one step played, its
    dead not culled"""
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=20, _lib=pc.CUDA_LIB, _num_arenas=A)
    env.set_seed(3)
    env.reset()
    h0, h1 = env.get_handles()
    env.add_agents(h0, method="random", n=N // A)
    env.set_random_legal_actions(h0, 5)
    env.step()
    assert (env.get_num(h0), env.get_num_bound(h0), env.get_slot_space(h0)) == (N, N, S)
    assert (env.get_num(h1), env.get_num_bound(h1), env.get_slot_space(h1)) == (0, 0, 0)
    env._lib = Recorder(env._lib)
    return env


def filled(shape, dtype):
    """a CUDA tensor of -7s, so that a part left unwritten shows"""
    import torch
    return torch.full(shape, -7, dtype=dtype, device="cuda")


def cases(env):
    """(torch method, args, out or None, numpy method, numpy args, the expected log); a caller's row-ordered out has
    five rows more than the group (get_observation_torch returns it whole: exactly the group)"""
    import torch
    h0, h1 = env.get_handles()
    na, k = env.get_action_space(h0)[0], 4
    vs, fs = env.get_view_space(h0), env.get_feature_space(h0)
    i32, f32, u8 = torch.int32, torch.float32, torch.uint8
    return [
        ("get_action_mask_torch", (h0,), None, "get_action_mask", (h0,),
         [num(0), ("magent_b200_get_action_mask", 0, P)]),
        ("get_action_mask_torch", (h0,), filled((N + 5, na), u8), "get_action_mask", (h0,),
         [num(0), NUM_BOUND, ("magent_b200_get_action_mask", 0, P)]),
        ("get_action_mask_torch", (h0,), filled((N + 5, na), torch.bool), "get_action_mask", (h0,),
         [num(0), NUM_BOUND, ("magent_b200_get_action_mask", 0, P)]),
        ("get_action_mask_torch", (h1,), None, "get_action_mask", (h1,),
         [num(1), ("magent_b200_get_action_mask", 1, NULL)]),
        ("get_action_mask_slots_torch", (h0,), None, "get_action_mask_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_action_mask_slots", 0, P)]),
        ("get_action_mask_slots_torch", (h0,), filled((A, S, na), torch.bool), "get_action_mask_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_action_mask_slots", 0, P)]),
        ("get_action_mask_slots_torch", (h1,), None, "get_action_mask_slots", (h1,), [SLOT_SPACE]),

        ("get_mean_action_torch", (h0,), None, "get_mean_action", (h0,),
         [num(0), ("magent_b200_get_mean_action", 0, 0, P, P)]),
        ("get_mean_action_torch", (h0, h1), (filled((N + 5, na), f32), filled((N + 5,), i32)), "get_mean_action",
         (h0, h1), [num(0), NUM_BOUND, ("magent_b200_get_mean_action", 0, 1, P, P)]),
        ("get_mean_action_torch", (h1,), None, "get_mean_action", (h1,),
         [num(1), ("magent_b200_get_mean_action", 1, 1, NULL, NULL)]),
        ("get_mean_action_slots_torch", (h0,), None, "get_mean_action_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_mean_action_slots", 0, 0, P, P)]),
        ("get_mean_action_slots_torch", (h0, h1), (filled((A, S, na), f32), None), "get_mean_action_slots", (h0, h1),
         [SLOT_SPACE, ("magent_b200_get_mean_action_slots", 0, 1, P, NULL)]),
        ("get_mean_action_slots_torch", (h1,), None, "get_mean_action_slots", (h1,), [SLOT_SPACE]),

        ("get_neighbours_torch", (h0, k), None, "get_neighbours", (h0, k),
         [num(0), ("magent_b200_get_neighbours", 0, 0, k, P, P, P)]),
        ("get_neighbours_torch", (h0, k), (filled((N + 5, k), i32), None, filled((N + 5,), i32)), "get_neighbours",
         (h0, k), [num(0), NUM_BOUND, ("magent_b200_get_neighbours", 0, 0, k, P, NULL, P)]),
        ("get_neighbours_torch", (h0, k, h1), (filled((N + 5, k), i32), filled((N + 5, k, 2), i32), None),
         "get_neighbours", (h0, k, h1), [num(0), NUM_BOUND, ("magent_b200_get_neighbours", 0, 1, k, P, P, NULL)]),
        # no row to write: an empty idx would reach the engine as NULL, which it refuses
        ("get_neighbours_torch", (h1, k), None, "get_neighbours", (h1, k), [num(1)]),
        ("get_neighbours_slots_torch", (h0, k), None, "get_neighbours_slots", (h0, k),
         [SLOT_SPACE, ("magent_b200_get_neighbours_slots", 0, 0, k, P, P, P)]),
        ("get_neighbours_slots_torch", (h0, k, h1), (filled((A, S, k), i32), None, filled((A, S), i32)),
         "get_neighbours_slots", (h0, k, h1), [SLOT_SPACE, ("magent_b200_get_neighbours_slots", 0, 1, k, P, NULL, P)]),
        ("get_neighbours_slots_torch", (h1, k), None, "get_neighbours_slots", (h1, k), [SLOT_SPACE]),

        ("get_rule_actions_torch", (h0, h1, "rush", 9), None, "get_rule_actions", (h0, h1, "rush", 9),
         [num(0), ("magent_b200_get_rule_actions", 0, 1, 0, 9, P)]),
        ("get_rule_actions_torch", (h0, h0, "flee", 2), filled((N + 5,), i32), "get_rule_actions", (h0, h0, "flee", 2),
         [num(0), NUM_BOUND, ("magent_b200_get_rule_actions", 0, 0, 1, 2, P)]),
        ("get_rule_actions_torch", (h1, h0), None, "get_rule_actions", (h1, h0), [num(1)]),
        ("get_rule_actions_slots_torch", (h0, h1, "rush", 9), None, "get_rule_actions_slots", (h0, h1, "rush", 9),
         [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 0, 1, 0, 9, P)]),
        ("get_rule_actions_slots_torch", (h0, h0, "flee", 2), filled((A, S), i32), "get_rule_actions_slots",
         (h0, h0, "flee", 2), [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 0, 0, 1, 2, P)]),
        ("get_rule_actions_slots_torch", (h1, h0), None, "get_rule_actions_slots", (h1, h0),
         [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 1, 0, 0, 0, NULL)]),

        ("get_reward_slots_torch", (h0,), None, "get_reward_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_reward_slots", 0, P, P)]),
        ("get_reward_slots_torch", (h0,), (None, filled((A, S), u8)), "get_reward_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_reward_slots", 0, NULL, P)]),
        ("get_reward_slots_torch", (h0,), (filled((A, S), f32), None), "get_reward_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_reward_slots", 0, P, NULL)]),
        ("get_reward_slots_torch", (h1,), None, "get_reward_slots", (h1,), [SLOT_SPACE]),

        ("get_observation_slots_torch", (h0,), None, "get_observation_slots", (h0,),
         [SLOT_SPACE, ("magent_b200_get_observation_slots", 0, (P, P), 0)]),
        ("get_observation_slots_torch", (h0,), (filled((A, S) + vs, f32), filled((A, S) + fs, f32)),
         "get_observation_slots", (h0,), [SLOT_SPACE, ("magent_b200_get_observation_slots", 0, (P, P), 0)]),
        ("get_observation_slots_torch", (h1,), None, "get_observation_slots", (h1,), [SLOT_SPACE]),

        ("get_observation_torch", (h0,), None, "get_observation", (h0,), [num(0), ("env_get_observation", 0, (P, P))]),
        ("get_observation_torch", (h0,), (filled((N,) + vs, f32), filled((N,) + fs, f32)), "get_observation",
         (h0,), [num(0), ("env_get_observation", 0, (P, P))]),
    ]


def test_torch_outputs_call_the_engine_as_pinned_and_equal_the_numpy_form(env):
    """every torch output method with new and with caller-owned tensors: its engine calls, its results equal to the
    numpy form's (None where a part was not asked for), a caller's tensors returned as views of themselves, row-ordered
    results trimmed to the group"""
    import torch
    for name, args, out, np_name, np_args, log in cases(env):
        what = "%s%s out=%s" % (name, args, "caller's" if out is not None else None)
        env._lib.take()
        got = getattr(env, name)(*args, out=out)
        torch.cuda.synchronize()
        assert env._lib.take() == log, what
        want = getattr(env, np_name)(*np_args)
        got, want = (x if isinstance(x, tuple) else (x,) for x in (got, want))
        outs = out if isinstance(out, tuple) else (out,) * len(got)
        assert len(got) == len(want), what
        for g, w, o in zip(got, want, outs):
            if o is None and out is not None:
                assert g is None, what
                continue
            assert g.is_cuda and tuple(g.shape) == w.shape, (what, tuple(g.shape), w.shape)
            assert str(g.dtype) == "torch." + str(w.dtype), (what, g.dtype, w.dtype)
            np.testing.assert_array_equal(g.cpu().numpy(), w, err_msg=what)
            if o is not None:
                assert g.data_ptr() == o.data_ptr(), what + ": not the caller's tensor"


def test_half_observations_round_the_float32_form(env):
    import torch
    h0 = env.get_handles()[0]
    want = [x.astype(np.float16) for x in env.get_observation_slots(h0)]
    for out in (None, tuple(torch.zeros(w.shape, dtype=torch.float16, device="cuda") for w in want)):
        env._lib.take()
        got = env.get_observation_slots_torch(h0, out=out, dtype=torch.float16)
        assert env._lib.take() == [SLOT_SPACE, ("magent_b200_get_observation_slots", 0, (P, P), 1)]
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g.cpu().numpy(), w)
    want = [x.astype(np.float16) for x in env.get_observation(h0)]
    for out in (None, tuple(torch.zeros(w.shape, dtype=torch.float16, device="cuda") for w in want)):
        env._lib.take()
        got = env.get_observation_torch(h0, out=out, dtype=torch.float16)
        assert env._lib.take() == [num(0), ("magent_b200_get_observation_f16", 0, (P, P))]
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g.cpu().numpy(), w)


def test_observation_torch_refuses_an_out_it_cannot_hold(env):
    """a short, misshapen, host, non-contiguous or mixed-dtype (view, feature) pair: ValueError, and the engine is
    never called, so nothing is written past a tensor"""
    import torch
    h0 = env.get_handles()[0]
    vs, fs = env.get_view_space(h0), env.get_feature_space(h0)
    v, f = filled((N,) + vs, torch.float32), filled((N,) + fs, torch.float32)
    bad_outs = [
        (v[:N - 1], f),                                                         # short
        (v, f[:N - 1]),
        (v.view((N * vs[0],) + vs[1:]), f),                                     # misshapen, as many bytes
        (v, f.view(N // 2, 2 * fs[0])),
        (v.cpu(), f.cpu()),                                                     # host tensors
        (v, f.half()),                                                          # mixed dtypes
        (v.double(), f.double()),                                               # dtype
        (filled((N,) + vs[:2] + (2 * vs[2],), torch.float32)[..., ::2], f),     # not contiguous
        (v, f, f), v,                                                           # not a pair
    ]
    for bad in bad_outs:
        env._lib.take()
        with pytest.raises(ValueError):
            env.get_observation_torch(h0, out=bad)
        assert env._lib.take() == [num(0)], "the observation was asked for"
    long_half = (filled((N + 1,) + vs, torch.float16), filled((N + 1,) + fs, torch.float16))
    got = env.get_observation_torch(h0, out=long_half)
    assert got[0].shape == (N + 1,) + vs and got[0].dtype == torch.float16
