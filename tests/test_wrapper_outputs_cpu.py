"""The wrapper's per-agent output methods on the host emulation: the engine calls each one makes, and its refusals.

GridWorld serves the action mask, the mean action, the neighbours and the rule actions in rows and in slots, and the
reward and the observation in slots, each in a numpy and a torch form.  A recording proxy in front of the engine library
logs every call the wrapper makes, and these tests hold each numpy method to a literal log: which entry points, with
which integer arguments, and which pointers are NULL, for a populated group, a group that never had an agent (S = 0)
and `of` (or `target`) set to the other group.  The log also pins how often a method reads the counts: the slot-ordered
methods never call get_num, so they never wait for the device.

Each torch method is fed a malformed `out` (wrong arity, a host tensor, a wrong dtype): it must raise ValueError naming
what is wrong before it allocates anything on a device, which a CPU-only machine could not do."""
import numpy as np
import pytest

import wide_common as wc
from wrapper_outputs_common import NULL, NUM_BOUND, PTR, SLOT_SPACE, Recorder, num

A, N, S = 2, 24, 12          # arenas, agents of group 0 over all arenas, its slot space


@pytest.fixture(scope="module")
def env():
    """battle in two arenas: group 0 holds 12 agents per arena, group 1 never had one (S = 0)"""
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=20, _lib=wc.emu_lib(), _num_arenas=A)
    env.set_seed(3)
    env.reset()
    env.add_agents(env.get_handles()[0], method="random", n=N // A)
    env._lib = Recorder(env._lib)
    return env


def numpy_cases(env):
    """(method, args, the expected log, the expected (shape, dtype) of each result) for every numpy method"""
    h0, h1 = env.get_handles()
    na, k = env.get_action_space(h0)[0], 4
    vs, fs = env.get_view_space(h0), env.get_feature_space(h0)
    i32, f32 = np.dtype(np.int32), np.dtype(np.float32)
    bool_, u8 = np.dtype(np.bool_), np.dtype(np.uint8)
    P = PTR
    return [
        ("get_action_mask", (h0,), [num(0), ("magent_b200_get_action_mask", 0, P)], [((N, na), bool_)]),
        ("get_action_mask", (h1,), [num(1), ("magent_b200_get_action_mask", 1, P)], [((0, na), bool_)]),
        ("get_action_mask_slots", (h0,), [SLOT_SPACE, ("magent_b200_get_action_mask_slots", 0, P)],
         [((A, S, na), bool_)]),
        ("get_action_mask_slots", (h1,), [SLOT_SPACE], [((A, 0, na), bool_)]),

        ("get_mean_action", (h0,), [num(0), ("magent_b200_get_mean_action", 0, 0, P, P)],
         [((N, na), f32), ((N,), i32)]),
        ("get_mean_action", (h1,), [num(1), ("magent_b200_get_mean_action", 1, 1, P, P)],
         [((0, na), f32), ((0,), i32)]),
        ("get_mean_action", (h0, h1), [num(0), ("magent_b200_get_mean_action", 0, 1, P, P)],
         [((N, na), f32), ((N,), i32)]),
        ("get_mean_action_slots", (h0,), [SLOT_SPACE, ("magent_b200_get_mean_action_slots", 0, 0, P, P)],
         [((A, S, na), f32), ((A, S), i32)]),
        ("get_mean_action_slots", (h1,), [SLOT_SPACE], [((A, 0, na), f32), ((A, 0), i32)]),
        ("get_mean_action_slots", (h0, h1), [SLOT_SPACE, ("magent_b200_get_mean_action_slots", 0, 1, P, P)],
         [((A, S, na), f32), ((A, S), i32)]),

        ("get_neighbours", (h0, k), [num(0), ("magent_b200_get_neighbours", 0, 0, k, P, P, P)],
         [((N, k), i32), ((N, k, 2), i32), ((N,), i32)]),
        ("get_neighbours", (h1, k), [num(1), ("magent_b200_get_neighbours", 1, 1, k, P, P, P)],
         [((0, k), i32), ((0, k, 2), i32), ((0,), i32)]),
        ("get_neighbours", (h0, k, h1), [num(0), ("magent_b200_get_neighbours", 0, 1, k, P, P, P)],
         [((N, k), i32), ((N, k, 2), i32), ((N,), i32)]),
        ("get_neighbours_slots", (h0, k), [SLOT_SPACE, ("magent_b200_get_neighbours_slots", 0, 0, k, P, P, P)],
         [((A, S, k), i32), ((A, S, k, 2), i32), ((A, S), i32)]),
        ("get_neighbours_slots", (h1, k), [SLOT_SPACE], [((A, 0, k), i32), ((A, 0, k, 2), i32), ((A, 0), i32)]),
        ("get_neighbours_slots", (h0, k, h1), [SLOT_SPACE, ("magent_b200_get_neighbours_slots", 0, 1, k, P, P, P)],
         [((A, S, k), i32), ((A, S, k, 2), i32), ((A, S), i32)]),

        # an empty group's rule actions are asked for with a NULL buffer
        ("get_rule_actions", (h0, h0, "flee", 7), [num(0), ("magent_b200_get_rule_actions", 0, 0, 1, 7, P)],
         [((N,), i32)]),
        ("get_rule_actions", (h1, h1), [num(1), ("magent_b200_get_rule_actions", 1, 1, 0, 0, NULL)], [((0,), i32)]),
        ("get_rule_actions", (h0, h1), [num(0), ("magent_b200_get_rule_actions", 0, 1, 0, 0, P)], [((N,), i32)]),
        ("get_rule_actions_slots", (h0, h0, "flee", 7),
         [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 0, 0, 1, 7, P)], [((A, S), i32)]),
        ("get_rule_actions_slots", (h1, h1), [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 1, 1, 0, 0, NULL)],
         [((A, 0), i32)]),
        ("get_rule_actions_slots", (h0, h1), [SLOT_SPACE, ("magent_b200_get_rule_actions_slots", 0, 1, 0, 0, P)],
         [((A, S), i32)]),

        ("get_reward_slots", (h0,), [SLOT_SPACE, ("magent_b200_get_reward_slots", 0, P, P)],
         [((A, S), f32), ((A, S), u8)]),
        ("get_reward_slots", (h1,), [SLOT_SPACE], [((A, 0), f32), ((A, 0), u8)]),

        ("get_observation_slots", (h0,), [SLOT_SPACE, ("magent_b200_get_observation_slots", 0, (P, P), 0)],
         [((A, S) + vs, f32), ((A, S) + fs, f32)]),
        ("get_observation_slots", (h1,), [SLOT_SPACE], [((A, 0) + vs, f32), ((A, 0) + fs, f32)]),
    ]


def as_tuple(got):
    return got if isinstance(got, tuple) else (got,)


def test_numpy_outputs_call_the_engine_as_pinned(env):
    """every numpy output method: its engine calls for a populated group, an empty one and the other group, and the
    shapes and dtypes it returns"""
    assert (env.get_num(0), env.get_slot_space(0), env.get_num(1), env.get_slot_space(1)) == (N, S, 0, 0)
    env._lib.take()
    for name, args, log, shapes in numpy_cases(env):
        got = as_tuple(getattr(env, name)(*args))
        what = "%s%s" % (name, args)
        assert env._lib.take() == log, what
        assert [(a.shape, a.dtype) for a in got] == shapes, what
        assert all(isinstance(a, np.ndarray) for a in got), what


def test_numpy_outputs_keep_their_own_buffers(env):
    """a result stays valid until the next call of the same method for the same group: no two methods, and no two
    groups, share a receive buffer"""
    results = []
    for name, args, _log, _shapes in numpy_cases(env):
        results += [(name, args, a) for a in as_tuple(getattr(env, name)(*args))]
    for i, (na_, ga, a) in enumerate(results):
        for nb_, gb, b in results[i + 1:]:
            if na_ != nb_ or env._hv(ga[0]) != env._hv(gb[0]):
                assert not np.shares_memory(a, b), (na_, ga, nb_, gb)
    env._lib.take()


def test_neighbours_k_is_checked_before_any_call(env):
    h0 = env.get_handles()[0]
    env._lib.take()
    for name in ("get_neighbours", "get_neighbours_slots", "get_neighbours_torch", "get_neighbours_slots_torch"):
        for k in (0, 33):
            with pytest.raises(ValueError, match=r"k must be in \[1, 32\], got %d" % k):
                getattr(env, name)(h0, k)
    assert env._lib.take() == []


def torch_refusals(env):
    """(method, args, out, the expected log, the ValueError text) of malformed outs"""
    import torch
    h0, h1 = env.get_handles()
    na, k = env.get_action_space(h0)[0], 4
    vs, fs = env.get_view_space(h0), env.get_feature_space(h0)
    cpu = lambda shape, dtype: torch.zeros(shape, dtype=dtype)            # noqa: E731
    i32, f32, u8 = torch.int32, torch.float32, torch.uint8
    tails = lambda tail: "".join(", %d" % d for d in tail) or ","                        # noqa: E731
    rows = lambda tail: r"\(rows%s\) with at least %d rows" % (tails(tail), N)             # noqa: E731
    dt = r"dtype torch\.%s"
    cuda = r" must be a contiguous CUDA tensor of "
    mean_arity = r"out must be an? \(mean, count\) (pair|tuple) of CUDA tensors"
    nbr_arity = r"out must be an? \(idx, rel, count\) (triple|tuple) of CUDA tensors"
    bound = [num(0), NUM_BOUND]
    return [
        ("get_action_mask_torch", (h0,), cpu((N, na), u8), bound,
         "out" + cuda + dt % r"bool or torch\.uint8 and shape " + rows((na,))),
        ("get_action_mask_torch", (h0,), cpu((N, na), i32), bound,
         "out" + cuda + dt % r"bool or torch\.uint8 and shape " + rows((na,))),
        ("get_action_mask_slots_torch", (h0,), cpu((A, S, na), u8), [SLOT_SPACE],
         "out" + cuda + dt % r"bool or torch\.uint8 and shape \(%d, %d, %d\)" % (A, S, na)),

        ("get_mean_action_torch", (h0,), cpu((N, na), f32), [num(0)], mean_arity),
        ("get_mean_action_torch", (h0, h1), (cpu((N, na), f32), cpu((N,), i32)), bound,
         "mean" + cuda + dt % r"float32 and shape " + rows((na,))),
        ("get_mean_action_torch", (h0,), (cpu((N, na), torch.float64), cpu((N,), i32)), bound,
         "mean" + cuda + dt % r"float32 and shape " + rows((na,))),
        ("get_mean_action_slots_torch", (h0,), (cpu((A, S, na), f32),), [SLOT_SPACE], mean_arity),
        ("get_mean_action_slots_torch", (h0, h1), (cpu((A, S, na), f32), None), [SLOT_SPACE],
         "mean" + cuda + dt % r"float32 and shape \(%d, %d, %d\)" % (A, S, na)),

        ("get_neighbours_torch", (h0, k), (cpu((N, k), i32), None), [num(0)], nbr_arity),
        ("get_neighbours_torch", (h0, k, h1), (cpu((N, k), i32), None, None), bound,
         "idx" + cuda + dt % r"int32 and shape " + rows((k,))),
        ("get_neighbours_slots_torch", (h0, k), cpu((A, S, k), i32), [SLOT_SPACE], nbr_arity),
        ("get_neighbours_slots_torch", (h0, k), (cpu((A, S, k), torch.int64), None, None), [SLOT_SPACE],
         "idx" + cuda + dt % r"int32 and shape \(%d, %d, %d\)" % (A, S, k)),

        ("get_rule_actions_torch", (h0, h1), cpu((N,), i32), bound, "out" + cuda + dt % r"int32 and shape " + rows(())),
        ("get_rule_actions_slots_torch", (h0, h1), cpu((A, S), torch.int64), [SLOT_SPACE],
         "out" + cuda + dt % r"int32 and shape \(%d, %d\)" % (A, S)),

        ("get_reward_slots_torch", (h0,), (None, None), [SLOT_SPACE],
         r"out must be an? \(reward, status\) (pair|tuple) of CUDA tensors"),
        ("get_reward_slots_torch", (h0,), (cpu((A, S), f32), None), [SLOT_SPACE],
         "reward" + cuda + dt % r"float32 and shape \(%d, %d\)" % (A, S)),
        ("get_reward_slots_torch", (h0,), (None, cpu((A, S), u8)), [SLOT_SPACE],
         "status" + cuda + dt % r"uint8 and shape \(%d, %d\)" % (A, S)),

        ("get_observation_slots_torch", (h0,), cpu((A, S) + vs, f32), [SLOT_SPACE],
         r"out must be an? \(view, feature\) (pair|tuple) of CUDA tensors"),
        ("get_observation_slots_torch", (h0,), (cpu((A, S) + vs, f32), cpu((A, S) + fs, f32)), [SLOT_SPACE],
         "view" + cuda + dt % r"float32 or torch\.float16 and shape \(%s\)" % ", ".join(map(str, (A, S) + vs))),
    ]


def test_torch_outputs_refuse_a_malformed_out_before_touching_a_device(env):
    """a host tensor, a wrong dtype or a wrong arity: ValueError naming the part and what it must be, after no more
    engine calls than the sizes need"""
    pytest.importorskip("torch")
    env._lib.take()
    for name, args, out, log, text in torch_refusals(env):
        with pytest.raises(ValueError, match=text):
            getattr(env, name)(*args, out=out)
        assert env._lib.take() == log, name
