"""The edge configurations of tests/wide_common.py on the host emulation: large views and wide action spaces, where the
side-output kernels' shared memory reaches the device's limits.

Every config is asserted to sit on the side of its limit it was made for, played for a few steps against the compiled
reference (or the oracle port where the reference is absent), and checked against the numpy restatements of the mean
action, the neighbours, the legal-action mask, the legal draws and their slot-ordered forms.  That pins the
restatements at these sizes, so that the GPU tests can hold the CUDA kernels to them."""
import os

import numpy as np
import pytest

import action_mask_common as am
import mean_action_common as ma
import nbr_slots_common as ns
import neighbours_common as nb
import parity_common as pc
import slot_loop_common as lc
import wide_common as wc


@pytest.fixture(scope="module")
def emu():
    return wc.emu_lib()


def checker():
    lib = next((p for p in (pc.REF_LIB, pc.PORT_LIB) if os.path.exists(p)), None)
    if lib is None:
        pytest.skip("neither the compiled reference nor the oracle port is built")
    return lib


def restatements(env, tmp_path, held, what, nbr=True):
    """mean, neighbours, mask and their slot-ordered forms against the restatements; returns the neighbours counted"""
    turn = bool(env.config.config_dict.get("turn_mode", False))
    dirs = am.frame_headings(env, str(tmp_path)) if turn else None
    total = ma.check_means(env, dirs, what, acts=wc.acts_by_id(env, held))
    if nbr:
        for k in (1, 32):
            nb.check_rows(env, k, dirs, "%s k %d" % (what, k))
        ns.check_all(env, ks=(1, 32), what=what)
    else:
        for h in env.get_handles():
            with pytest.raises(RuntimeError, match="too large to order its cells"):
                env.get_neighbours(h, 1)
    am.check_masks(env, dirs, what=what)
    for h in env.get_handles():
        lc.check_mask(env, h, what=what)
    return total


@pytest.mark.parametrize("name", sorted(wc.EDGES))
def test_edge_config_against_the_reference_and_the_restatements(emu, name, tmp_path):
    """the config on its side of every limit it was made for; three steps equal to the reference's (observations too
    where the render holds the view); the restatements after every step"""
    with_obs = wc.EDGES[name][2].get("render") == "in"
    ref = checker()
    want = wc.state_trace(wc.make(ref, name, seed=3), 3, 5, with_obs)
    env = wc.make(emu, name, seed=3)
    wc.check_edge(env, name)
    pc.compare_traces(want, wc.state_trace(env, 3, 5, with_obs), name)
    env = wc.make(emu, name, seed=4)
    if env.config.config_dict.get("turn_mode", False):
        env.set_render_dir(str(tmp_path))
    rs = np.random.RandomState(6)
    held = {}
    nbr = wc.EDGES[name][2].get("nbr", "in") == "in"
    listed = 0
    for t in range(2):
        wc.random_step(env, rs, held)
        listed += restatements(env, tmp_path, held, "%s step %d" % (name, t), nbr)
    assert listed > 0


@pytest.mark.parametrize("na", sorted(wc.MASK_SPACES))
def test_wide_action_space_against_the_reference_and_the_restatements(emu, na, tmp_path):
    """a crowded game with `na` actions per agent: long move chains in the step against the reference, the mask, the
    legal draws, the mean action and the neighbours against the restatements"""
    ref = checker()
    steps = 2 if na > 800 else 4
    pc.compare_traces(wc.state_trace(wc.make_mask(ref, na, seed=2), steps, 9, True),
                      wc.state_trace(wc.make_mask(emu, na, seed=2), steps, 9, True), "%d actions" % na)
    nbytes = wc.STATIC_ENGINE + 256 * na + 16
    assert wc.side(nbytes, "mask") == ("in" if na < 167 else "optin" if na <= 881 else "past"), (na, nbytes)
    env = wc.make_mask(emu, na, seed=3)
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmp_path))
    rs = np.random.RandomState(na)
    held = {}
    calls = 0
    for t in range(steps):
        restatements(env, tmp_path, held, "%d actions step %d" % (na, t))
        for g, h in enumerate(env.get_handles()):
            mask = env.get_action_mask(h).copy()
            env.set_random_legal_actions(h, 11 + t)
            calls += 1
            acts = am.last_actions(env, h)
            np.testing.assert_array_equal(acts, am.restate_draws(mask, 11 + t, calls, t))
            for i, x in zip(env.get_agent_id(h), acts):
                held[(g, int(i))] = int(x)
        env.step()
        env.clear_dead()
