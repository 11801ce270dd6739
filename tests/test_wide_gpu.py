"""The edge configurations of tests/wide_common.py on the CUDA library: large views and wide action spaces, where the
side-output kernels' shared memory reaches the H100's limits (49152 bytes per block by default, 232448 with the opt-in).

Inside the limits every output is held bit for bit to the compiled reference (observations through host dense, host
wire, device float32 and float16 buffers, row- and slot-ordered) and to the numpy restatements (mean action, neighbours,
mask, legal draws, row- and slot-ordered, through host and device pointers), and the mask rows go into unaligned
tensors with guard bytes.  One step past a ceiling every call is refused with -1 and a message that names the bytes,
writes nothing, and the engine steps on.

The mask of 167 actions is the first that needs the dynamic shared-memory opt-in: 256 rows of 167 bytes + 16 bytes of
alignment shift + the kernel's 6400 bytes of static shared memory are 49168 bytes, past the 49152 a block gets without
it.  A budget that counted sizeof(EngineDev) (6368 bytes) instead of the kernel's static size passed that launch
without the opt-in, and the launch failed."""
import os

import numpy as np
import pytest

import action_mask_common as am
import mean_action_common as ma
import nbr_slots_common as ns
import neighbours_common as nb
import obs_slots_common as osc
import parity_common as pc
import slot_loop_common as lc
import wide_common as wc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

RENDERED = sorted(n for n, e in wc.EDGES.items() if e[2].get("render") == "optin")
SERVED = sorted(n for n, e in wc.EDGES.items() if e[2].get("mean") != "past")
REFUSED = sorted(n for n, e in wc.EDGES.items() if e[2].get("mean") == "past")


def checker():
    lib = next((p for p in (pc.REF_LIB, pc.PORT_LIB) if os.path.exists(p)), None)
    if lib is None:
        pytest.skip("neither the compiled reference nor the oracle port is built")
    return lib


def device_reads(env):
    """read hooks for the restatement checks: the host call, with the device call asserted bit for bit equal to it"""
    def mean(env, h, o):
        hm, hc = (x.copy() for x in env.get_mean_action(h, o))
        dm, dc = env.get_mean_action_torch(h, o)
        assert np.array_equal(dm.cpu().numpy().view(np.uint32), hm.view(np.uint32)) and np.array_equal(dc.cpu().numpy(), hc)
        return hm, hc

    def nbr(env, h, o, k):
        hi, hr, hn = (x.copy() for x in env.get_neighbours(h, k, o))
        di, dr, dn = env.get_neighbours_torch(h, k, o)
        assert np.array_equal(di.cpu().numpy(), hi) and np.array_equal(dr.cpu().numpy(), hr)
        assert np.array_equal(dn.cpu().numpy(), hn)
        return hi, hr, hn

    def mask(env, h):
        host = env.get_action_mask(h).copy()
        np.testing.assert_array_equal(env.get_action_mask_torch(h).cpu().numpy(), host)
        return host
    return mean, nbr, mask


def slot_outputs_on_the_device(env, what):
    """the slot-ordered mean, neighbours and mask through device pointers equal the host ones (checked against the row
    calls by nbr_slots_common.check_all and slot_loop_common.check_mask)"""
    for h, o in ns.pairs(env):
        hm, hc = (x.copy() for x in env.get_mean_action_slots(h, o))
        dm, dc = env.get_mean_action_slots_torch(h, o)
        assert np.array_equal(dm.cpu().numpy().view(np.uint32), hm.view(np.uint32)), what + ": device mean slots"
        assert np.array_equal(dc.cpu().numpy(), hc), what
        for k in (1, 32):
            hi, hr, hn = (x.copy() for x in env.get_neighbours_slots(h, k, o))
            di, dr, dn = env.get_neighbours_slots_torch(h, k, o)
            assert np.array_equal(di.cpu().numpy(), hi) and np.array_equal(dr.cpu().numpy(), hr), what
            assert np.array_equal(dn.cpu().numpy(), hn), what
    for h in env.get_handles():
        np.testing.assert_array_equal(env.get_action_mask_slots_torch(h).cpu().numpy(),
                                      env.get_action_mask_slots(h), err_msg=what + ": device mask slots")


def restatements(env, tmp_path, held, what):
    turn = bool(env.config.config_dict.get("turn_mode", False))
    dirs = am.frame_headings(env, str(tmp_path)) if turn else None
    mean, nbr, mask = device_reads(env)
    total = ma.check_means(env, dirs, what, read=mean, acts=wc.acts_by_id(env, held))
    for k in (1, 32):
        nb.check_rows(env, k, dirs, "%s k %d" % (what, k), read=nbr)
    am.check_masks(env, dirs, what=what, read=mask)
    ns.check_all(env, ks=(1, 32), what=what)
    for h in env.get_handles():
        lc.check_mask(env, h, what=what)
    slot_outputs_on_the_device(env, what)
    return total


@pytest.mark.parametrize("name", RENDERED + ["wire_r38"])
def test_observations_through_every_path_equal_the_reference(name):
    """host dense, host wire (forced: past the wire kernel's limit it must fall back to dense records), device float32
    and float16, and the slot-ordered render, against the reference's observations"""
    import torch
    want = wc.state_trace(wc.make(checker(), name, seed=3), 3, 5, True)
    paths = ("wire",) if name == "wire_r38" else ("dense", "wire", "auto")
    for path in paths:
        env = wc.make(pc.CUDA_LIB, name, seed=3, _host_path=path)
        wc.check_edge(env, name)
        pc.compare_traces(want, wc.state_trace(env, 3, 5, True), "%s host %s" % (name, path))
    if name == "wire_r38":
        return                                     # the render cannot hold this view: only the wire path serves it
    env = wc.make(pc.CUDA_LIB, name, seed=3)
    rs = np.random.RandomState(2)
    for t in range(3):
        for h in env.get_handles():
            v, f = (x.copy() for x in env.get_observation(h))
            dv, df = env.get_observation_torch(h)
            assert np.array_equal(dv.cpu().numpy().view(np.uint32), v.view(np.uint32)), "%s step %d device view" % (name, t)
            assert np.array_equal(df.cpu().numpy().view(np.uint32), f.view(np.uint32)), "%s step %d device feature" % (name, t)
            hv, hf = env.get_observation_torch(h, dtype=torch.float16)
            assert torch.equal(hv, dv.half()) and torch.equal(hf, df.half()), "%s step %d float16" % (name, t)
            for half in (False, True):
                osc.check(env, h, half, what="%s step %d slots half %d" % (name, t, half))
                osc.check(env, h, half, get=lambda e, h, half: tuple(
                    x.cpu().numpy() for x in e.get_observation_slots_torch(h, dtype=torch.float16 if half else None)),
                    what="%s step %d device slots half %d" % (name, t, half))
        wc.random_step(env, rs)


@pytest.mark.parametrize("name", SERVED)
def test_side_outputs_equal_the_restatements(name, tmp_path):
    env = wc.make(pc.CUDA_LIB, name, seed=4)
    wc.check_edge(env, name)
    if env.config.config_dict.get("turn_mode", False):
        env.set_render_dir(str(tmp_path))
    rs = np.random.RandomState(6)
    held = {}
    listed = 0
    for t in range(2):
        wc.random_step(env, rs, held)
        listed += restatements(env, tmp_path, held, "%s step %d" % (name, t))
    assert listed > 0


def guarded_refusals(env, what, mean, mask):
    """every mean-action call (mean) and every mask call (mask) refused with -1, a message naming the shared memory,
    and its guard values untouched, through host and device pointers"""
    import torch
    L = env._lib
    for h, o in (ns.pairs(env) if mean else ()):
        g, og = env._hv(h), env._hv(o)
        na = env.get_action_space(o)[0]
        n, S = env.get_num(h), env.get_slot_space(h)
        for slots, rows in ((False, n), (True, env.num_arenas * S)):
            fn = L.magent_b200_get_mean_action_slots if slots else L.magent_b200_get_mean_action
            mean = np.full((rows + 1, na), -7.0, np.float32)
            count = np.full((rows + 1,), -7, np.int32)
            L.magent_b200_last_error()
            assert fn(env.game, g, og, mean.ctypes.data, count.ctypes.data) == -1, what
            msg = L.magent_b200_last_error().decode()
            assert "shared memory" in msg and "get_mean_action" in msg, msg
            assert (mean == -7.0).all() and (count == -7).all(), what + ": a refused call wrote its host buffers"
            dmean = torch.full((rows + 1, na), -7.0, device="cuda")
            dcount = torch.full((rows + 1,), -7, dtype=torch.int32, device="cuda")
            assert fn(env.game, g, og, dmean.data_ptr(), dcount.data_ptr()) == -1, what
            torch.cuda.synchronize()
            assert bool((dmean == -7.0).all()) and bool((dcount == -7).all()), what + ": a refused call wrote device buffers"
        with pytest.raises(RuntimeError, match="shared memory"):
            env.get_mean_action(h, o)
        with pytest.raises(RuntimeError, match="shared memory"):
            env.get_mean_action_slots_torch(h, o)
    if not mask:
        return
    for h in env.get_handles():
        g, na = env._hv(h), env.get_action_space(h)[0]
        for slots, rows in ((False, env.get_num(h)), (True, env.num_arenas * env.get_slot_space(h))):
            fn = L.magent_b200_get_action_mask_slots if slots else L.magent_b200_get_action_mask
            buf = np.full((rows + 1, na), 7, np.uint8)
            assert fn(env.game, g, buf.ctypes.data) == -1, what
            msg = L.magent_b200_last_error().decode()
            assert "shared memory" in msg and ("%d actions" % na) in msg, msg
            assert (buf == 7).all(), what + ": a refused mask call wrote its host buffer"
            dbuf = torch.full((rows + 1, na), 7, dtype=torch.uint8, device="cuda")
            assert fn(env.game, g, dbuf.data_ptr()) == -1, what
            torch.cuda.synchronize()
            assert bool((dbuf == 7).all()), what + ": a refused mask call wrote its device buffer"


@pytest.mark.parametrize("name", REFUSED)
def test_past_the_mean_action_ceiling_every_call_is_refused(name, tmp_path):
    """refused with nothing written; the engine steps on and the calls inside their limits still serve"""
    env = wc.make(pc.CUDA_LIB, name, seed=5)
    wc.check_edge(env, name)
    if env.config.config_dict.get("turn_mode", False):
        env.set_render_dir(str(tmp_path))
    rs = np.random.RandomState(3)
    held = {}
    for t in range(2):
        guarded_refusals(env, "%s step %d" % (name, t), True, False)
        wc.random_step(env, rs, held)
    turn = bool(env.config.config_dict.get("turn_mode", False))
    dirs = am.frame_headings(env, str(tmp_path)) if turn else None
    _mean, nbr, mask = device_reads(env)
    am.check_masks(env, dirs, what=name, read=mask)
    if wc.EDGES[name][2].get("nbr", "in") == "in":
        nb.check_rows(env, 32, dirs, name, read=nbr)
    else:
        with pytest.raises(RuntimeError, match="too large to order its cells"):
            env.get_neighbours(env.get_handles()[0], 1)


@pytest.mark.parametrize("na", sorted(wc.MASK_SPACES))
def test_wide_action_spaces(na, tmp_path):
    """the step against the reference; then the mask (row, slot, host, device, unaligned tensors with guard bytes), the
    legal draws and the mean action against the restatements; past the opt-in limit every mask call is refused"""
    import torch
    steps = 2 if na > 800 else 3
    obs = na <= wc.HEADER_MAX_ACTIONS
    pc.compare_traces(wc.state_trace(wc.make_mask(checker(), na, seed=2), steps, 9, obs),
                      wc.state_trace(wc.make_mask(pc.CUDA_LIB, na, seed=2), steps, 9, obs), "%d actions" % na)
    env = wc.make_mask(pc.CUDA_LIB, na, seed=3)
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmp_path))
    past = wc.side(wc.STATIC_ENGINE + 256 * na + 16, "mask") == "past"
    rs = np.random.RandomState(na)
    held = {}
    calls = 0
    for t in range(steps):
        what = "%d actions step %d" % (na, t)
        if past:
            guarded_refusals(env, what, False, True)
            with pytest.raises(RuntimeError, match="shared memory"):
                env.get_action_mask_torch(env.get_handles()[0])
        else:
            dirs = am.frame_headings(env, str(tmp_path)) if turn and obs else None
            mean, _nbr, mask = device_reads(env)
            am.check_masks(env, dirs, what=what, read=mask)
            ma.check_means(env, dirs, what, read=mean, acts=wc.acts_by_id(env, held))
            for h in env.get_handles():
                lc.check_mask(env, h, what=what)
                np.testing.assert_array_equal(env.get_action_mask_slots_torch(h).cpu().numpy(),
                                              env.get_action_mask_slots(h), err_msg=what)
                want = env.get_action_mask(h).copy()
                n = len(want)
                for lead in range(16):
                    big = torch.full((lead + (n + 3) * na + 40,), 7, dtype=torch.uint8, device="cuda")
                    out = big[lead:lead + (n + 3) * na].view(n + 3, na)
                    np.testing.assert_array_equal(env.get_action_mask_torch(h, out=out).cpu().numpy(), want)
                    assert bool((big[:lead] == 7).all()) and bool((big[lead + n * na:] == 7).all()), \
                        "%s offset %d: bytes outside the rows were written" % (what, lead)
        if not obs:                                    # no feature rows to read the drawn actions back from
            wc.random_step(env, rs, held)
            continue
        for g, h in enumerate(env.get_handles()):
            mask = None if past else env.get_action_mask(h).copy()
            env.set_random_legal_actions(h, 11 + t)
            calls += 1
            acts = am.last_actions(env, h)
            if not past:
                np.testing.assert_array_equal(acts, am.restate_draws(mask, 11 + t, calls, t), err_msg=what)
            for i, x in zip(env.get_agent_id(h), acts):
                held[(g, int(i))] = int(x)
        env.step()
        env.clear_dead()
