"""The slot-ordered step loop (magent_b200_set_action_slots, _get_reward_slots, _get_action_mask_slots) restated from
the row-ordered calls, and a twin driver to check an engine against it.

set_action_slots(act) must leave the engine bit for bit where set_action(act.flat[row_slot]) leaves it, row_slot being
the engine's own get_slots map.  `Twin` drives two engines made alike, one through set_action_slots (vacant slots full of
garbage), the other through set_action in rows, and compares everything the engines serve after every step and cull.
The reward, status and mask restatements gather the row-ordered get_reward, get_alive and get_action_mask through
get_slots."""
import ctypes

import numpy as np

import slots_common as sc


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view("u%d" % a.dtype.itemsize)


def state(env):
    """everything the twins must agree on: per-arena done flags and, per group, ids, positions, alive, hp, rewards,
    observations and the mean action"""
    out = {"done": env.get_arena_done().copy()}
    for g, h in enumerate(env.get_handles()):
        n = env.get_num(h)
        out["id", g] = env.get_agent_id(h).copy()
        out["pos", g] = env.get_pos(h).copy()
        out["alive", g] = env.get_alive(h).copy()
        out["hp", g] = env._info(h, b"hp", np.empty((n,), np.float32)).copy()
        out["reward", g] = env.get_reward(h).copy()
        if n:
            v, f = env.get_observation(h)
            out["view", g], out["feature", g] = v.copy(), f.copy()
            m, c = env.get_mean_action(h)
            out["mean", g], out["count", g] = m.copy(), c.copy()
    return out


def compare_states(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(_bits(a[k]), _bits(b[k])), "%s: %s differs" % (what, k)


def slot_actions(env, h, rs):
    """random legal-range actions (num_arenas, S) int32 with arbitrary ints, out-of-range ids included, in the slots
    that are vacant now"""
    _row_slot, slot_row = sc.read_host(env, h)
    na = env.get_action_space(h)[0]
    act = rs.randint(0, na, size=slot_row.shape).astype(np.int32)
    vac = slot_row < 0
    act[vac] = rs.randint(-2 ** 31, 2 ** 31 - 1, size=int(vac.sum()), dtype=np.int64).astype(np.int32)
    return act


def rows_of(env, h, act):
    """the row-ordered actions set_action_slots(act) stands for: act.flat[row_slot]"""
    row_slot, _slot_row = sc.read_host(env, h)
    return np.ascontiguousarray(act.reshape(-1)[row_slot])


def set_host(env, h, act):
    env.set_action_slots(h, act)


class Twin:
    """two engines made alike: `s` driven in slot order through set(env, h, act) (default: host arrays), `r` in rows"""

    def __init__(self, make, lib, set_slots=set_host):
        self.s, self.r = make(lib), make(lib)
        self.hs = self.s.get_handles()
        self.set_slots = set_slots
        self.checked = 0

    def both(self, fn):
        return fn(self.s), fn(self.r)

    def check(self, what):
        compare_states(state(self.s), state(self.r), what)
        self.checked += 1

    def act(self, rs, order=None, mix=False):
        """actions for every group, in `order`; mix: a group's slot engine may instead get set_action in rows, or both
        kinds in either order (the last one counts)"""
        order = list(range(len(self.hs))) if order is None else order
        for g in order:
            h = self.hs[g]
            act = slot_actions(self.r, h, rs)
            rows = rows_of(self.r, h, act)
            kind = int(rs.randint(0, 4)) if mix else 0
            if kind == 1:                               # rows only
                self.s.set_action(h, rows)
            elif kind == 2:                             # other rows first, overwritten by the slots
                self.s.set_action(h, rs.randint(0, 3, size=len(rows)).astype(np.int32))
                self.set_slots(self.s, h, act)
            elif kind == 3:                             # other slots first, overwritten by the rows
                self.set_slots(self.s, h, slot_actions(self.r, h, rs))
                self.s.set_action(h, rows)
            else:
                self.set_slots(self.s, h, act)
            self.r.set_action(h, rows)

    def step(self, rs, t, cull=True, order=None, mix=False):
        self.act(rs, order, mix)
        self.both(lambda e: e.step())
        self.check("step %d" % t)
        if cull:
            self.both(lambda e: e.clear_dead())
            self.check("step %d after clear_dead" % t)


# ---------------------------------------------------------------- reward, status and mask restated
def expected_reward(env, h):
    """(reward float32 [A, S], status uint8 [A, S], slot_row) gathered from get_reward and get_alive"""
    _row_slot, slot_row = sc.read_host(env, h)
    occ = slot_row >= 0
    reward = np.zeros(slot_row.shape, np.float32)
    status = np.zeros(slot_row.shape, np.uint8)
    if occ.any():
        rows = slot_row[occ]
        reward[occ] = env.get_reward(h)[rows]
        status[occ] = np.where(env.get_alive(h)[rows], 1, 2)
    return reward, status, slot_row


def expected_mask(env, h):
    """uint8 [A, S, n_action] gathered from get_action_mask"""
    _row_slot, slot_row = sc.read_host(env, h)
    na = env.get_action_space(h)[0]
    out = np.zeros(slot_row.shape + (na,), np.uint8)
    occ = slot_row >= 0
    if occ.any():
        out[occ] = env.get_action_mask(h).view(np.uint8)[slot_row[occ]]
    return out


def check_reward(env, h, got=None, what=""):
    """got: (reward, status) as numpy arrays (default: the host call); returns the occupied slots compared"""
    want_r, want_s, slot_row = expected_reward(env, h)
    got_r, got_s = got if got is not None else env.get_reward_slots(h)
    assert got_r.dtype == np.float32 and got_s.dtype == np.uint8 and got_r.shape == want_r.shape == got_s.shape, what
    assert np.array_equal(_bits(got_r), _bits(want_r)), "%s: rewards differ from the rows' (or a vacant slot is not +0.0)" % what
    assert np.array_equal(got_s, want_s), "%s: status differs" % what
    return int((slot_row >= 0).sum())


def check_mask(env, h, got=None, what=""):
    want = expected_mask(env, h)
    got = got if got is not None else env.get_action_mask_slots(h)
    got = np.ascontiguousarray(got).view(np.uint8)
    assert got.shape == want.shape, "%s: shape %s, want %s" % (what, got.shape, want.shape)
    bad = np.argwhere((got != want).any(-1))
    assert len(bad) == 0, "%s: %d slots' mask rows differ, first (arena, slot) %s" % (what, len(bad), tuple(bad[0]))
    return int(want.any(-1).sum())


def check_outputs(env, tally=None, what=""):
    """reward, status and mask of every group against the restatements"""
    for h in env.get_handles():
        n = check_reward(env, h, what=what)
        check_mask(env, h, what=what)
        if tally is not None:
            tally.append(n)


def call_reward(env, h, reward, status):
    """the raw call with numpy buffers (or None): return code"""
    return env._lib.magent_b200_get_reward_slots(env.game, env._hv(h), None if reward is None else reward.ctypes.data,
                                                 None if status is None else status.ctypes.data)


def call_mask(env, h, mask):
    return env._lib.magent_b200_get_action_mask_slots(env.game, env._hv(h), None if mask is None else mask.ctypes.data)


def call_set(env, h, act):
    ptr = None if act is None else ctypes.c_void_p(act.ctypes.data)
    return env._lib.magent_b200_set_action_slots(env.game, env._hv(h), ptr)
