"""The slot-ordered mean action and neighbours (magent_b200_get_mean_action_slots, _get_neighbours_slots) restated from
the row-ordered calls and get_slots alone.

    mean_s[a, s]     = mean_rows[slot_row[a, s]], a +0.0 row where the slot is vacant; count the same way, 0 where vacant
    idx_s[a, s, r]   = row_slot_of[idx_rows[slot_row[a, s], r]], -1 where the entry is unused or the slot vacant
    rel_s, count_s   = rel_rows, count_rows gathered through slot_row, -1 / 0 where vacant

slot_row is get_slots(group)'s map and row_slot_of get_slots(of)'s.  Floats are compared by their bits."""
import numpy as np

import slots_common as sc


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view("u%d" % a.dtype.itemsize)


def expected_mean(env, h, of):
    """(mean float32 [A, S, n_action(of)], count int32 [A, S])"""
    _row_slot, slot_row = sc.read_host(env, h)
    mean = np.zeros(slot_row.shape + (env.get_action_space(of)[0],), np.float32)
    count = np.zeros(slot_row.shape, np.int32)
    occ = slot_row >= 0
    if occ.any():
        m, c = env.get_mean_action(h, of)
        mean[occ] = m[slot_row[occ]]
        count[occ] = c[slot_row[occ]]
    return mean, count


def expected_neighbours(env, h, of, k):
    """(idx int32 [A, S, k], rel int32 [A, S, k, 2], count int32 [A, S])"""
    _row_slot, slot_row = sc.read_host(env, h)
    row_slot_of, _slot_row_of = sc.read_host(env, of)
    idx = np.full(slot_row.shape + (k,), -1, np.int32)
    rel = np.full(slot_row.shape + (k, 2), -1, np.int32)
    count = np.zeros(slot_row.shape, np.int32)
    occ = slot_row >= 0
    if occ.any():
        i, r, c = (x.copy() for x in env.get_neighbours(h, k, of))
        rows = slot_row[occ]
        used = i[rows]
        idx[occ] = np.append(row_slot_of, -1)[np.where(used >= 0, used, -1)]        # -1 stays -1
        rel[occ] = r[rows]
        count[occ] = c[rows]
    return idx, rel, count


def check_mean(env, h, of, got=None, what=""):
    """got: (mean, count) as numpy arrays, count possibly None (default: the host call).  Returns the slots with
    neighbours."""
    want_m, want_c = expected_mean(env, h, of)
    got_m, got_c = got if got is not None else env.get_mean_action_slots(h, of)
    assert got_m.dtype == np.float32 and got_m.shape == want_m.shape, "%s: mean %s %s" % (what, got_m.dtype, got_m.shape)
    bad = np.argwhere((_bits(got_m) != _bits(want_m)).any(-1))
    assert len(bad) == 0, "%s: %d slots' mean rows differ (or a vacant row is not +0.0), first (arena, slot) %s" % (
        what, len(bad), tuple(bad[0]))
    if got_c is not None:
        assert got_c.dtype == np.int32 and np.array_equal(got_c, want_c), "%s: count differs" % what
    return int((want_c > 0).sum())


def check_neighbours(env, h, of, k, got=None, what=""):
    """got: (idx, rel, count) as numpy arrays, rel and count possibly None (default: the host call).  Returns the listed
    neighbours compared."""
    want_i, want_r, want_c = expected_neighbours(env, h, of, k)
    got_i, got_r, got_c = got if got is not None else env.get_neighbours_slots(h, k, of)
    assert got_i.dtype == np.int32 and got_i.shape == want_i.shape, "%s: idx %s %s" % (what, got_i.dtype, got_i.shape)
    bad = np.argwhere((got_i != want_i).any(-1))
    assert len(bad) == 0, "%s: %d slots' idx rows differ, first (arena, slot) %s: %s, want %s" % (
        what, len(bad), tuple(bad[0]), got_i[tuple(bad[0])], want_i[tuple(bad[0])])
    if got_r is not None:
        assert got_r.shape == want_r.shape and np.array_equal(got_r, want_r), "%s: rel differs" % what
    if got_c is not None:
        assert np.array_equal(got_c, want_c), "%s: count differs" % what
    return int((want_i >= 0).sum())


def pairs(env):
    """every (group, of) pair of handles: of == group and of != group"""
    hs = env.get_handles()
    return [(h, o) for h in hs for o in hs]


def check_all(env, ks=(1, 3, 32), what=""):
    """the mean action and the neighbours of every (group, of) pair and k, through the host calls.  Returns the listed
    neighbours compared."""
    n = 0
    for h, o in pairs(env):
        check_mean(env, h, o, what="%s mean %d of %d" % (what, env._hv(h), env._hv(o)))
        for k in ks:
            n += check_neighbours(env, h, o, k, what="%s neighbours %d of %d k %d" % (what, env._hv(h), env._hv(o), k))
    return n


def call_mean(env, h, of, mean, count):
    """the raw call with numpy buffers (or None): return code"""
    return env._lib.magent_b200_get_mean_action_slots(env.game, env._hv(h), env._hv(of),
                                                      None if mean is None else mean.ctypes.data,
                                                      None if count is None else count.ctypes.data)


def call_neighbours(env, h, of, k, idx, rel, count):
    return env._lib.magent_b200_get_neighbours_slots(env.game, env._hv(h), env._hv(of), k,
                                                     None if idx is None else idx.ctypes.data,
                                                     None if rel is None else rel.ctypes.data,
                                                     None if count is None else count.ctypes.data)
