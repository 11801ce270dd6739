"""The slot-ordered observation (magent_b200_get_observation_slots) restated from the row-ordered one, and helpers to
check an engine against it.

Slot (a, s) of a group holds, bit for bit, the view record and feature row env_get_observation (or
magent_b200_get_observation_f16) writes for row slot_row[a, s], and all zeros (+0.0) when the slot is vacant.  The
restatement gathers the engine's own row-ordered observation through its get_slots map; tests/slots_common.py pins that
map to the sequence of calls.
"""
import ctypes

import numpy as np

import slots_common as sc


def _uint(half):
    return np.uint16 if half else np.uint32


def _float(half):
    return np.float16 if half else np.float32


def row_observation(env, h, half):
    """(view, feature) of the group in row order, as copies"""
    if env.get_num(h) == 0:
        g = env._hv(h)
        return (np.zeros((0,) + env.view_space[g], _float(half)), np.zeros((0,) + env.feature_space[g], _float(half)))
    v, f = env.get_observation_f16(h) if half else env.get_observation(h)
    return v.copy(), f.copy()


def gather(rows, slot_row):
    """rows [n, ...] into [A, S, ...]: rows[slot_row[a, s]], zeros where slot_row is -1"""
    out = np.zeros(slot_row.shape + rows.shape[1:], rows.dtype)
    occ = slot_row >= 0
    out[occ] = rows[slot_row[occ]]
    return out


def expected(env, h, half):
    """(view, feature) of the group in slot order, restated from the row-ordered observation and get_slots"""
    v, f = row_observation(env, h, half)
    _row_slot, slot_row = sc.read_host(env, h)
    return gather(v, slot_row), gather(f, slot_row), slot_row


def call_host(env, h, half):
    """the call into fresh host arrays of the ABI's shapes: (return code, view, feature)"""
    g = env._hv(h)
    lead = (env.num_arenas, env.get_slot_space(h))
    view = np.empty(lead + env.view_space[g], _float(half))
    feat = np.empty(lead + env.feature_space[g], _float(half))
    bufs = (ctypes.c_void_p * 2)(view.ctypes.data, feat.ctypes.data)
    rc = env._lib.magent_b200_get_observation_slots(env.game, g, bufs, 1 if half else 0)
    return rc, view, feat


def compare(got_v, got_f, want_v, want_f, slot_row, half, what=""):
    """bit equality, and every vacant slot +0.0 throughout"""
    u = _uint(half)
    assert got_v.shape == want_v.shape and got_f.shape == want_f.shape, "%s: shapes %s %s, want %s %s" % (
        what, got_v.shape, got_f.shape, want_v.shape, want_f.shape)
    gv, gf = np.ascontiguousarray(got_v).view(u), np.ascontiguousarray(got_f).view(u)
    vac = slot_row < 0
    assert not gv[vac].any() and not gf[vac].any(), "%s: a vacant slot is not all +0.0" % what
    bad = np.argwhere((gv != want_v.view(u)).reshape(gv.shape[:2] + (int(np.prod(gv.shape[2:])),)).any(-1))
    assert len(bad) == 0, "%s: %d slots differ from their row's record, first (arena, slot) %s, row %d" % (
        what, len(bad), tuple(bad[0]), slot_row[tuple(bad[0])])
    bad = np.argwhere((gf != want_f.view(u)).any(-1))
    assert len(bad) == 0, "%s: %d feature rows differ, first (arena, slot) %s" % (what, len(bad), tuple(bad[0]))
    return int((~vac).sum())


def check(env, h, half, get=None, what=""):
    """the call (get(env, h, half) -> (view, feature); default call_host) against the restatement; returns the
    occupied slots compared"""
    want_v, want_f, slot_row = expected(env, h, half)
    if get is None:
        rc, got_v, got_f = call_host(env, h, half)
        assert rc == 0, env._lib.magent_b200_last_error()
    else:
        got_v, got_f = get(env, h, half)
    return compare(got_v, got_f, want_v, want_f, slot_row, half, what)


def slots_reader(half, get=None, tally=None):
    """a `read` hook for slots_common.check/play_*: checks the slot-ordered observation of the group first, then reads
    the slots.  tally: a list that collects the occupied slots compared"""
    def read(env, h):
        n = check(env, h, half, get)
        if tally is not None:
            tally.append(n)
        return sc.read_host(env, h)
    return read
