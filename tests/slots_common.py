"""The stable agent slots (magent_b200_get_slots) restated from the sequence of calls, and helpers to check an engine
against it.

An agent's slot is the number of agents of its group placed into its arena before it since the arena's last reset.
`Slots` follows an environment through reset, add_agents (any method, select_arena included), snapshot_arenas,
free_snapshot and restore_arenas, and rebuilds every slot from what those calls leave behind: the ids each add_agents
created (read with get_agent_id and get_arena_nums; ids are handed out in placement order, so new ids sort into new
slots), the per-arena state at every snapshot and the restore sources.  From that it derives the two maps:
row_slot[r] = a * S + slot for every row r, slot_row[a, slot] = r or -1.  S(g) is recomputed where the engine may change
it (reset, add_agents, snapshot_arenas, free_snapshot): the largest slot count over the arenas now and over every live
snapshot's arenas.  It shares no code with magent_b200/csrc/slot_phases.h.
"""
import copy

import numpy as np


def rows_by_arena(env, h):
    """(ids, arena of every row) of one group"""
    ids = env.get_agent_id(h).astype(np.int64).copy()
    nums = env.get_arena_nums(h)
    return ids, np.repeat(np.arange(len(nums)), nums)


class Slots:
    """the restatement of one environment's slots; wrap every placement, snapshot and restore call through it"""

    def __init__(self, env, placed=True):
        """placed: the environment was just reset and populated; its agents take slots in id order"""
        self.env = env
        self.hs = env.get_handles()
        self.A = env.num_arenas
        self.state = [[dict() for _ in self.hs] for _ in range(self.A)]      # [a][g]: id -> slot
        self.count = [[0 for _ in self.hs] for _ in range(self.A)]           # [a][g]: slots handed out
        self.snaps = {}
        if placed:
            self._take_new()
        self._space()

    # ---- the calls
    def reset(self):
        self.env.reset()
        self.state = [[dict() for _ in self.hs] for _ in range(self.A)]
        self.count = [[0 for _ in self.hs] for _ in range(self.A)]
        self._space()

    def add(self, h, **kw):
        self.env.add_agents(h, **kw)
        self._take_new()
        self._space()

    def snapshot(self):
        pool = self.env.snapshot_arenas()
        self.snaps[pool] = (copy.deepcopy(self.state), copy.deepcopy(self.count))
        self._space()
        return pool

    def free(self, pool):
        self.env.free_snapshot(pool)
        del self.snaps[pool]
        self._space()

    def restore(self, pool, src=None, keep_rng=False, src_kind="host"):
        """src: a list (None: the arenas whose last step reported done take their own snapshot arena)"""
        chosen = list(src) if src is not None else [a if d else -1 for a, d in enumerate(self.env.get_arena_done())]
        if src is None:
            self.env.restore_arenas(pool, None, keep_rng=keep_rng)
        elif src_kind == "host":
            self.env.restore_arenas(pool, np.asarray(src, dtype=np.int32), keep_rng=keep_rng)
        else:
            import torch
            self.env.restore_arenas(pool, torch.tensor(src, dtype=torch.int32, device="cuda"), keep_rng=keep_rng)
        self.restored(pool, chosen)

    def restored(self, pool, chosen):
        """book a restore the engine made with sources `chosen` (e.g. inside a graph)"""
        st, ct = self.snaps[pool]
        for a, s in enumerate(chosen):
            if 0 <= s < self.A:
                self.state[a] = copy.deepcopy(st[s])
                self.count[a] = list(ct[s])

    def _take_new(self):
        for g, h in enumerate(self.hs):
            ids, arena = rows_by_arena(self.env, h)
            for a in range(self.A):
                known = self.state[a][g]
                for i in np.sort(ids[arena == a]):
                    if int(i) not in known:
                        known[int(i)] = self.count[a][g]
                        self.count[a][g] += 1

    def _space(self):
        S = [max(self.count[a][g] for a in range(self.A)) for g in range(len(self.hs))]
        for _st, ct in self.snaps.values():
            S = [max(S[g], max(ct[a][g] for a in range(self.A))) for g in range(len(self.hs))]
        self.S = S

    # ---- the maps
    def expected(self, g):
        """(row_slot int32 [n], slot_row int32 [A, S]) of group g as the rows are now"""
        ids, arena = rows_by_arena(self.env, self.hs[g])
        S = self.S[g]
        row_slot = np.empty(len(ids), np.int32)
        slot_row = np.full((self.A, S), -1, np.int32)
        for r, (i, a) in enumerate(zip(ids, arena)):
            s = self.state[a][g][int(i)]
            assert s < S
            row_slot[r] = a * S + s
            slot_row[a, s] = r
        return row_slot, slot_row


def read_host(env, h):
    r, m = env.get_slots(h)
    return r.copy(), m.copy()


def check_invariants(env, h, row_slot, slot_row, culled):
    """slot_row inverts row_slot; slots increase with ids inside an (arena, group); after clear_dead the occupied slots
    are exactly the live agents'"""
    ids, arena = rows_by_arena(env, h)
    n = len(ids)
    S = slot_row.shape[1]
    assert (row_slot[:n] >= 0).all()
    np.testing.assert_array_equal(slot_row.reshape(-1)[row_slot[:n]], np.arange(n))
    assert (slot_row >= 0).sum() == n
    if culled:
        assert env.get_alive(h)[:n].all()
    if n == 0:
        return
    assert (row_slot[:n] // S == arena).all()
    for a in range(slot_row.shape[0]):
        sel = arena == a
        order = np.argsort(ids[sel])
        assert (np.diff((row_slot[:n][sel] % S)[order]) > 0).all()


def check(tr, what="", read=None, culled=True):
    """every group's maps as the engine gives them (read(env, h) -> (row_slot, slot_row), default get_slots) against the
    restatement, plus the invariants.  Returns the slots compared."""
    env = tr.env
    read = read or read_host
    n_checked = 0
    for g, h in enumerate(tr.hs):
        assert env.get_slot_space(h) == tr.S[g], "%s group %d: slot space %d, want %d" % (
            what, g, env.get_slot_space(h), tr.S[g])
        want_r, want_m = tr.expected(g)
        got_r, got_m = read(env, h)
        n = len(want_r)
        assert got_r.dtype == np.int32 and got_m.dtype == np.int32 and got_m.shape == want_m.shape, (
            "%s group %d: %s %s, want %s" % (what, g, got_r.dtype, got_m.shape, want_m.shape))
        assert (got_r[n:] == -1).all(), "%s group %d: rows past the count are not -1" % (what, g)
        bad = np.flatnonzero(got_r[:n] != want_r)
        assert len(bad) == 0, "%s group %d: %d wrong row_slot entries, first row %d: %d, want %d" % (
            what, g, len(bad), bad[0], got_r[bad[0]], want_r[bad[0]])
        bad = np.argwhere(got_m != want_m)
        assert len(bad) == 0, "%s group %d: %d wrong slot_row entries, first %s: %d, want %d" % (
            what, g, len(bad), bad[0], got_m[tuple(bad[0])], want_m[tuple(bad[0])])
        check_invariants(env, h, got_r, got_m, culled)
        n_checked += want_m.size
    return n_checked


def add_somewhere(tr, arena, seed, n=8):
    """custom placements of every group at random cells of one arena (select_arena; -1: every arena): the ones on
    occupied cells are refused, so this never fails on a crowded map, and the restatement sees which ids were made"""
    env = tr.env
    H, W, _C = env.get_state_space()
    rs = np.random.RandomState(seed)
    env.select_arena(arena)
    for h in tr.hs:
        pos = [[int(rs.randint(1, W - 1)), int(rs.randint(1, H - 1)), 3] for _ in range(n)]
        tr.add(h, method="custom", pos=pos)
    env.select_arena(-1)


def random_step(env, rs, cull=True):
    for h in env.get_handles():
        env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
    env.step()
    if cull:
        env.clear_dead()


def play_irregular(tr, steps, seed, read=None):
    """the misbehaving caller of fuzz_common.trace_irregular, batched: clear_dead skipped on some steps, agents of a
    random group added mid-episode into every arena or (select_arena) into one.  The maps after every call that moves
    rows.  Returns the slots compared."""
    env = tr.env
    rs = np.random.RandomState(seed ^ 0x51075)
    n = 0
    culled = True
    for t in range(steps):
        random_step(env, rs, cull=False)
        culled = False
        n += check(tr, "irregular step %d" % t, read, culled=False)
        if rs.rand() < 0.65:
            env.clear_dead()
            culled = True
            n += check(tr, "irregular step %d after clear_dead" % t, read)
        if rs.rand() < 0.3:
            arena = int(rs.randint(-1, tr.A))
            H, W, _C = env.get_state_space()
            pos = [[int(rs.randint(1, W - 1)), int(rs.randint(1, H - 1)), int(rs.randint(0, 4))] for _ in range(6)]
            env.select_arena(arena)
            tr.add(tr.hs[int(rs.randint(0, len(tr.hs)))], method="custom", pos=pos)
            env.select_arena(-1)
            n += check(tr, "irregular step %d after adding into arena %d" % (t, arena), read, culled=culled)
    return n


def play_and_check(tr, steps, seed, read=None):
    """random play: the maps after every step (before its clear_dead, while dead agents keep their rows) and after every
    clear_dead.  Returns the slots compared."""
    rs = np.random.RandomState(seed)
    n = check(tr, "start", read)
    for t in range(steps):
        random_step(tr.env, rs, cull=False)
        n += check(tr, "step %d before clear_dead" % t, read, culled=False)
        tr.env.clear_dead()
        n += check(tr, "step %d" % t, read)
    return n
