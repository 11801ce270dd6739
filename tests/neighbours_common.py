"""The nearest visible neighbours (magent_b200_get_neighbours) restated in plain numpy, and helpers to check an engine
against it.

The neighbour sets are those of the mean neighbour action: the owner grid of mean_action_common, the windows of
global_state_common.window_cells.  On top of them, every view cell (vx, vy) of observer i's window has the key
(d2, vy * view_w + vx), compared in that order, where d2 is the squared Euclidean distance, in map cells, from the map
cell it shows to i's footprint [x, x + bw) x [y, y + bh) (body dimensions rotated by i's heading; 0 on the footprint).  A
neighbour's key is the smallest key among the in-range, on-board cells of i's window that its body covers.  Row i lists
the first k neighbours by key: idx = the neighbour's row in group `of`'s ABI concatenation, rel = (vy, vx) of its
smallest-key cell; unused slots hold -1.  count = |N(i)|.  It shares no code with magent_b200/csrc/nbr_phases.h.
"""
import numpy as np

import action_mask_common as am
import global_state_common as gs
import mean_action_common as ma


def _keys(env, g, pos, dirs, X, Y):
    """int64 [n, vh, vw]: d2 * (vh * vw) + vy * vw + vx of every view cell of every observer"""
    _m, _x1, _y1, w, l = gs.view_geometry(env, g)
    n, vh, vw = X.shape
    x = pos[:, 0].reshape(-1, 1, 1)
    y = pos[:, 1].reshape(-1, 1, 1)
    if dirs is None:
        bw = np.full((n, 1, 1), w, np.int64)
        bh = np.full((n, 1, 1), l, np.int64)
    else:
        upright = np.isin(np.where(dirs < 0, gs.DIR_NORTH, dirs), (gs.DIR_NORTH, gs.DIR_SOUTH)).reshape(-1, 1, 1)
        bw = np.where(upright, w, l).astype(np.int64)
        bh = np.where(upright, l, w).astype(np.int64)
    ex = np.maximum(np.maximum(x - X, X - (x + bw - 1)), 0)
    ey = np.maximum(np.maximum(y - Y, Y - (y + bh - 1)), 0)
    cell = np.arange(vh * vw, dtype=np.int64).reshape(1, vh, vw)
    return (ex * ex + ey * ey) * (vh * vw) + cell


def arena_rows(env, g, of, k, pos_g, alive_g, dirs_g, owner, base):
    """(idx [n, k], rel [n, k, 2], count [n], keys [n, k]) of one arena's observers; base: the arena's offset in `of`'s
    concatenation.  keys holds the neighbours' keys (-1 in unused slots)."""
    n = len(pos_g)
    idx = np.full((n, k), -1, np.int32)
    rel = np.full((n, k, 2), -1, np.int32)
    keys = np.full((n, k), -1, np.int64)
    count = np.zeros((n,), np.int32)
    if n == 0:
        return idx, rel, count, keys
    H, W = owner.shape
    nbrs, X, Y, on = ma.neighbour_sets(env, g, of, pos_g, alive_g, dirs_g, owner)
    seen = np.where(on, owner[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)], -1)
    key = _keys(env, g, pos_g.astype(np.int64), dirs_g, X, Y)
    vw = X.shape[2]
    for i in range(n):
        if not alive_g[i]:
            continue
        hit = seen[i] >= 0
        if of == g:
            hit &= seen[i] != i
        js, ks = seen[i][hit], key[i][hit]
        order = np.argsort(ks, kind="stable")
        js, ks = js[order], ks[order]
        _u, first = np.unique(js, return_index=True)
        first = np.sort(first)                      # each neighbour at its smallest key, in key order
        assert len(first) == len(nbrs[i])
        count[i] = len(first)
        take = first[:k]
        m = len(take)
        idx[i, :m] = base + js[take]
        cell = ks[take] % (X.shape[1] * vw)
        rel[i, :m, 0] = cell // vw
        rel[i, :m, 1] = cell % vw
        keys[i, :m] = ks[take]
    return idx, rel, count, keys


def expected(env, g, of, k, dirs=None, with_keys=False):
    """the restated (idx, rel, count) of group g over group `of`, every arena, in ABI order.  dirs: per-group headings of
    a single-arena turn_mode game."""
    hs = env.get_handles()
    H, W, _C = env.get_state_space()
    _m, _x1, _y1, w, l = gs.view_geometry(env, of)
    pos = [env.get_pos(hs[q]).astype(np.int64) for q in (g, of)]
    alive = [env.get_alive(hs[q]).copy() for q in (g, of)]
    offs = [np.concatenate([[0], np.cumsum(env.get_arena_nums(hs[q]))]) for q in (g, of)]
    assert dirs is None or env.num_arenas == 1
    parts = []
    for a in range(env.num_arenas):
        sg, so = (slice(offs[q][a], offs[q][a + 1]) for q in (0, 1))
        owner = ma.owner_grid(H, W, pos[1][so], alive[1][so], None if dirs is None else dirs[of], w, l)
        parts.append(arena_rows(env, g, of, k, pos[0][sg], alive[0][sg], None if dirs is None else dirs[g], owner,
                                offs[1][a]))
    out = tuple(np.concatenate([p[q] for p in parts]) for q in range(4))
    return out if with_keys else out[:3]


def read_host(env, h, of, k):
    return tuple(x.copy() for x in env.get_neighbours(h, k, of))


def check_rows(env, k, dirs=None, what="", read=None, pairs=None):
    """every (group, of) pair's rows as the engine gives them (read(env, h, of, k), default get_neighbours) against the
    restatement; rows of observers with an unknown heading are not compared.  Returns the neighbours listed."""
    hs = env.get_handles()
    pairs = [(g, o) for g in range(len(hs)) for o in range(len(hs))] if pairs is None else pairs
    read = read or read_host
    listed = 0
    for g, o in pairs:
        want = expected(env, g, o, k, dirs)
        got = read(env, hs[g], hs[o], k)
        for name, x, y in zip(("idx", "rel", "count"), got, want):
            assert x.dtype == np.int32 and x.shape == y.shape, "%s %d over %d %s: %s %s, want %s" % (
                what, g, o, name, x.dtype, x.shape, y.shape)
        known = np.ones(len(want[2]), dtype=bool) if dirs is None else dirs[g] >= 0
        bad = np.flatnonzero(((got[0] != want[0]).any(axis=1) | (got[1] != want[1]).any(axis=(1, 2)) |
                              (got[2] != want[2])) & known)
        assert len(bad) == 0, "%s k=%d group %d over %d: %d wrong rows, first %d: idx %s rel %s count %d, want %s %s %d" % (
            what, k, g, o, len(bad), bad[0], got[0][bad[0]], got[1][bad[0]].tolist(), got[2][bad[0]],
            want[0][bad[0]], want[1][bad[0]].tolist(), want[2][bad[0]])
        listed += int((want[0][known] >= 0).sum())
    return listed


def play_and_check(env, steps, seed, ks, tmpdir=None, uncull_every=0, read=None):
    """random play; every (group, of) pair at every k in ks against the restatement after every clear_dead and
    (uncull_every) also between a step and its clear_dead, while dead agents still hold rows.  Returns the neighbours
    listed."""
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmpdir))
    rs = np.random.RandomState(seed)
    listed = 0
    for t in range(steps):
        dirs = am.frame_headings(env, str(tmpdir)) if turn else None
        for k in ks:
            listed += check_rows(env, k, dirs, "step %d" % t, read)
        uncull = uncull_every and t % uncull_every == uncull_every - 1 and not turn
        am.random_step(env, rs, cull=not uncull)
        if uncull:
            for k in ks:
                listed += check_rows(env, k, None, "step %d before clear_dead" % t, read)
            for h in env.get_handles():
                dead = ~env.get_alive(h)
                idx, rel, c = (read or read_host)(env, h, h, ks[0])
                assert (idx[dead] == -1).all() and (rel[dead] == -1).all() and not c[dead].any()
            env.clear_dead()
    return listed
