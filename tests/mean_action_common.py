"""The mean neighbour action (magent_b200_get_mean_action) restated in plain numpy, and helpers to check an engine
against it.

`expected` rebuilds, for every agent i of group g, its neighbours N(i) in group `of` and its (mean, count) row from what
the public getters give: positions and alive flags (dead agents have left the map), the body size of `of` (rotated by the
heading in turn_mode), the view windows of global_state_common.window_cells and the actions the agents hold, read back
through the one-hot of their feature rows.  It shares no code with magent_b200/csrc/nbr_phases.h.  Headings in turn_mode
are read from a replay frame (action_mask_common.frame_headings).

The definition: N(i) = the distinct agents j != i of `of` in i's arena that cover some on-board, in-range cell of i's view
window; count[i] = |N(i)|; mean[i][k] = float32(#{j in N(i): act_j == k}) / float32(count[i]) for k < n_action(of), where
an action outside [0, n_action) is in no bin; a row without neighbours, or of a dead agent, is all zero with count 0.
"""
import numpy as np

import action_mask_common as am
import global_state_common as gs

DIR_NORTH = gs.DIR_NORTH


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def held_actions(env, h):
    """the action every agent of the group holds, -1 where its one-hot is empty (an agent added since the last step, or
    an action id outside [0, n_action))"""
    acts = am.last_actions(env, h)
    na = env.get_action_space(h)[0]
    feat = env.get_observation(h)[1]
    emb = feat.shape[1] - na - 1 - (2 if env.config.config_dict.get("minimap_mode", False) else 0) \
        - (2 if env.config.config_dict.get("goal_mode", False) else 0)
    hot = feat[np.arange(len(acts)), emb + acts] == 1.0 if len(acts) else np.zeros((0,), dtype=bool)
    return np.where(hot, acts, -1).astype(np.int64)


def owner_grid(H, W, pos, alive, dirs, w, l):
    """index of the live agent covering each cell, -1 where none"""
    owner = np.full((H, W), -1, np.int64)
    for j, (x, y) in enumerate(pos):
        if not alive[j]:
            continue
        d = DIR_NORTH if dirs is None or dirs[j] < 0 else int(dirs[j])
        bw, bh = (w, l) if d in (gs.DIR_NORTH, gs.DIR_SOUTH) else (l, w)
        assert (owner[y:y + bh, x:x + bw] == -1).all(), "two agents of one group on one cell"
        owner[y:y + bh, x:x + bw] = j
    return owner


def neighbour_sets(env, g, of, pos, alive, dirs, owner):
    """per observer of group g (one arena): the sorted indices N(i) in group `of`; also the window (X, Y, on) with
    on = in range and on the board"""
    H, W = owner.shape
    if len(pos) == 0:
        return [], None, None, None
    X, Y, mask = gs.window_cells(env, g, pos.astype(np.int64), dirs)
    on = (X >= 0) & (X < W) & (Y >= 0) & (Y < H) & mask.reshape((1,) + mask.shape)
    seen = np.where(on, owner[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)], -1)
    out = []
    for i in range(len(pos)):
        ids = np.unique(seen[i]) if alive[i] else np.zeros((0,), np.int64)
        ids = ids[ids >= 0]
        if of == g:
            ids = ids[ids != i]
        out.append(ids)
    return out, X, Y, on


def rows(nbrs, acts, na):
    """(mean float32 [n, na], count int32 [n]) from the neighbour sets and the actions of `of`"""
    mean = np.zeros((len(nbrs), na), np.float32)
    count = np.zeros((len(nbrs),), np.int32)
    for i, ids in enumerate(nbrs):
        count[i] = len(ids)
        if len(ids):
            a = acts[ids]
            a = a[(a >= 0) & (a < na)]
            mean[i] = np.bincount(a, minlength=na).astype(np.float32) / np.float32(len(ids))
    return mean, count


def expected(env, g, of, dirs=None, acts=None):
    """the restated (mean, count) of group g over group `of`, every arena, in ABI order.  dirs: per-group headings of a
    single-arena turn_mode game; acts: the actions group `of` holds (default: held_actions)."""
    hs = env.get_handles()
    H, W, _C = env.get_state_space()
    _m, _x1, _y1, w, l = gs.view_geometry(env, of)
    na = env.get_action_space(hs[of])[0]
    pos = [env.get_pos(hs[k]).astype(np.int64) for k in (g, of)]
    alive = [env.get_alive(hs[k]).copy() for k in (g, of)]
    acts = held_actions(env, hs[of]) if acts is None else np.asarray(acts, np.int64)
    offs = [np.concatenate([[0], np.cumsum(env.get_arena_nums(hs[k]))]) for k in (g, of)]
    assert dirs is None or env.num_arenas == 1
    means, counts = [], []
    for a in range(env.num_arenas):
        sg, so = (slice(offs[k][a], offs[k][a + 1]) for k in (0, 1))
        owner = owner_grid(H, W, pos[1][so], alive[1][so], None if dirs is None else dirs[of], w, l)
        nbrs = neighbour_sets(env, g, of, pos[0][sg], alive[0][sg], None if dirs is None else dirs[g], owner)[0]
        m, c = rows(nbrs, acts[so], na)
        means.append(m)
        counts.append(c)
    return np.concatenate(means), np.concatenate(counts)


def check_means(env, dirs=None, what="", read=None, acts=None, pairs=None):
    """every (group, of) pair's rows as the engine gives them (read(env, h, of), default get_mean_action) against the
    restatement, bit for bit; rows of observers with an unknown heading are not compared.  Returns the number of
    neighbours counted."""
    hs = env.get_handles()
    pairs = [(g, o) for g in range(len(hs)) for o in range(len(hs))] if pairs is None else pairs
    total = 0
    for g, o in pairs:
        want_m, want_c = expected(env, g, o, dirs, None if acts is None else acts[o])
        got_m, got_c = read(env, hs[g], hs[o]) if read else env.get_mean_action(hs[g], hs[o])
        assert got_m.dtype == np.float32 and got_m.shape == want_m.shape, "%s %d over %d: %s %s, want %s" % (
            what, g, o, got_m.dtype, got_m.shape, want_m.shape)
        assert got_c.dtype == np.int32 and got_c.shape == want_c.shape
        known = np.ones(len(want_c), dtype=bool) if dirs is None else dirs[g] >= 0
        bad = np.flatnonzero(((got_c != want_c) | (_bits(got_m) != _bits(want_m)).any(axis=1)) & known)
        assert len(bad) == 0, "%s group %d over %d: %d wrong rows, first %d: count %d want %d, mean %s want %s" % (
            what, g, o, len(bad), bad[0], got_c[bad[0]], want_c[bad[0]], got_m[bad[0]], want_m[bad[0]])
        total += int(want_c[known].sum())
    return total


def play_and_check(env, steps, seed, tmpdir=None, uncull_every=0, read=None):
    """random play; every (group, of) pair against the restatement after every clear_dead and (uncull_every) also
    between a step and its clear_dead, while dead agents still hold rows.  Returns the neighbours counted."""
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmpdir))
    rs = np.random.RandomState(seed)
    total = 0
    for t in range(steps):
        dirs = am.frame_headings(env, str(tmpdir)) if turn else None
        total += check_means(env, dirs, "step %d" % t, read)
        uncull = uncull_every and t % uncull_every == uncull_every - 1 and not turn
        am.random_step(env, rs, cull=not uncull)
        if uncull:
            total += check_means(env, None, "step %d before clear_dead" % t, read)
            for g, h in enumerate(env.get_handles()):
                dead = ~env.get_alive(h)
                m, c = (read(env, h, h) if read else env.get_mean_action(h))
                assert not m[dead].any() and not c[dead].any()
            env.clear_dead()
    return total
