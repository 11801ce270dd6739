"""The built-in scripted opponents (magent_b200_rule_actions, _get_rule_actions, _get_rule_actions_slots) restated in
plain numpy, and helpers to check an engine against it.

The restatement is built from the other restatements and the public getters only; it shares no code with
magent_b200/csrc/rule_phases.h.  For agent i of group g against group t:
  rush  1. the legal attack (action_mask_common) whose aimed cell holds an agent of t other than i with the lowest hp
           (get_info "hp"); ties to the lowest action
        2. else, when neighbours_common lists a first neighbour of t for i, its (vy, vx) cell mapped to the map by
           global_state_common.window_cells is c; the legal move whose moved footprint has the smallest squared box
           distance to c; ties to the lowest action
        3. else action_mask_common.restate_draws for the call random_legal_actions(seed) would be next
  flee  2 with the largest distance, else 3
A dead agent and an agent without a legal action take 0.
"""
import numpy as np

import action_mask_common as am
import global_state_common as gs
import mean_action_common as ma
import neighbours_common as nc

RUSH, FLEE = 0, 1
POLICIES = {RUSH: "rush", FLEE: "flee"}
# which step decided an agent's action (expected's second result)
NONE, ATTACK, APPROACH, FALLBACK = 0, 1, 2, 3


class State:
    """what the restatement needs of one moment of a game: every group's mask, hp, positions and headings"""

    def __init__(self, env, dirs=None, tracker=None, call=1, steps=0):
        self.env, self.dirs, self.call, self.steps = env, dirs, call, steps
        self.hs = env.get_handles()
        self.types = [am.GroupType(env, g) for g in range(len(self.hs))]
        self.masks = am.expected_masks(env, dirs, tracker)
        self.pos = [env.get_pos(h).astype(np.int64) for h in self.hs]
        self.alive = [env.get_alive(h).copy() for h in self.hs]
        self.hp = [env._info(h, b"hp", np.empty((env.get_num(h),), dtype=np.float32)).copy() for h in self.hs]
        self.offs = [np.concatenate([[0], np.cumsum(env.get_arena_nums(h))]) for h in self.hs]

    def heading(self, g):
        n = len(self.pos[g])
        return np.full(n, am.DIR_NORTH) if self.dirs is None else np.where(self.dirs[g] < 0, am.DIR_NORTH, self.dirs[g])

    def expected(self, g, t, policy, seed):
        """(actions int32 [n], step int [n]) of group g against t in ABI order"""
        env, T, mask = self.env, self.types[g], self.masks[g]
        n = len(mask)
        acts, step = np.zeros(n, np.int32), np.full(n, NONE)
        draws = am.restate_draws(mask, seed, self.call, self.steps)
        idx, rel, _count = nc.expected(env, g, t, 1, self.dirs)
        dg = self.heading(g)
        X, Y, _m = gs.window_cells(env, g, self.pos[g], None if self.dirs is None else dg)
        H, W, _C = env.get_state_space()
        _m, _x1, _y1, tw, tl = gs.view_geometry(env, t)
        for a in range(env.num_arenas):
            st = slice(self.offs[t][a], self.offs[t][a + 1])
            owner = ma.owner_grid(H, W, self.pos[t][st], self.alive[t][st],
                                  None if self.dirs is None else self.dirs[t][st], tw, tl)
            for i in range(self.offs[g][a], self.offs[g][a + 1]):
                if not self.alive[g][i] or not mask[i].any():
                    continue
                x, y = (int(v) for v in self.pos[g][i])
                d = int(dg[i])
                if policy == RUSH:
                    best = None
                    for q, (ax, ay) in enumerate(T.attacks):
                        k = T.attack_base + q
                        if not mask[i, k]:
                            continue
                        ox, oy = T.w // 2 + ax, T.l // 2 + ay
                        if T.turn_mode:
                            rx, ry = am._real(d, T.w, T.l)
                            dx, dy = am._rot(d, ox, oy)
                            tx, ty = x + rx + dx, y + ry + dy
                        else:
                            tx, ty = x + ox, y + oy
                        j = int(owner[ty, tx])
                        if j < 0 or (t == g and self.offs[t][a] + j == i):
                            continue
                        v = self.hp[t][self.offs[t][a] + j]
                        if best is None or v < best[1]:
                            best = (k, v)
                    if best is not None:
                        acts[i], step[i] = best[0], ATTACK
                        continue
                if idx[i, 0] >= 0:
                    vy, vx = (int(v) for v in rel[i, 0])
                    cx, cy = int(X[i, vy, vx]), int(Y[i, vy, vx])
                    bw, bh = am._dims(d, T.w, T.l)
                    best = None
                    for k, (mx, my) in enumerate(T.moves):
                        if not mask[i, k]:
                            continue
                        dx, dy = am._rot(d, mx, my) if T.turn_mode else (mx, my)
                        nx, ny = x + dx, y + dy
                        ex = max(nx - cx, cx - (nx + bw - 1), 0)
                        ey = max(ny - cy, cy - (ny + bh - 1), 0)
                        dd = ex * ex + ey * ey
                        if best is None or (dd > best[1] if policy == FLEE else dd < best[1]):
                            best = (k, dd)
                    if best is not None:
                        acts[i], step[i] = best[0], APPROACH
                        continue
                acts[i], step[i] = draws[i], FALLBACK
        return acts, step

    def known(self, g):
        """rows whose heading is known (all but never-absorbing absorbers in turn_mode)"""
        return np.ones(len(self.pos[g]), dtype=bool) if self.dirs is None else self.dirs[g] >= 0


def read_rows(env, h, t, policy, seed):
    return env.get_rule_actions(h, t, POLICIES[policy], seed).copy()


def check(state, pairs, seed, read=None, what=""):
    """every (g, t, policy) of `pairs` as the engine gives it (read(env, h, target_handle, policy, seed), default
    get_rule_actions) against the restatement; returns the count of agents each step decided, [NONE .. FALLBACK]"""
    read = read or read_rows
    hs = state.hs
    steps = np.zeros(4, np.int64)
    for g, t, policy in pairs:
        want, step = state.expected(g, t, policy, seed)
        got = read(state.env, hs[g], hs[t], policy, seed)
        assert got.dtype == np.int32 and got.shape == want.shape, "%s %d vs %d %s: %s %s, want %s" % (
            what, g, t, POLICIES[policy], got.dtype, got.shape, want.shape)
        known = state.known(g)
        bad = np.flatnonzero((got != want) & known)
        assert len(bad) == 0, "%s group %d vs %d %s: %d wrong of %d, first row %d: engine %d, want %d (step %d)" % (
            what, g, t, POLICIES[policy], len(bad), len(want), bad[0], got[bad[0]], want[bad[0]], step[bad[0]])
        steps += np.bincount(step[known], minlength=4)
    return steps


def all_pairs(env):
    G = len(env.get_handles())
    return [(g, t, p) for g in range(G) for t in range(G) for p in (RUSH, FLEE)]


def play_and_check(env, steps, seed, tmpdir=None, uncull_every=0, read=None, pairs=None):
    """random play, with random_legal_actions for group 0 every other step (so the fallback's call number moves); every
    pair against the restatement after every clear_dead and (uncull_every) also between a step and its clear_dead.
    Returns the count of agents each step decided."""
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmpdir))
    tracker = am.AbsorbTracker(env)
    rs = np.random.RandomState(seed)
    pairs = all_pairs(env) if pairs is None else pairs
    hs = env.get_handles()
    calls = 0
    total = np.zeros(4, np.int64)
    for t in range(steps):
        tracker.update()
        dirs = am.frame_headings(env, str(tmpdir)) if turn else None
        total += check(State(env, dirs, tracker, calls + 1, t), pairs, seed + t, read, "step %d" % t)
        uncull = uncull_every and t % uncull_every == uncull_every - 1 and not turn
        for h in hs:
            env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
        if t % 2:
            env.set_random_legal_actions(hs[0], 100 + t)
            calls += 1
        env.step()
        if uncull:
            tracker.update()
            total += check(State(env, None, tracker, calls + 1, t + 1), pairs, seed, read,
                           "step %d before clear_dead" % t)
        env.clear_dead()
    return total
