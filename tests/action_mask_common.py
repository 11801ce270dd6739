"""The legal-action mask (magent_b200_get_action_mask) restated in plain numpy, and helpers to check an engine against it.

`restate_masks` rebuilds the mask of every group of one arena from what the public getters give -- positions, alive
flags, the wall / food planes, group sizes -- and the agent type tables of the config (body, speed, attack range,
attack_in_group, can_absorb).  It shares no code with magent_b200/csrc/mask_phases.h.  Two things no getter reports are
passed in by the caller: headings in turn_mode (read from a replay frame, frame_headings below) and which
absorbers have already absorbed (AbsorbTracker below).

The definition, per agent i and action k, "taken alone on the state as it is now":
  move    the target footprint is inside the board by the reference's test (x < 0 or y < 0 or x + w >= W or y + h >= H is
          out), and every cell is empty or the mover's own; or else the first other agent in the footprint, scanning x
          outer / y inner and passing over walls and food, is a can_absorb type that has not absorbed yet
  turn    the rotated footprint is inside the board and empty or the agent's own
  attack  the aimed cell is on the board and holds an agent of another group, of the own group with attack_in_group, or
          food
  a dead agent has no legal action; an absorbed absorber has no legal move.
"""
import math

import numpy as np

DIR_EAST, DIR_SOUTH, DIR_WEST, DIR_NORTH = 0, 1, 2, 3


# ------------------------------------------------------------------ type tables (Range.h:104-190, AgentType.cc:86-117)
def circle_deltas(radius, inner, parity):
    r, eps = float(np.float32(radius)), 1e-8
    width = 2 * int(r + eps) + parity
    center = int(r)
    if width % 2 != parity:
        width += 1
    delta = 0.5 if parity == 0 else 0.0
    out = []
    for i in range(width):
        for j in range(width):
            dis = math.sqrt(abs(j - center + delta) ** 2 + abs(i - center + delta) ** 2)
            if dis < r + eps and dis > float(np.float32(inner)) - eps:
                out.append((j - center, i - center))
    return out


def sector_deltas(angle, radius, parity):
    kpi, eps = 3.1415926536, 0.00001
    a, r = float(np.float32(angle)), float(np.float32(radius))
    h = int(r + 0.5)
    w = int(2 * r * math.sin(a / 2 * (kpi / 180)) + 0.5)
    if w % 2 != parity:
        w -= 1
    w = max(w, 0)
    lim = math.tan(a / 2 * kpi / 180) + eps
    out = []
    for i in range(h):
        for j in range(w):
            dx, dy = abs(j - (w - 1) / 2.0), abs(float(h - i))
            if math.sqrt(dx * dx + dy * dy) < r + 0.2 + eps and dx / dy < lim:
                out.append((j - w // 2, i - h))
    return out


class GroupType:
    def __init__(self, env, g):
        attrs = env.config.agent_type_dict[env.config.groups[g]]
        self.turn_mode = bool(env.config.config_dict.get("turn_mode", False))
        self.w, self.l = int(attrs.get("width", 1)), int(attrs.get("length", 1))
        self.moves = circle_deltas(attrs.get("speed", 1.0), 0.0, 1)
        ar = attrs.get("attack_range")
        radius, angle = (0.0, 0.0) if ar is None else (ar.radius, ar.angle)
        parity = self.w % 2
        self.attacks = circle_deltas(radius, self.w / 2.0, parity) if angle >= 180 else sector_deltas(angle, radius, parity)
        self.attack_in_group = bool(attrs.get("attack_in_group", False))
        self.can_absorb = bool(attrs.get("can_absorb", False))
        self.n_move = len(self.moves)
        self.attack_base = self.n_move + (2 if self.turn_mode else 0)
        self.n_action = self.attack_base + len(self.attacks)


def _rot(d, rx, ry):
    return {DIR_NORTH: (rx, ry), DIR_SOUTH: (-rx, -ry), DIR_WEST: (ry, -rx), DIR_EAST: (-ry, rx)}[d]


def _real(d, w, l):
    return {DIR_NORTH: (0, 0), DIR_SOUTH: (w - 1, l - 1), DIR_WEST: (0, w - 1), DIR_EAST: (l - 1, 0)}[d]


def _dims(d, w, l):
    return (w, l) if d in (DIR_NORTH, DIR_SOUTH) else (l, w)


# ------------------------------------------------------------------ the restatement
def restate_masks(types, wall, food, groups):
    """types: [GroupType]; wall, food: bool [H, W]; groups: per group dict(pos int [n, 2], alive bool [n], dirs int [n] or
    None, absorbed bool [n] or None).  Returns per group a bool [n, n_action] array."""
    H, W = wall.shape
    owner_g = np.full((H, W), -1, np.int64)
    owner_i = np.full((H, W), -1, np.int64)

    def heading(g, i):
        d = groups[g].get("dirs")
        return DIR_NORTH if d is None or d[i] < 0 else int(d[i])   # unknown: a 1x1 absorber, whose row is not compared

    for g, (t, grp) in enumerate(zip(types, groups)):
        for i, (x, y) in enumerate(grp["pos"]):
            if not grp["alive"][i]:
                continue
            bw, bh = _dims(heading(g, i), t.w, t.l)
            assert (owner_g[y:y + bh, x:x + bw] == -1).all(), "two agents on one cell"
            owner_g[y:y + bh, x:x + bw] = g
            owner_i[y:y + bh, x:x + bw] = i

    def footprint(g, i, nx, ny, bw, bh):
        """(in board, blank or self, first other agent) of a target footprint"""
        if nx < 0 or ny < 0 or nx + bw >= W or ny + bh >= H:
            return False, False, None
        blank, hit = True, None
        for bx in range(bw):
            for by in range(bh):
                cx, cy = nx + bx, ny + by
                other = owner_g[cy, cx] >= 0 and not (owner_g[cy, cx] == g and owner_i[cy, cx] == i)
                if wall[cy, cx] or food[cy, cx] or other:
                    blank = False
                if other and hit is None:
                    hit = (int(owner_g[cy, cx]), int(owner_i[cy, cx]))
        return True, blank, hit

    out = []
    for g, (t, grp) in enumerate(zip(types, groups)):
        n = len(grp["pos"])
        mask = np.zeros((n, t.n_action), dtype=bool)
        for i in range(n):
            if not grp["alive"][i]:
                continue
            x, y = (int(v) for v in grp["pos"][i])
            d = heading(g, i)
            bw, bh = _dims(d, t.w, t.l)
            absorbed = grp.get("absorbed") is not None and bool(grp["absorbed"][i])
            for k, (mx, my) in enumerate(t.moves):
                if absorbed:
                    break
                dx, dy = _rot(d, mx, my) if t.turn_mode else (mx, my)
                inb, blank, hit = footprint(g, i, x + dx, y + dy, bw, bh)
                if blank:
                    mask[i, k] = True
                elif inb and hit is not None and types[hit[0]].can_absorb:
                    ab = groups[hit[0]].get("absorbed")
                    mask[i, k] = not (ab is not None and bool(ab[hit[1]]))
            if t.turn_mode:
                for q in (0, 1):
                    k = t.n_move + q
                    nd = (d + 2 * k - 1 + 4) % 4            # the caller's quirk: wise = 2 * act - 1 with the raw action
                    rx, ry = _real(d, t.w, t.l)
                    qx, qy = _real(nd, t.w, t.l)
                    _inb, blank, _hit = footprint(g, i, x + rx - qx, y + ry - qy, bh, bw)
                    mask[i, k] = blank
            for q, (ax, ay) in enumerate(t.attacks):
                ox, oy = t.w // 2 + ax, t.l // 2 + ay
                if t.turn_mode:
                    rx, ry = _real(d, t.w, t.l)
                    dx, dy = _rot(d, ox, oy)
                    tx, ty = x + rx + dx, y + ry + dy
                else:
                    tx, ty = x + ox, y + oy
                if tx < 0 or tx >= W or ty < 0 or ty >= H:
                    continue
                if food[ty, tx]:
                    mask[i, t.attack_base + q] = True
                elif owner_g[ty, tx] >= 0:
                    mask[i, t.attack_base + q] = owner_g[ty, tx] != g or t.attack_in_group
        out.append(mask)
    return out


# ------------------------------------------------------------------ reading an engine
class AbsorbTracker:
    """Which absorbers have absorbed: no getter says, but an absorber's hp only ever rises when it swallows a mover (it
    doubles; absorbing types here neither recover, kill nor eat), so "hp rose since the last look" is sticky per id."""

    def __init__(self, env):
        self.env = env
        self.types = [GroupType(env, g) for g in range(len(env.get_handles()))]
        self.last, self.done = {}, set()
        self.update()

    def _hp(self, h):
        return self.env._info(h, b"hp", np.empty((self.env.get_num(h),), dtype=np.float32))

    def update(self):
        for g, h in enumerate(self.env.get_handles()):
            if not self.types[g].can_absorb:
                continue
            ids, hp, nums = self.env.get_agent_id(h), self._hp(h), self.env.get_arena_nums(h)
            arena = np.repeat(np.arange(len(nums)), nums)
            for a, i, v in zip(arena, ids, hp):
                key = (g, int(a), int(i))
                if key in self.last and v > self.last[key]:
                    self.done.add(key)
                self.last[key] = float(v)

    def forget(self):
        """after a reset or restore: hp histories no longer apply"""
        self.last, self.done = {}, set()
        self.update()

    def absorbed(self, g, h):
        if not self.types[g].can_absorb:
            return None
        ids, nums = self.env.get_agent_id(h), self.env.get_arena_nums(h)
        arena = np.repeat(np.arange(len(nums)), nums)
        return np.array([(g, int(a), int(i)) in self.done for a, i in zip(arena, ids)], dtype=bool)


def frame_headings(env, render_dir):
    """per group: the heading of every agent in group order, from the replay frame env_render writes (matched by id).
    The frame leaves out absorbers that have not absorbed yet: their heading is -1, unknown."""
    import os
    env.render()
    files = sorted((f for f in os.listdir(render_dir) if f.startswith("video_")), key=lambda f: int(f[6:-4]))
    lines = open(os.path.join(render_dir, files[-1])).read().splitlines()
    start = max(i for i, s in enumerate(lines) if s.startswith("F "))
    seen = {}
    for s in lines[start + 1:start + 1 + int(lines[start].split()[1])]:
        _id, _hp, angle, _x, _y, g = (int(v) for v in s.split())
        seen[(g, _id)] = angle // 90
    return [np.array([seen.get((g, int(i)), -1) for i in env.get_agent_id(h)], dtype=np.int64)
            for g, h in enumerate(env.get_handles())]


def expected_masks(env, dirs=None, tracker=None):
    """the restated mask of every group of `env` (any number of arenas), in ABI order.  dirs: per-group headings of a
    single-arena turn_mode game."""
    hs = env.get_handles()
    types = [GroupType(env, g) for g in range(len(hs))]
    food_mode = bool(env.config.config_dict.get("food_mode", False))
    state = env.get_global_state().copy()
    A = state.shape[0]
    assert dirs is None or A == 1
    pos = [env.get_pos(h).astype(np.int64) for h in hs]
    alive = [env.get_alive(h).copy() for h in hs]
    absorbed = [None if tracker is None else tracker.absorbed(g, h) for g, h in enumerate(hs)]
    offs = [np.concatenate([[0], np.cumsum(env.get_arena_nums(h))]) for h in hs]
    out = [[] for _ in hs]
    for a in range(A):
        wall = state[a, :, :, 0] != 0
        food = state[a, :, :, 1] != 0 if food_mode else np.zeros_like(wall)
        groups = []
        for g in range(len(hs)):
            s = slice(offs[g][a], offs[g][a + 1])
            groups.append(dict(pos=pos[g][s], alive=alive[g][s], dirs=None if dirs is None else dirs[g],
                               absorbed=None if absorbed[g] is None else absorbed[g][s]))
        for g, m in enumerate(restate_masks(types, wall, food, groups)):
            out[g].append(m)
    return [np.concatenate(m, axis=0) for m in out]


def check_masks(env, dirs=None, tracker=None, what="", read=None):
    """every group's mask as the engine gives it (read(env, h), default get_action_mask) against the restatement;
    returns the masks"""
    want = expected_masks(env, dirs, tracker)
    got = []
    for g, h in enumerate(env.get_handles()):
        m = (read(env, h) if read else env.get_action_mask(h)).copy()
        assert m.dtype == np.bool_ and m.shape == want[g].shape, "%s group %d: %s %s, want %s" % (what, g, m.dtype, m.shape, want[g].shape)
        known = np.ones(len(m), dtype=bool) if dirs is None else dirs[g] >= 0
        bad = np.argwhere((m != want[g]) & known[:, None])
        assert len(bad) == 0, "%s group %d: %d wrong bits, first (agent, action) %s: engine %d" % (
            what, g, len(bad), tuple(bad[0]), m[tuple(bad[0])])
        got.append(m)
    return got


def random_step(env, rs, cull=True):
    for h in env.get_handles():
        env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
    env.step()
    if cull:
        env.clear_dead()


def play_and_check(env, steps, seed, tmpdir=None, uncull_every=0, read=None):
    """random play; the mask against the restatement after every clear_dead, and (uncull_every) also between a step and
    its clear_dead, when dead agents still hold rows.  Returns (bits checked, bits set)."""
    turn = bool(env.config.config_dict.get("turn_mode", False))
    if turn:
        env.set_render_dir(str(tmpdir))
    tracker = AbsorbTracker(env)
    rs = np.random.RandomState(seed)
    bits = ones = 0
    for t in range(steps):
        tracker.update()
        masks = check_masks(env, frame_headings(env, str(tmpdir)) if turn else None, tracker, "step %d" % t, read)
        bits += sum(m.size for m in masks)
        ones += sum(int(m.sum()) for m in masks)
        uncull = uncull_every and t % uncull_every == uncull_every - 1 and not turn
        random_step(env, rs, cull=not uncull)
        if uncull:
            tracker.update()
            for g, m in enumerate(check_masks(env, None, tracker, "step %d before clear_dead" % t, read)):
                dead = ~env.get_alive(env.get_handles()[g])
                assert not m[dead].any()
            env.clear_dead()
    return bits, ones


# ------------------------------------------------------------------ the draw of magent_b200_random_legal_actions
M64 = (1 << 64) - 1


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def restate_draws(mask, seed, call, steps):
    """the actions random_legal_actions(seed) sets for a group whose mask is `mask`: `call` = how many random_actions /
    random_legal_actions calls the game has served, this one included; `steps` = env_step calls so far.  Agent o with L
    legal actions takes the r-th in ascending order, r = (splitmix64(s ^ o * 0xD1342543DE82EF95) >> 33) % L with
    s = seed * 0x9E3779B97F4A7C15 + call + steps * 0xA24BAED4963EE407 (all mod 2^64); action 0 when L = 0."""
    s = (seed * 0x9E3779B97F4A7C15 + call + steps * 0xA24BAED4963EE407) & M64
    acts = np.zeros(len(mask), dtype=np.int32)
    for o, row in enumerate(mask):
        legal = np.flatnonzero(row)
        if len(legal):
            acts[o] = legal[(_splitmix64(s ^ ((o * 0xD1342543DE82EF95) & M64)) >> 33) % len(legal)]
    return acts


def last_actions(env, h):
    """the action every agent of the group holds, read back through the one-hot of its feature row"""
    g = env._hv(h)
    na = env.get_action_space(h)[0]
    feat = env.get_observation(h)[1]
    emb = feat.shape[1] - na - 1 - (2 if env.config.config_dict.get("minimap_mode", False) else 0) \
        - (2 if env.config.config_dict.get("goal_mode", False) else 0)
    return np.argmax(feat[:, emb:emb + na], axis=1).astype(np.int32)
