"""Checks of the global state (magent_b200_get_global_state) against a reference engine in the same state.

The state of one arena is a float32 [H][W][C] image, C = 1 + food_mode + 2 * G: wall, food (food_mode only), then per
group g (absolute order) presence at base + 2g and hp / max_hp at base + 2g + 1, base = 1 + food_mode.  Every such
value must be what the reference's Map::extract_view writes for that map cell into any view that covers it.  So
`check_arena_state` compares the state
  * with every reference observer's view, cell by cell (bit for bit, after mapping the view's observer-relative group
    channels to absolute ones), wherever the view window is in range and on the map, and
  * everywhere, with a restatement from the reference's own getters: walls from walls_info (Map::get_wall lists every
    wall cell, the border included), presence from get_pos and the body size (rotated by the heading in turn_mode).
hp and food are thereby checked at every cell some observer sees, and must be 0 where no agent stands.

The view window of an observer (engine: obs_phases.h obs_compose_cell) needs the view range's mask and offset:
`view_geometry` restates the reference's CircleRange / SectorRange tables (Range.h:104-190, AgentType.cc:86-108).
Headings in turn_mode are only exposed through the reference's replay frames (RenderGenerator.cc:148-167: the
heading as an angle of 90 * Direction), which `headings` reads back.
"""
import math
import os

import numpy as np

DIR_EAST, DIR_SOUTH, DIR_WEST, DIR_NORTH = 0, 1, 2, 3


def _circle_mask(radius, parity):
    r, eps = float(np.float32(radius)), 1e-8
    width = 2 * int(r + eps) + parity
    center = int(r)
    if width % 2 != parity:
        width += 1
    delta = 0.5 if parity == 0 else 0.0
    i, j = np.meshgrid(np.arange(width), np.arange(width), indexing="ij")
    dis = np.sqrt(np.abs(j - center + delta) ** 2 + np.abs(i - center + delta) ** 2)
    return (dis < r + eps) & (dis > -eps), -center, -center


def _sector_mask(angle, radius, parity):
    kpi, eps = 3.1415926536, 0.00001
    a, r = float(np.float32(angle)), float(np.float32(radius))
    h = int(r + 0.5)
    w = int(2 * r * math.sin(a / 2 * (kpi / 180)) + 0.5)
    if w % 2 != parity:
        w -= 1
    w = max(w, 0)
    lim = math.tan(a / 2 * kpi / 180) + eps
    i, j = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    dis_x, dis_y = np.abs(j - (w - 1) / 2.0), np.abs(h - i).astype(np.float64)
    dis = np.sqrt(dis_x ** 2 + dis_y ** 2)
    return (dis < r + 0.2 + eps) & (dis_x / dis_y < lim), -(w // 2), -h


def view_geometry(env, g):
    """(in-range mask [vh, vw], x1, y1, body width, body length) of group g's view"""
    attrs = env.config.agent_type_dict[env.config.groups[g]]
    w, l = int(attrs.get("width", 1)), int(attrs.get("length", 1))
    vr = attrs.get("view_range")
    radius, angle = (1, 360) if vr is None else (vr.radius, vr.angle)          # AgentType defaults (AgentType.cc:20-50)
    mask, x1, y1 = _circle_mask(radius, w % 2) if angle >= 180 else _sector_mask(angle, radius, w % 2)
    return mask, x1, y1, w, l


def _rot(d, rx, ry):
    """displacement in the agent's frame -> map displacement (obs_phases.h dir_rot)"""
    return {DIR_NORTH: (rx, ry), DIR_SOUTH: (-rx, -ry), DIR_WEST: (ry, -rx), DIR_EAST: (-ry, rx)}[d]


def _real(d, w, l):
    """offset of the head corner from the stored top-left corner (obs_phases.h dir_real)"""
    return {DIR_NORTH: (0, 0), DIR_SOUTH: (w - 1, l - 1), DIR_WEST: (0, w - 1), DIR_EAST: (l - 1, 0)}[d]


def window_cells(env, g, pos, dirs=None):
    """map x, y [n, vh, vw] of every view cell of group g's observers at pos [n, 2], and the in-range mask"""
    mask, x1, y1, w, l = view_geometry(env, g)
    vh, vw = mask.shape
    rx = (w // 2 + x1 + np.arange(vw)).reshape(1, 1, vw)
    ry = (l // 2 + y1 + np.arange(vh)).reshape(1, vh, 1)
    ax, ay = pos[:, 0].reshape(-1, 1, 1).astype(np.int64), pos[:, 1].reshape(-1, 1, 1).astype(np.int64)
    if dirs is None:
        return ax + rx + 0 * ry, ay + ry + 0 * rx, mask
    X = np.empty((len(pos), vh, vw), np.int64)
    Y = np.empty_like(X)
    for d in (DIR_EAST, DIR_SOUTH, DIR_WEST, DIR_NORTH):
        sel = dirs == d
        if not sel.any():
            continue
        dx, dy = _rot(d, rx + 0 * ry, ry + 0 * rx)
        ox, oy = _real(d, w, l)
        X[sel] = ax[sel] + ox + dx
        Y[sel] = ay[sel] + oy + dy
    return X, Y, mask


def headings(ref, render_dir):
    """per group: the heading (Direction) of every agent, in group order, from the replay frame env_render writes"""
    ref.render()
    files = sorted((f for f in os.listdir(render_dir) if f.startswith("video_")), key=lambda f: int(f[6:-4]))
    lines = open(os.path.join(render_dir, files[-1])).read().splitlines()
    start = max(i for i, s in enumerate(lines) if s.startswith("F "))
    n = int(lines[start].split()[1])
    G = len(ref.get_handles())
    dirs = [[] for _ in range(G)]
    for s in lines[start + 1:start + 1 + n]:
        _id, _hp, angle, _x, _y, g = (int(v) for v in s.split())
        dirs[g].append(angle // 90)
    return [np.asarray(d, dtype=np.int64) for d in dirs]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def check_arena_state(state, ref, dirs=None, what=""):
    """state: float32 [H, W, C] of one arena; ref: the reference environment in the same state (after clear_dead);
    dirs: per-group headings (turn_mode) or None"""
    H, W, C = state.shape
    cd = ref.config.config_dict
    food, minimap = bool(cd.get("food_mode", False)), bool(cd.get("minimap_mode", False))
    hs = ref.get_handles()
    G = len(hs)
    base, stride = 1 + food, 2 + minimap
    assert C == base + 2 * G, "%s: %d channels" % (what, C)
    # walls everywhere (border included)
    buf = np.zeros((1 + H * W, 2), dtype=np.int32)
    ref._lib.env_get_info(ref.game, -1, b"walls_info", buf.ctypes.data)
    n = int(buf[0, 0])
    wall = np.zeros((H, W), dtype=bool)
    wall[buf[1:1 + n, 1], buf[1:1 + n, 0]] = True
    np.testing.assert_array_equal(_bits(state[..., 0]), _bits(wall), err_msg=what + " wall channel")
    # presence everywhere, from positions and bodies; hp only where an agent stands
    taken = wall.astype(np.int64)
    for g, h in enumerate(hs):
        pos = ref.get_pos(h).astype(np.int64)
        _m, _x1, _y1, w, l = view_geometry(ref, g)
        pres = np.zeros((H, W), dtype=bool)
        for i, (x, y) in enumerate(pos):
            bw, bl = (w, l) if dirs is None or dirs[g][i] in (DIR_NORTH, DIR_SOUTH) else (l, w)
            pres[y:y + bl, x:x + bw] = True
        np.testing.assert_array_equal(_bits(state[..., base + 2 * g]), _bits(pres), err_msg="%s presence g%d" % (what, g))
        assert (state[..., base + 2 * g + 1][~pres] == 0).all(), "%s: hp of group %d where it does not stand" % (what, g)
        taken += pres
    if food:
        taken += state[..., 1] != 0
    assert (taken <= 1).all(), what + ": a cell shows more than one of wall / food / agent"
    # every observer's view
    pairs = [(0, 0)] + ([(1, 1)] if food else [])
    for g, h in enumerate(hs):
        if ref.get_num(h) == 0:
            continue
        pos = ref.get_pos(h)
        view = ref.get_observation(h)[0]
        X, Y, mask = window_cells(ref, g, pos, None if dirs is None else dirs[g])
        assert view.shape[1:3] == mask.shape, "%s: restated view range of group %d has the wrong shape" % (what, g)
        gp = pairs + [(base + ((j - g) % G) * stride + k, base + 2 * j + k) for j in range(G) for k in (0, 1)]
        on = (X >= 0) & (X < W) & (Y >= 0) & (Y < H) & mask.reshape((1,) + mask.shape)
        seen = state[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)]
        for vc, sc in gp:
            np.testing.assert_array_equal(_bits(view[..., vc][on]), _bits(seen[..., sc][on]),
                                          err_msg="%s: view of group %d channel %d vs state channel %d" % (what, g, vc, sc))
            assert (view[..., vc][~mask.reshape((1,) + mask.shape).repeat(len(pos), 0)] == 0).all(), \
                "%s: group %d marks a view cell outside the restated range" % (what, g)


def play_lockstep(make, engine_lib, ref_lib, steps, seed, read_states, tmpdir=None, turn=False):
    """Drive the engine and the reference with the same uniform random actions (after get_observation, as in the
    standard loop).  read_states(engine) returns float32 [A, H, W, C] arrays that must all be equal; arena 0 is checked
    against the reference every step.  Returns the number of steps played."""
    ref, eng = make(ref_lib), make(engine_lib)
    if turn:
        ref.set_render_dir(tmpdir)
    rs = np.random.RandomState(seed)
    hs, rhs = eng.get_handles(), ref.get_handles()
    for t in range(steps):
        states = read_states(eng)
        for s in states[1:]:
            np.testing.assert_array_equal(_bits(s), _bits(states[0]), err_msg="step %d: two reads differ" % t)
        for h, rh in zip(hs, rhs):
            np.testing.assert_array_equal(eng.get_pos(h), ref.get_pos(rh), err_msg="step %d: engines diverged" % t)
        dirs = headings(ref, tmpdir) if turn else None
        check_arena_state(states[0][0], ref, dirs, "step %d" % t)
        for h, rh in zip(hs, rhs):
            act = rs.randint(0, ref.get_action_space(rh)[0], size=ref.get_num(rh)).astype(np.int32)
            eng.set_action(h, act)
            ref.set_action(rh, act)
        ref.step()
        eng.step()
        ref.clear_dead()
        eng.clear_dead()
    return steps


def play_batch_lockstep(make, engine_lib, ref_lib, arenas, steps, seed, read_states):
    """An arena batch behind one handle (seeded `seed`) against independent references seeded seed + a: every arena's
    state checked against its reference every step."""
    eng = make(engine_lib, seed, _num_arenas=arenas)
    refs = [make(ref_lib, seed + a) for a in range(arenas)]
    rs = np.random.RandomState(seed)
    hs = eng.get_handles()
    for t in range(steps):
        states = read_states(eng)
        for s in states[1:]:
            np.testing.assert_array_equal(_bits(s), _bits(states[0]), err_msg="step %d: two reads differ" % t)
        for a, ref in enumerate(refs):
            check_arena_state(states[0][a], ref, None, "step %d arena %d" % (t, a))
        for g, h in enumerate(hs):
            nums = eng.get_arena_nums(h)
            act = rs.randint(0, eng.get_action_space(h)[0], size=int(nums.sum())).astype(np.int32)
            off = np.concatenate([[0], np.cumsum(nums)])
            eng.set_action(h, act)
            for a, ref in enumerate(refs):
                ref.set_action(ref.get_handles()[g], np.ascontiguousarray(act[off[a]:off[a + 1]]))
        eng.step()
        for ref in refs:
            ref.step()
        eng.clear_dead()
        for ref in refs:
            ref.clear_dead()
