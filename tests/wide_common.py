"""Edge configurations for the kernels whose shared memory grows with the view or the action space.

Every side-output kernel sizes its dynamic shared memory from the view (a LUT of its in-range cells, four in turn_mode)
or from the action space (rows or histograms of n_action entries), and adds its own static shared memory (6400 bytes for
the kernels holding an EngineDev copy, 128 for the render and the wire kernel; nvcc -Xptxas -v, CUDA 12.9, sm_90a).
Each one has a band at the device's default per-block limit (49152 bytes on an H100: the dynamic opt-in above it) and a
ceiling at the opt-in limit (232448 bytes).  `EDGES` names configs on either side of those limits; `check_edge`
recomputes the bytes from get_view_space, get_action_space and get_feature_space and asserts that each config is still
on the side it was made for, within a margin, so that no config can drift off its edge unnoticed.

`config` builds a two-army game over the parameters the limits depend on: the view range (circle or sector), turn_mode,
the body size, the speed (the move disc), the attack range, the number of groups and the minimap.
"""
import numpy as np

import global_state_common as gs
import parity_common as pc

BLOCK = 48 * 1024            # cudaDevAttrMaxSharedMemoryPerBlock on an H100
OPTIN = 227 * 1024           # cudaDevAttrMaxSharedMemoryPerBlockOptin on an H100
STATIC_ENGINE = 6400         # action_mask(_slots)_kernel, mean_action(_slots)_kernel
STATIC_SMALL = 128           # obs_render_kernel, obs_wire_kernel
MASK_THREADS, MEAN_WARPS = 256, 8


def config(size=64, view=("circle", 6), turn=False, body=(1, 1), speed=2, attack=1.5, groups=2, minimap=True):
    """view: ("circle", r) or ("sector", r, angle); body: (width, length)"""
    import magent_b200 as magent
    gw = magent.gridworld
    cfg = gw.Config()
    cfg.set({"map_width": size, "map_height": size, "minimap_mode": minimap, "turn_mode": turn, "embedding_size": 4})
    vr = gw.CircleRange(view[1]) if view[0] == "circle" else gw.SectorRange(view[1], view[2])
    t = cfg.register_agent_type("wide", dict(width=body[0], length=body[1], hp=10, speed=speed, damage=2,
                                             step_recover=0.1, step_reward=-0.005, kill_reward=5, dead_penalty=-0.1,
                                             attack_penalty=-0.1, view_range=vr, attack_range=gw.CircleRange(attack)))
    gs_ = [cfg.add_group(t) for _ in range(groups)]
    syms = [gw.AgentSymbol(g, index='any') for g in gs_]
    for a in syms:
        for b in syms:
            if a is not b:
                cfg.add_reward_rule(gw.Event(a, 'attack', b), receiver=a, value=0.1)
    return cfg


# name -> (config kwargs, agents per group, {kernel: side}); side "in" = inside the limit, "optin" = past the default
# per-block limit but inside the opt-in one, "past" = past the ceiling (the call is refused, or takes another path)
EDGES = {
    # the render's ceiling: the narrow tile (16 bytes of records per cell and channel) plus the view LUT, always with
    # the opt-in.  2 groups + minimap = 7 channels.  Radius 22 / turn radius 20 are past it: an abort, documented.
    "render_r21": (dict(size=48, view=("circle", 21)), 80, {"render": "optin", "wire": "in", "mean": "in"}),
    "render_turn_r19": (dict(size=44, view=("circle", 19), turn=True), 70, {"render": "optin", "wire": "in", "mean": "in"}),
    # the widest wire LUT that fits the default limit (the render cannot hold this view: only the wire path serves it),
    # and one past it with a render that fits: the host path falls back to dense records
    "wire_r38": (dict(size=40, view=("circle", 38), groups=1, minimap=False), 60, {"wire": "in", "render": "past"}),
    "wire_turn_r20": (dict(size=44, view=("circle", 20), turn=True, groups=1), 60,
                      {"wire": "past", "render": "optin", "mean": "in"}),
    # the mean action: the last radius without the opt-in, the first with it, the last that fits, and one past
    "mean_r40": (dict(size=60, view=("circle", 40)), 120, {"mean": "in"}),
    "mean_r41": (dict(size=60, view=("circle", 41)), 120, {"mean": "optin"}),
    "mean_r94": (dict(size=60, view=("circle", 94)), 100, {"mean": "optin"}),
    "mean_r95": (dict(size=60, view=("circle", 95)), 40, {"mean": "past"}),
    "mean_turn_r21": (dict(size=40, view=("circle", 21), turn=True), 80, {"mean": "optin", "render": "past"}),
    "mean_turn_r47": (dict(size=40, view=("circle", 47), turn=True), 60, {"mean": "optin"}),
    "mean_turn_r48": (dict(size=40, view=("circle", 48), turn=True), 30, {"mean": "past"}),
    "mean_sector_r80": (dict(size=60, view=("sector", 80, 120)), 120, {"mean": "optin"}),
    # the neighbours' cell key, (2 kpad^2 + 1) * cells < 2^31: radius 127 is the last whose key fits, 128 is refused;
    # every observer sees more than 32 neighbours
    "nbr_r127": (dict(size=40, view=("circle", 127)), 60, {"nbr": "in", "mean": "past"}),
    "nbr_r128": (dict(size=40, view=("circle", 128)), 20, {"nbr": "past", "mean": "past"}),
}


def n_cells(env, h):
    vh, vw, _c = env.get_view_space(h)
    return vh * vw


def view_count(env, g):
    return int(gs.view_geometry(env, g)[0].sum())


def kernel_bytes(env, kernel, g=0, of=None):
    """the shared memory (static + dynamic) of `kernel` for group g (over group `of`), from the public spaces"""
    hs = env.get_handles()
    of = g if of is None else of
    turn = bool(env.config.config_dict.get("turn_mode", False))
    nh = 4 if turn else 1
    cells = n_cells(env, hs[g])
    lut = nh * ((cells + 1) & ~1) * 8
    if kernel == "mask":
        return STATIC_ENGINE + MASK_THREADS * env.get_action_space(hs[g])[0] + 16
    if kernel == "mean":
        return STATIC_ENGINE + nh * view_count(env, g) * 8 + MEAN_WARPS * env.get_action_space(hs[of])[0] * 4
    if kernel == "wire":
        return STATIC_SMALL + lut
    if kernel == "render":
        return STATIC_SMALL + 16 * cells * env.get_view_space(hs[g])[2] + lut
    raise ValueError(kernel)


def side(nbytes, kernel):
    """which side of the limits `nbytes` of `kernel` is on; the wire kernel does not opt in"""
    if nbytes <= BLOCK:
        return "in"
    if kernel == "wire":
        return "past"
    return "optin" if nbytes <= OPTIN else "past"


def check_edge(env, name, margin=16 * 1024):
    """every kernel of EDGES[name] on its side, and the first (the one the config is named for) within `margin` bytes
    of a limit"""
    for n, (kernel, want) in enumerate(EDGES[name][2].items()):
        if kernel == "nbr":
            vh, vw, _c = env.get_view_space(env.get_handles()[0])
            key = (2 * ((vw - 1) // 2) ** 2 + 1) * vh * vw
            assert (key < 2 ** 31) == (want == "in") and abs(key - 2 ** 31) < 2 ** 31 // 16, (name, key)
            continue
        got = kernel_bytes(env, kernel)
        assert side(got, kernel) == want, "%s: %s needs %d bytes: %s, made for %s" % (name, kernel, got, side(got, kernel), want)
        off = min(abs(got - BLOCK), abs(got - OPTIN))
        assert n > 0 or off <= margin, "%s: %s at %d bytes, %d from the nearest limit" % (name, kernel, got, off)


def make(lib, name, seed=0, arenas=1, **kw):
    import magent_b200 as magent
    cargs, n, _k = EDGES[name]
    env = magent.GridWorld(config(**cargs), _lib=lib, _num_arenas=arenas, **kw)
    env.set_seed(seed)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=n)
    return env


# mask and step configs: n_action -> (speed, attack radius, turn), 1 x 1 bodies.  With circle ranges the move disc and
# the attack ring are symmetric about the body, so n_action is odd (turn_mode adds two): the counts straddle the warp's
# 32-byte strides of a mask row.  167 is the first count past the default limit (256 * 167 + 16 + 6400 = 49168 > 49152:
# the launch needs the opt-in), 881 the last inside the opt-in limit (232,000 bytes), 883 the first past it (refused).
# 165, 167 and 205 (205 + 3 = 208 floats of feature row: 32 threads in the header pre-pass) are the long move chains of
# the step as well.
# The observation's header pre-pass holds at least 32 feature rows in the default 48 KB: rows of 384 floats, 377 actions
# with this config's embedding and minimap.  Wider action spaces take no observation on the GPU.
HEADER_MAX_ACTIONS = 377
MASK_SPACES = {
    31: (1.5, 2.5, True), 33: (1.0, 3.0, False), 63: (4.0, 2.0, True), 65: (2.25, 3.75, False),
    95: (2.0, 5.0, True), 97: (3.0, 4.5, False), 127: (3.0, 5.5, True), 129: (4.0, 5.0, False),
    165: (4.5, 5.5, False), 167: (6.5, 3.0, True), 205: (7.5, 3.0, False), 881: (16.5, 2.5, False),
    883: (16.5, 2.5, True),
}


def make_mask(lib, na, seed=0, arenas=1, n=150, size=36, **kw):
    """a crowded game whose groups have `na` actions (MASK_SPACES); asserts the count"""
    import magent_b200 as magent
    speed, attack, turn = MASK_SPACES[na]
    env = magent.GridWorld(config(size=size, view=("circle", 4), turn=turn, speed=speed, attack=attack),
                           _lib=lib, _num_arenas=arenas, **kw)
    assert env.get_action_space(env.get_handles()[0])[0] == na
    env.set_seed(seed)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=n)
    return env


def acts_by_id(env, held):
    """the actions every agent of every group holds, in group order, from {(g, id): action} of the last set_action"""
    return [np.array([held.get((g, int(i)), -1) for i in env.get_agent_id(h)], np.int64)
            for g, h in enumerate(env.get_handles())]


def random_step(env, rs, held=None, cull=True):
    """uniform random actions for every group (remembered in `held` by id), a step and (cull) clear_dead"""
    for g, h in enumerate(env.get_handles()):
        n, na = env.get_num(h), env.get_action_space(h)[0]
        a = rs.randint(0, na, size=n).astype(np.int32)
        env.set_action(h, a)
        if held is not None:
            for i, x in zip(env.get_agent_id(h), a):
                held[(g, int(i))] = int(x)
    done = env.step()
    if cull:
        env.clear_dead()
    return done


def state_trace(env, steps, seed, with_obs):
    """positions, ids, rewards and alive flags of every step of uniform random play, and (with_obs) the observations"""
    if with_obs:
        return pc.run_trace(env, steps, seed, keep_obs=False, stop_on_done=False)
    hs = env.get_handles()
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(steps):
        rec = {"num": [env.get_num(h) for h in hs], "obs": {}}
        rec["id"] = [env.get_agent_id(h).copy() for h in hs]
        rec["pos"] = [env.get_pos(h).copy() for h in hs]
        for h in hs:
            env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
        rec["done"] = bool(env.step())
        rec["reward"] = [env.get_reward(h).copy() for h in hs]
        rec["alive"] = [env.get_alive(h).copy() for h in hs]
        rec["pos_after"] = [env.get_pos(h).copy() for h in hs]
        env.clear_dead()
        out.append(rec)
    return out


EMU_LIB = pc.os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_wide.so")


def emu_lib():
    """the host emulation with every per-feature loop (tests/emu/*_emu.cc), rebuilt when a source is newer"""
    import os
    import subprocess
    emu_dir, src_dir = os.path.join(pc.REPO, "tests", "emu"), os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(emu_dir, f) for f in sorted(os.listdir(emu_dir)) if f.endswith("_emu.cc")]
    newest = max(os.path.getmtime(f) for f in emu_srcs + [os.path.join(src_dir, f) for f in os.listdir(src_dir)])
    if not os.path.exists(EMU_LIB) or os.path.getmtime(EMU_LIB) < newest:
        os.makedirs(os.path.dirname(EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", EMU_LIB], check=True, capture_output=True)
    return EMU_LIB
