"""Observation render CTAs that render many tiles, in every instantiation, bit-exact against reference arenas.

A render CTA keeps its shared-memory tile from one tile to the next.  When a warp's next observer lives in the same
arena, it only undoes what it marked for the previous observer (the marked cells with the previous observer's heading,
the large-view tail beyond NIT * 32 cells, the self marker) and marks the new one; it rebuilds the record only when the
arena changes.  At the sizes a test can check, the automatic launch gives every CTA a single tile, so none of that runs.
These tests force small grids through the engine's "obs_grid" / "obs_chunk" / "obs_tile" keys, read back the launch
from "obs_launch" to prove which instantiation ran with more tiles than CTAs, and compare every observation of a
four-arena batch with four independent reference games (arena a seeded SEED + a), element by element."""
import functools
import itertools
import os
import shutil
import tempfile

import numpy as np
import pytest

import parity_common as pc

pytestmark = pytest.mark.gpu

# any seed does; the reference games are deterministic only single-threaded (OMP_NUM_THREADS=1, tests/conftest.py)
SEED = 22
A = 4
MAP = 48
WALLS = 40
STEPS = 7
PRE_CULL = (1, 3, 5)            # steps whose observations are also taken between env_step and clear_dead
# agents per group and arena: no multiple of any tile width, one arena with each group empty (NaN minimap channels)
COUNTS = ([137, 1, 0, 253], [61, 96, 45, 0])
RENDERED = 0                    # the arena whose headings the reference's replay dump gives (both groups stay non-empty:
                                # the compiled reference does not survive rendering an empty group)
SMEM_PER_BLOCK = 227 * 1024

# view name -> (range, turn_mode, minimap_mode, body length); in-range cells: CircleRange(6) 113, (8) 197, (10) 317,
# (16) 797.  The dispatch slots: <= 128 cells NIT 4, 129..256 NIT 8, more NIT 8 plus the tail loop; turn mode NIT 8
VIEWS = {
    "circle6": ("circle", 6, False, True, 1),
    "circle8": ("circle", 8, False, True, 1),
    "circle8_nominimap": ("circle", 8, False, False, 1),
    "circle10": ("circle", 10, False, True, 1),
    "circle16": ("circle", 16, False, True, 1),        # no wide tile fits in shared memory
    "turn_sector": ("sector", 7, True, True, 2),
    "turn_circle10": ("circle", 10, True, True, 1),   # the tail, with headings
}
TAIL_VIEWS = ("circle10", "circle16", "turn_circle10")
SHAPES = [(1, 1), (2, 3), (3, 8)]


def view_range(view):
    import magent_b200 as magent
    kind, radius = VIEWS[view][:2]
    return magent.gridworld.CircleRange(radius) if kind == "circle" else magent.gridworld.SectorRange(radius, 120)


def make_config(view):
    import magent_b200 as magent
    gw = magent.gridworld
    _, _, turn, minimap, length = VIEWS[view]
    cfg = gw.Config()
    cfg.set({"map_width": MAP, "map_height": MAP, "turn_mode": turn, "minimap_mode": minimap, "embedding_size": 10})
    unit = cfg.register_agent_type("unit", dict(
        width=1, length=length, hp=2, speed=2, damage=2.5, step_recover=0.0, step_reward=-0.005, kill_reward=5,
        dead_penalty=-0.1, attack_penalty=-0.1, view_range=view_range(view), attack_range=gw.CircleRange(1.5)))
    g0, g1 = cfg.add_group(unit), cfg.add_group(unit)
    a, b = gw.AgentSymbol(g0, index='any'), gw.AgentSymbol(g1, index='any')
    cfg.add_reward_rule(gw.Event(a, 'attack', b), receiver=a, value=0.2)
    cfg.add_reward_rule(gw.Event(b, 'attack', a), receiver=b, value=0.2)
    return cfg


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


def populate(env, arenas):
    """walls, then the agents of each group; `arenas` = the arena indices env holds (a batch) or [a] (one game)"""
    for a in arenas:
        if len(arenas) > 1:
            env.select_arena(a)
        env.add_walls(method="random", n=WALLS)
        for g, h in enumerate(env.get_handles()):
            if COUNTS[g][a]:
                env.add_agents(h, method="random", n=COUNTS[g][a])
    if len(arenas) > 1:
        env.select_arena(-1)


def read_headings(render_dir):
    """per frame of the reference's render dump: per group, the heading (0..3) of every agent in group order"""
    frames = []
    videos = [n for n in os.listdir(render_dir) if n.startswith("video_")]
    assert len(videos) == 1, videos                        # the first file's number differs between implementations
    with open(os.path.join(render_dir, videos[0])) as f:
        lines = f.read().split("\n")
    i = int(lines[0].split()[1]) + 1                       # "W n" and the walls
    while i < len(lines) and lines[i].startswith("F"):
        _, n_agents, n_attacks, _ = lines[i].split()
        dirs = {}
        for line in lines[i + 1:i + 1 + int(n_agents)]:
            _, _, angle, _, _, g = (int(v) for v in line.split())
            dirs.setdefault(g, []).append(angle // 90)
        frames.append(dirs)
        i += 1 + int(n_agents) + int(n_attacks)
    return frames


class Trace:
    """what four reference games observed, step by step, concatenated over arenas as the batch presents them"""

    def __init__(self, view):
        import magent_b200 as magent
        lib = checker_lib()
        turn, minimap = VIEWS[view][2], VIEWS[view][3]
        refs = []
        for a in range(A):
            env = magent.GridWorld(make_config(view), _lib=lib)
            env.set_seed(SEED + a)
            env.reset()
            populate(env, [a])
            refs.append(env)
        self.handles = range(len(refs[0].get_handles()))
        self.view_space = refs[0].get_view_space(refs[0].get_handles()[0])
        tmp = tempfile.mkdtemp() if turn else None
        if turn:
            refs[RENDERED].set_render_dir(tmp)
        self.rounds, self.actions = [], []
        rs = np.random.RandomState(SEED)
        self.dead_seen = 0
        for step in range(STEPS):
            if turn:                                        # the headings this round's observers have
                refs[RENDERED].render()
            self.rounds.append(self.observe(refs, "step %d" % step))
            acts = {}
            for g in self.handles:
                n_act = refs[0].get_action_space(refs[0].get_handles()[g])[0]
                acts[g] = rs.randint(0, n_act, size=int(sum(self.rounds[-1]["nums"][g]))).astype(np.int32)
                off = np.concatenate([[0], np.cumsum(self.rounds[-1]["nums"][g])])
                for a, env in enumerate(refs):
                    env.set_action(env.get_handles()[g], np.ascontiguousarray(acts[g][off[a]:off[a + 1]]))
            self.actions.append(acts)
            for env in refs:
                env.step()
            if step in PRE_CULL:
                self.rounds.append(self.observe(refs, "step %d before clear_dead" % step))
                self.dead_seen += sum(int((~env.get_alive(h).astype(bool)).sum()) for env in refs for h in env.get_handles())
            for env in refs:
                env.clear_dead()
        if turn:
            frames = read_headings(tmp)
            shutil.rmtree(tmp)
            assert len(frames) == STEPS, "rendered frames: %d" % len(frames)
            starts = [r for r in self.rounds if "before" not in r["label"]]
            for r, frame in zip(starts, frames):
                r["headings"] = {}                          # -1: not known (the arenas that are not rendered)
                for g in self.handles:
                    r["headings"][g] = np.concatenate([np.asarray(frame[g], np.int64) if a == RENDERED else
                                                       np.full(r["nums"][g][a], -1, np.int64) for a in range(A)])
                    assert len(r["headings"][g]) == len(r["obs"][g][0])
        # view cells that ever showed a wall or an agent (minimap channels aside): > 256 means the tail had marks
        mm = {1 + 3 * k + 2 for k in self.handles} if minimap else set()
        keep = [c for c in range(self.view_space[2]) if c not in mm]
        marked = np.zeros(self.view_space[:2], bool)
        for r in self.rounds:
            for g in self.handles:
                marked |= (r["obs"][g][0][..., keep] != 0).any(axis=(0, 3))
        self.marked_cells = int(marked.sum())

    def observe(self, refs, label):
        rnd = {"label": label, "obs": {}, "nums": {}, "headings": None}
        for g in self.handles:
            parts = [self.observe_one(env, env.get_handles()[g]) for env in refs]
            rnd["nums"][g] = [len(v) for v, _ in parts]
            rnd["obs"][g] = (np.concatenate([v for v, _ in parts]), np.concatenate([f for _, f in parts]))
        return rnd

    @staticmethod
    def observe_one(env, h):
        n = env.get_num(h)
        if n == 0:                                         # the reference does not observe an empty group
            return (np.zeros((0,) + env.get_view_space(h), np.float32), np.zeros((0,) + env.get_feature_space(h), np.float32))
        v, f = env.get_observation(h)
        return v.copy(), f.copy()


@functools.lru_cache(maxsize=2)
def reference(view):
    return Trace(view)


def make_batch(view, obs_launch=None):
    import magent_b200 as magent
    env = magent.GridWorld(make_config(view), _lib=pc.CUDA_LIB, _num_arenas=A, _obs_launch=obs_launch)
    env.set_seed(SEED)
    env.reset()
    populate(env, list(range(A)))
    return env


def replay(trace, engines, check):
    """drive the batch engines with the reference's actions; check(round, engine index, engine) at every round"""
    k = 0
    for step in range(STEPS):
        for e, env in enumerate(engines):
            check(trace.rounds[k], e, env)
        k += 1
        for env in engines:
            for g, h in enumerate(env.get_handles()):
                env.set_action(h, trace.actions[step][g])
            env.step()
        if step in PRE_CULL:
            for e, env in enumerate(engines):
                check(trace.rounds[k], e, env)
            k += 1
        for env in engines:
            env.clear_dead()


def bits(x, half):
    x = np.ascontiguousarray(x)
    return x.astype(np.float16).view(np.uint16) if half and x.dtype == np.float32 else x.view(np.uint16 if half else np.uint32)


def compare(got, want, half, nums, what, channels=None):
    """bit equality; on a mismatch, say which record (and arena, view cell, channel) differs first"""
    g, w = bits(got, half), bits(want, half)
    assert g.shape == w.shape, "%s: shape %s vs %s" % (what, g.shape, w.shape)
    if np.array_equal(g, w):
        return
    g2, w2 = g.reshape(len(g), -1), w.reshape(len(w), -1)
    bad = np.nonzero((g2 != w2).any(axis=1))[0]
    r = int(bad[0])
    e = int(np.nonzero(g2[r] != w2[r])[0][0])
    arena = int(np.searchsorted(np.cumsum(nums), r, side="right"))
    where = "element %d" % e if channels is None else "cell %d channel %d" % (e // channels, e % channels)
    raise AssertionError("%s: %d of %d records differ; first: record %d (arena %d), %s: got %#x, want %#x"
                         % (what, len(bad), len(g), r, arena, where, g2[r, e], w2[r, e]))


def wide_fits(trace, view, esz):
    h, w, c = trace.view_space
    lut = (4 if VIEWS[view][2] else 1) * ((h * w + 1) & ~1) * 8
    return (32 // esz) * h * w * c * esz + lut <= SMEM_PER_BLOCK


def reuse_pairs(arena, ta, grid, chunk):
    """(observer, next observer of the same warp) for every pair of consecutive tiles of one CTA (the kernel's
    tile order: chunks of `chunk` tiles dealt round-robin over `grid` CTAs), split into same-arena pairs (undo) and
    arena changes (rebuild)"""
    n = len(arena)
    tiles = -(-n // ta)
    same, change = [], 0
    for b in range(grid):
        seq = [t for t in range(tiles) if (t // chunk) % grid == b]
        for t1, t2 in zip(seq, seq[1:]):
            for w in range(ta):
                o1, o2 = t1 * ta + w, t2 * ta + w
                if o2 < n:
                    if arena[o1] == arena[o2]:
                        same.append((o1, o2))
                    else:
                        change += 1
    return same, change


def launch_cases():
    cases = []
    for view, dtype in itertools.product(VIEWS, ("f32", "f16")):
        cases.append((view, dtype, 0, None))
        cases += [(view, dtype, tile, shape) for tile in (1, 2) for shape in SHAPES]
    return cases


def case_id(c):
    view, dtype, tile, shape = c
    return "%s-%s-%s" % (view, dtype, "auto" if shape is None else "tile%d-g%dc%d" % ((tile,) + shape))


@pytest.mark.parametrize("case", launch_cases(), ids=case_id)
def test_tile_reuse_is_bit_exact(case):
    import torch
    view, dtype, tile, shape = case
    half = dtype == "f16"
    esz = 2 if half else 4
    trace = reference(view)
    assert trace.dead_seen > 0, "no agent died: the rounds before clear_dead render no dead observer"
    if view in TAIL_VIEWS:
        assert trace.marked_cells > 256, "only %d view cells were ever marked: the tail loop had no work" % trace.marked_cells
    env = make_batch(view, None if shape is None else (shape[0], shape[1], tile))
    nit = 4 if view == "circle6" else 8
    turn = int(VIEWS[view][2])
    stats = {"undo": 0, "rebuild": 0, "turned": 0, "turned_later": 0}

    def check(rnd, _, env):
        for g, h in enumerate(env.get_handles()):
            v, f = env.get_observation_torch(h, dtype=torch.float16 if half else None)
            rep = env._get_obs_launch()
            what = "%s group %d" % (rnd["label"], g)
            n = len(rnd["obs"][g][0])
            assert (rep["elem_bytes"], rep["nit"], rep["turn"]) == (esz, nit, turn), "%s: launch %s" % (what, rep)
            assert rep["aligned"] == 1
            compare(f.cpu().numpy(), rnd["obs"][g][1], half, rnd["nums"][g], what + " features")
            compare(v.cpu().numpy(), rnd["obs"][g][0], half, rnd["nums"][g], what + " views", trace.view_space[2])
            if shape is None:
                continue
            ta = (32 if tile == 2 and wide_fits(trace, view, esz) else 16) // esz
            tiles = -(-n // ta)
            grid = min(shape[0], tiles)
            want = dict(rep, tile_agents=ta, tiles=tiles, grid=grid, chunk=min(shape[1], -(-tiles // grid)))
            assert rep == want, "%s: launch %s, expected %s" % (what, rep, want)
            assert tiles > grid
            arena = np.repeat(np.arange(A), rnd["nums"][g])
            same, change = reuse_pairs(arena, ta, rep["grid"], rep["chunk"])
            stats["undo"] += len(same)
            stats["rebuild"] += change
            if rnd["headings"] is not None:
                hd = rnd["headings"][g]
                turned = sum(hd[o1] != hd[o2] for o1, o2 in same if hd[o1] >= 0)
                stats["turned"] += turned
                if rnd["label"] != "step 0":                # headings that turn actions set
                    stats["turned_later"] += turned

    replay(trace, [env], check)
    if shape is not None:
        assert stats["undo"] > 0 and stats["rebuild"] > 0, stats
        if turn:
            assert stats["turned_later"] > 0, "no warp followed an observer with one of another heading: %s" % stats


def unaligned(n_elems, half):
    """a CUDA region of n_elems starting one element past a 16-byte boundary, between guard elements holding a
    NaN sentinel: (region, the whole buffer as integers, guard elements on each side, sentinel)"""
    import torch
    guard = 17
    sentinel = 0x7da5 if half else 0x7fa5a5a5
    raw = torch.full((n_elems + 2 * guard,), sentinel, dtype=torch.int16 if half else torch.int32, device="cuda")
    buf = raw.view(torch.float16 if half else torch.float32)
    region = buf[guard:guard + n_elems]
    assert region.data_ptr() % 16 == (2 if half else 4)
    return region, raw, guard, sentinel


@pytest.mark.parametrize("view,dtype,tile", list(itertools.product(("circle6", "circle10", "turn_circle10"), ("f32", "f16"),
                                                                   (1, 2))))
def test_unaligned_output_takes_the_element_stores(view, dtype, tile):
    """view and feature rows written one element past a 16-byte boundary: every tile's element-store path and the
    header kernel's scalar path; the result equals the aligned call and the reference, the guards stay untouched"""
    import torch
    half = dtype == "f16"
    tdt = torch.float16 if half else torch.float32
    trace = reference(view)
    env = make_batch(view, (2, 3, tile))

    def check(rnd, _, env):
        for g, h in enumerate(env.get_handles()):
            n = len(rnd["obs"][g][0])
            vshape, fshape = (n,) + env.get_view_space(h), (n,) + env.get_feature_space(h)
            vr, vraw, guard, sentinel = unaligned(int(np.prod(vshape)), half)
            fr, fraw, _, _ = unaligned(int(np.prod(fshape)), half)
            v, f = env.get_observation_torch(h, out=(vr.view(vshape), fr.view(fshape)))
            rep = env._get_obs_launch()
            av, af = env.get_observation_torch(h, dtype=tdt)
            what = "%s group %d" % (rnd["label"], g)
            assert rep["aligned"] == 0 and env._get_obs_launch()["aligned"] == 1, what
            assert rep["tiles"] > rep["grid"], rep
            for raw in (vraw, fraw):
                edge = torch.cat([raw[:guard], raw[-guard:]]).cpu().numpy()
                assert (edge == sentinel).all(), "%s: a guard element was overwritten" % what
            compare(v.cpu().numpy(), av.cpu().numpy(), half, rnd["nums"][g], what + " views (aligned call)")
            compare(f.cpu().numpy(), af.cpu().numpy(), half, rnd["nums"][g], what + " features (aligned call)")
            compare(v.cpu().numpy(), rnd["obs"][g][0], half, rnd["nums"][g], what + " views", trace.view_space[2])
            compare(f.cpu().numpy(), rnd["obs"][g][1], half, rnd["nums"][g], what + " features")

    replay(trace, [env], check)


def test_forced_launch_stays_with_its_engine():
    """a forced engine and an automatic one, interleaved call by call: identical observations, and the forced
    launches never show up in the other engine's report or settings"""
    import torch  # noqa: F401
    view = "circle10"
    trace = reference(view)
    forced, auto = make_batch(view, (3, 8, 1)), make_batch(view)
    assert forced._get_obs_override() == (3, 8, 1) and auto._get_obs_override() == (0, 0, 0)
    last = {}

    def check(rnd, e, env):
        for g, h in enumerate(env.get_handles()):
            v, f = env.get_observation_torch(h)
            rep = env._get_obs_launch()
            what = "%s group %d engine %d" % (rnd["label"], g, e)
            compare(v.cpu().numpy(), rnd["obs"][g][0], False, rnd["nums"][g], what + " views", trace.view_space[2])
            compare(f.cpu().numpy(), rnd["obs"][g][1], False, rnd["nums"][g], what + " features")
            if e == 0:
                assert rep["grid"] == min(3, rep["tiles"]) and rep["tile_agents"] == 4, rep
                assert auto._get_obs_launch() == last.get("auto", auto._get_obs_launch()), what
            else:
                assert rep["grid"] == rep["tiles"], "the automatic engine launched %s" % rep
                last["auto"] = rep
                assert forced._get_obs_launch()["grid"] == min(3, forced._get_obs_launch()["tiles"])
        assert auto._get_obs_override() == (0, 0, 0)

    replay(trace, [forced, auto], check)
