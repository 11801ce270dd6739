"""Checks of the reset pool (snapshot_arenas / restore_arenas) against reference games.

A batch of A arenas behind one handle, seeded `seed`, places arena a exactly as a single-arena reference game seeded
seed + a does (play_batch_lockstep in global_state_common.py relies on the same).  `Lockstep` drives such a batch and
one reference game per arena with the same random actions and compares every arena with its reference at every step:
views and features bit for bit, num / arena_num, ids, positions, alive and done exactly, rewards within 1e-6.

A restore replaces the reference of every restored arena a by a *twin*: a new reference game seeded seed + s (s the
source arena) with the same placement, fed the actions source arena s received up to the snapshot.  With keep_rng the
twin is then re-seeded with the arena's RNG state read before the restore (minstd's seed(x) sets the state x), so its
stream is the arena's own.  Arenas that are not restored keep their reference.
"""
import numpy as np

import parity_common as pc
from magent_b200 import gridworld as gw
from magent_b200.builtin.config.battle import SMALL


def duel_config(size):
    """battle with one-hit kills and speed 1: small dense arenas finish (one army wiped out) within a few dozen steps"""
    cfg = gw.Config()
    cfg.set({"map_width": size, "map_height": size, "minimap_mode": True, "embedding_size": 10})
    t = cfg.register_agent_type("small", dict(SMALL, damage=10, speed=1, view_range=gw.CircleRange(4),
                                              attack_range=gw.CircleRange(1.5)))
    g = [cfg.add_group(t), cfg.add_group(t)]
    who = [gw.AgentSymbol(x, index="any") for x in g]
    cfg.add_reward_rule(gw.Event(who[0], "kill", who[1]), receiver=who[0], value=1.0)
    return cfg


def make_duel(lib, seed, n=8, **kw):
    import magent_b200 as magent
    env = magent.GridWorld(duel_config(7), _lib=lib, **kw)
    env.set_seed(seed)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=n)
    return env


# make(lib, seed, **kw): every game mode the engine has
SCENARIOS = {
    "battle": lambda lib, seed, **kw: pc.make_battle(lib, 20, 40, seed, **kw),
    "pursuit": lambda lib, seed, **kw: pc.make_pursuit(lib, 24, seed, **kw),
    "gather": lambda lib, seed, **kw: pc.make_gather(lib, 24, seed, 20, 60, **kw),
    "forest": lambda lib, seed, **kw: pc.make_builtin(lib, "forest", 24, seed, 40, 20, **kw),
    "double_attack": lambda lib, seed, **kw: pc.make_builtin(lib, "double_attack", 24, seed, 40, 20, **kw),
    "multi4": lambda lib, seed, **kw: pc.make_multi4(lib, 30, seed, 30, **kw),
    "food": lambda lib, seed, **kw: pc.make_food(lib, 24, seed, **kw),
    "turn": lambda lib, seed, **kw: pc.make_turn(lib, 30, seed, **kw),
    "arrange": lambda lib, seed, **kw: pc.make_arrange(lib, 24, seed, 30, 60, **kw),
}

# restores after the clear_dead of these steps: cross-arena sources, every arena from itself, the done flags, a subset
PLAN = {2: [-1, 2, -1, 0], 4: [0, 1, 2, 3], 6: None, 7: [3, -1, 1, -1]}


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def as_src(src, kind):
    """src list -> what restore_arenas takes: None, an int32 numpy array ("host") or an int32 CUDA tensor ("device")"""
    if src is None:
        return None
    arr = np.asarray(src, dtype=np.int32)
    if kind == "host":
        return arr
    import torch
    return torch.from_numpy(arr).cuda()


class Lockstep:
    def __init__(self, make, eng_lib, ref_lib, arenas, seed):
        self.make, self.ref_lib, self.A, self.seed = make, ref_lib, arenas, seed
        self.eng = make(eng_lib, seed, _num_arenas=arenas)
        self.refs = [make(ref_lib, seed + a) for a in range(arenas)]
        self.hist = [[] for _ in range(arenas)]     # per arena: the actions (one array per group) of every step it played
        self.snap_hist = {}
        self.rs = np.random.RandomState(seed + 1000)
        self.t = 0

    def snapshot(self):
        pool = self.eng.snapshot_arenas()
        self.snap_hist[pool] = [list(h) for h in self.hist]
        return pool

    def twin(self, pool, s):
        """a reference game in the state of arena s of the snapshot"""
        ref = self.make(self.ref_lib, self.seed + s)
        for acts in self.snap_hist[pool][s]:
            for rh, x in zip(ref.get_handles(), acts):
                ref.set_action(rh, x)
            ref.step()
            ref.clear_dead()
        return ref

    def check(self, what=""):
        eng, hs = self.eng, self.eng.get_handles()
        tag = "step %d%s" % (self.t, what)
        for g, h in enumerate(hs):
            nums = eng.get_arena_nums(h).copy()
            assert eng.get_num(h) == int(nums.sum()), "%s: num of group %d" % (tag, g)
            off = np.concatenate([[0], np.cumsum(nums)])
            view, feat = (x.copy() for x in eng.get_observation(h)) if nums.sum() else (None, None)
            ids, pos = eng.get_agent_id(h).copy(), eng.get_pos(h).copy()
            for a, ref in enumerate(self.refs):
                rh = ref.get_handles()[g]
                m = "%s arena %d group %d" % (tag, a, g)
                assert nums[a] == ref.get_num(rh), "%s: %d agents, the reference has %d" % (m, nums[a], ref.get_num(rh))
                if nums[a] == 0:
                    continue
                sl = slice(off[a], off[a + 1])
                np.testing.assert_array_equal(ids[sl], ref.get_agent_id(rh), err_msg=m + " ids")
                np.testing.assert_array_equal(pos[sl], ref.get_pos(rh), err_msg=m + " pos")
                rv, rf = ref.get_observation(rh)
                np.testing.assert_array_equal(_bits(view[sl]), _bits(rv), err_msg=m + " views")
                np.testing.assert_array_equal(_bits(feat[sl]), _bits(rf), err_msg=m + " features")

    def step(self):
        eng, hs = self.eng, self.eng.get_handles()
        offs = []
        for g, h in enumerate(hs):
            nums = eng.get_arena_nums(h)
            off = np.concatenate([[0], np.cumsum(nums)])
            offs.append(off)
            act = self.rs.randint(0, eng.get_action_space(h)[0], size=int(off[-1])).astype(np.int32)
            eng.set_action(h, act)
            for a, ref in enumerate(self.refs):
                x = np.ascontiguousarray(act[off[a]:off[a + 1]])
                ref.set_action(ref.get_handles()[g], x)
                if g == 0:
                    self.hist[a].append([])
                self.hist[a][-1].append(x)
        eng.step()
        ref_done = [ref.step() for ref in self.refs]
        tag = "step %d" % self.t
        np.testing.assert_array_equal(eng.get_arena_done(), np.asarray(ref_done, dtype=np.int32), err_msg=tag + " done")
        for g, h in enumerate(hs):
            rew, alive, off = eng.get_reward(h), eng.get_alive(h), offs[g]
            for a, ref in enumerate(self.refs):
                rh = ref.get_handles()[g]
                if off[a + 1] == off[a]:
                    continue
                np.testing.assert_allclose(rew[off[a]:off[a + 1]], ref.get_reward(rh), rtol=0, atol=pc.REWARD_TOL,
                                           err_msg="%s arena %d group %d reward" % (tag, a, g))
                np.testing.assert_array_equal(alive[off[a]:off[a + 1]], ref.get_alive(rh),
                                              err_msg="%s arena %d group %d alive" % (tag, a, g))
        eng.clear_dead()
        for ref in self.refs:
            ref.clear_dead()
        self.t += 1

    def restore(self, pool, src, src_kind="host", keep_rng=False):
        """restore_arenas(pool, src) on the engine and the matching twins in place of the restored arenas' references;
        returns the number of arenas restored"""
        chosen = src if src is not None else [a if d else -1 for a, d in enumerate(self.eng.get_arena_done())]
        rng = self.eng.get_arena_rng() if keep_rng else None
        self.eng.restore_arenas(pool, as_src(src, src_kind), keep_rng=keep_rng)
        n = 0
        for a, s in enumerate(chosen):
            if s < 0 or s >= self.A:
                continue
            self.refs[a] = self.twin(pool, s)
            if keep_rng:
                self.refs[a].set_seed(int(rng[a]))
            self.hist[a] = list(self.snap_hist[pool][s])
            n += 1
        return n


def play_restarts(make, eng_lib, ref_lib, steps=10, seed=5, plan=PLAN, src_kind="host", keep_rng=False, arenas=4):
    """snapshot right after placement, play `steps` steps with every arena checked against its reference every step,
    restore after the steps in `plan`; returns the number of arenas restored"""
    L = Lockstep(make, eng_lib, ref_lib, arenas, seed)
    pool = L.snapshot()
    restored = 0
    for t in range(steps):
        L.check()
        L.step()
        if t in plan:
            restored += L.restore(pool, plan[t], src_kind, keep_rng)
            L.check(" (after the restore)")
    L.check()
    return restored


def mid_episode_replay(make, lib, t_snap=4, k=6, seed=3, arenas=3, src_kind="host"):
    """snapshot at step t_snap, record k steps of outputs under an action stream, restore every arena and replay the
    stream: the outputs must be identical, and the event counters keep counting"""
    env = make(lib, seed, _num_arenas=arenas)
    hs = env.get_handles()
    rs = np.random.RandomState(seed)

    def acts():
        return [rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32) for h in hs]

    for _ in range(t_snap):
        for h, x in zip(hs, acts()):
            env.set_action(h, x)
        env.step()
        env.clear_dead()
    pool = env.snapshot_arenas()

    def record(stream):
        out = []
        for step_acts in stream:
            rec = {"nums": [env.get_arena_nums(h).copy() for h in hs], "state": env.get_global_state().copy()}
            rec["obs"] = [[x.copy() for x in env.get_observation(h)] if env.get_num(h) else None for h in hs]
            rec["ids"] = [env.get_agent_id(h).copy() for h in hs]
            rec["pos"] = [env.get_pos(h).copy() for h in hs]
            for h, x in zip(hs, step_acts):
                env.set_action(h, x)
            rec["done"] = env.step()
            rec["arena_done"] = env.get_arena_done().copy()
            rec["reward"] = [env.get_reward(h).copy() for h in hs]
            rec["alive"] = [env.get_alive(h).copy() for h in hs]
            env.clear_dead()
            out.append(rec)
        return out

    first, stream = [], []
    for _ in range(k):                                  # the stream is drawn while playing it the first time
        stream.append(acts())
        first.extend(record(stream[-1:]))
    c0 = env.get_counters()
    env.restore_arenas(pool, as_src(list(range(arenas)), src_kind))
    second = record(stream)
    c1 = env.get_counters()
    assert c1[7] == c0[7] + k and all(b >= a for a, b in zip(c0, c1)), "counters %s -> %s" % (c0, c1)
    for i, (a, b) in enumerate(zip(first, second)):
        tag = "replayed step %d" % i
        for key in ("nums", "ids", "pos", "reward", "alive"):
            for g in range(len(hs)):
                np.testing.assert_array_equal(a[key][g], b[key][g], err_msg="%s %s group %d" % (tag, key, g))
        np.testing.assert_array_equal(_bits(a["state"]), _bits(b["state"]), err_msg=tag + " global state")
        for g in range(len(hs)):
            if a["obs"][g] is not None:
                np.testing.assert_array_equal(_bits(a["obs"][g][0]), _bits(b["obs"][g][0]), err_msg=tag + " views")
                np.testing.assert_array_equal(_bits(a["obs"][g][1]), _bits(b["obs"][g][1]), err_msg=tag + " features")
        assert a["done"] == b["done"], tag + " done"
        np.testing.assert_array_equal(a["arena_done"], b["arena_done"], err_msg=tag + " arena done")
