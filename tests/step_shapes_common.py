"""Scenarios of the step / clear_dead launch-shape tests (tests/test_step_shapes_gpu.py, tests/test_step_shapes_cpu.py)
and the child process that plays them on the CUDA engine.

The step and cull kernels run as three kinds of team: a CTA per arena with the step scratch in shared memory, a CTA
per arena with the scratch in HBM, and the cooperative whole-grid team above GRID_THRESHOLD agents per arena.  The
CTA width and the scratch placement can be forced through MAGENT_B200_STEP_THREADS, MAGENT_B200_CULL_THREADS and
MAGENT_B200_STEP_SMEM=0; the engine reads them once per process, so every forced shape runs in a child process:

    python tests/step_shapes_common.py OUT.pkl

plays SCENARIOS and the ARENAS-arena batch on the CUDA library and pickles, per scenario, the trace
(parity_common.run_trace records, observations as hashes), the event-counter deltas and the "step_launch" report after
every step.  GRID_SCENARIOS are arenas of 34,000 to 36,000 agents for the whole-grid team; they need no knobs.
"""
import os
import pickle
import sys

import numpy as np

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import fuzz_common as fz  # noqa: E402
import parity_common as pc  # noqa: E402

GRID_THRESHOLD = 32768      # agents per arena above which the step and cull run as the whole-grid team


def make_crowd(lib):
    """2x700 battle agents on 60x60: 1400 agents in the move order, ~44 per thread of a 32-thread CTA"""
    return pc.make_battle(lib, 60, 700, 17)


def fuzz_scenario(seed):
    """fuzz_common.make_env with the acting groups and call order of fuzz_common.play"""
    rs = np.random.RandomState(seed)
    n_groups = fz.random_config(seed)[1]["n_groups"]
    order = [int(g) for g in rs.permutation(n_groups)]
    acting = sorted(int(g) for g in rs.choice(n_groups, size=int(rs.randint(1, n_groups + 1)), replace=False))
    return (lambda lib: fz.make_env(lib, seed), 20, seed,
            dict(act_groups=acting, order=[g for g in order if g in acting], stop_on_done=False))


# name -> (builder(lib), steps, action seed, run_trace keywords)
SCENARIOS = {
    "battle_kills": (lambda lib: pc.make_battle(lib, 30, 300, 3), 40, 3, {}),
    "crowd": (make_crowd, 30, 17, {}),
    "pursuit": (lambda lib: pc.make_pursuit(lib, 40, 1), 40, 1, {}),
    "gather_infight": (lambda lib: pc.make_gather(lib, 24, 2, n_agent=150, n_food=60), 40, 2, dict(act_groups=[1])),
    "forest": (lambda lib: pc.make_builtin(lib, "forest", 30, 3), 40, 3, {}),
    "double_attack": (lambda lib: pc.make_builtin(lib, "double_attack", 30, 4, n0=150, n1=120), 40, 4, {}),
    "mixed": (lambda lib: pc.make_mixed(lib, 36, 6), 40, 6, dict(order=[2, 0, 1])),
    "multi4": (lambda lib: pc.make_multi4(lib), 30, 8, dict(order=[3, 1, 0, 2])),
    "general_rules": (lambda lib: pc.make_general_rules(lib), 70, 21, dict(stop_on_done=False)),
    "arrange": (lambda lib: pc.make_arrange(lib, 30, 12), 50, 12, dict(act_groups=[1], stop_on_done=False)),
    "arrange_goals_move": (lambda lib: pc.make_arrange(lib, 24, 14, n_goal=60, n_agent=150), 40, 14,
                           dict(stop_on_done=False)),
    "sector": (lambda lib: pc.make_sector(lib), 40, 9, dict(order=[1, 0])),
    "turn_3": (lambda lib: pc.make_turn(lib, 30, 3), 50, 3, dict(order=[1, 2, 0], stop_on_done=False)),
    "turn_5": (lambda lib: pc.make_turn(lib, 30, 5), 50, 5, dict(order=[2, 0, 1], stop_on_done=False)),
    "food_3": (lambda lib: pc.make_food(lib, 30, 3), 50, 3, dict(order=[1, 2, 0], stop_on_done=False)),
    "food_5": (lambda lib: pc.make_food(lib, 30, 5), 50, 5, dict(order=[2, 0, 1], stop_on_done=False)),
    "non_square": (lambda lib: pc.make_battle_rect(lib), 40, 2, {}),
}
# turn + absorbers (4 groups), turn + food + goal_mode, food + goal_mode (8 groups), turn + goal_mode + absorbers (7 groups)
FUZZ_SEEDS = (1007, 1013, 70011, 70016)
SCENARIOS.update({"fuzz_%d" % s: fuzz_scenario(s) for s in FUZZ_SEEDS})

# many small arenas behind one handle: more arenas than a grid of 1024-thread CTAs, so CTAs loop over arenas
ARENAS, ARENA_MAP, ARENA_AGENTS, ARENA_SEED, ARENA_STEPS = 300, 16, 12, 40, 40


def make_arena_batch(lib):
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=ARENA_MAP, _lib=lib, _num_arenas=ARENAS)
    env.set_seed(ARENA_SEED)                                     # arena a draws from seed ARENA_SEED + a
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=ARENA_AGENTS)
    return env


def make_arena_games(lib):
    """the arenas of make_arena_batch as independent games"""
    import magent_b200 as magent
    games = []
    for a in range(ARENAS):
        env = magent.GridWorld("battle", map_size=ARENA_MAP, _lib=lib)
        env.set_seed(ARENA_SEED + a)
        env.reset()
        for h in env.get_handles():
            env.add_agents(h, method="random", n=ARENA_AGENTS)
        games.append(env)
    return games


class Batch:
    """one engine with several arenas, seen as a list of games"""
    def __init__(self, env):
        self.env, self.hs = env, env.get_handles()
        self.n_act = [env.get_action_space(h)[0] for h in self.hs]

    def nums(self, g):
        return tuple(int(v) for v in self.env.get_arena_nums(self.hs[g]))

    def observation(self, g):
        return self.env.get_observation(self.hs[g])

    def set_action(self, g, act, nums):
        self.env.set_action(self.hs[g], act)

    def step(self):
        self.env.step()
        return tuple(bool(v) for v in self.env.get_arena_done() != 0)

    def get(self, what, g):
        return getattr(self.env, "get_" + what)(self.hs[g]).copy()

    def clear_dead(self):
        self.env.clear_dead()


class Games:
    """independent single-arena games, seen like a Batch (per-agent arrays concatenated in arena order)"""
    def __init__(self, games):
        self.games = games
        self.n_act = [games[0].get_action_space(h)[0] for h in games[0].get_handles()]

    def nums(self, g):
        return tuple(int(e.get_num(e.get_handles()[g])) for e in self.games)

    def observation(self, g):
        parts = [e.get_observation(e.get_handles()[g]) for e in self.games if e.get_num(e.get_handles()[g])]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    def set_action(self, g, act, nums):
        off = np.concatenate([[0], np.cumsum(nums)])
        for a, e in enumerate(self.games):
            e.set_action(e.get_handles()[g], np.ascontiguousarray(act[off[a]:off[a + 1]]))

    def step(self):
        return tuple(bool(e.step()) for e in self.games)

    def get(self, what, g):
        return np.concatenate([getattr(e, "get_" + what)(e.get_handles()[g]) for e in self.games])

    def clear_dead(self):
        for e in self.games:
            e.clear_dead()


def arena_trace(play, steps, seed):
    """run_trace for a Batch or Games: the same action stream, records with per-arena counts as "num", per-arena done
    flags as "done" and every per-agent array in arena order (agent ids are not compared: they are per arena)"""
    G = len(play.n_act)
    rs = np.random.RandomState(seed)
    trace = []
    for t in range(steps):
        rec = {"num": [play.nums(g) for g in range(G)], "obs": {}, "id": [np.zeros((0,), np.int32)] * G}
        for g in range(G):
            if sum(rec["num"][g]):
                v, f = play.observation(g)
                rec["obs"][g] = (pc.sha(v), pc.sha(f))
        rec["pos"] = [play.get("pos", g) for g in range(G)]
        for g in range(G):
            play.set_action(g, rs.randint(0, play.n_act[g], size=sum(rec["num"][g])).astype(np.int32), rec["num"][g])
        rec["done"] = play.step()
        rec["reward"] = [play.get("reward", g) for g in range(G)]
        rec["alive"] = [play.get("alive", g) for g in range(G)]
        rec["pos_after"] = [play.get("pos", g) for g in range(G)]
        play.clear_dead()
        trace.append(rec)
    return trace


class LaunchLog:
    """an engine (or a Batch around one) for parity_common.run_trace / arena_trace whose clear_dead also records the
    engine's "step_launch" report: launches[t] = (the launch of step t, the launch of the clear_dead after it)"""
    def __init__(self, target, engine):
        self.target, self.engine, self.launches = target, engine, []

    def __getattr__(self, name):
        return getattr(self.target, name)

    def clear_dead(self):
        self.target.clear_dead()
        self.launches.append(self.engine._get_step_launch())


# ------------------------------------------------------------------ whole-grid team: 34,000 to 36,000 agents per arena
def populate(lib, cfg, seed, walls, counts):
    import magent_b200 as magent
    env = magent.GridWorld(cfg, _lib=lib)
    env.set_seed(seed)
    env.reset()
    env.add_walls(method="random", n=walls)
    for h, n in zip(env.get_handles(), counts):
        env.add_agents(h, method="random", n=n)
    return env


GRID_SCENARIOS = {
    "turn": (lambda lib: populate(lib, pc.turn_config(320), 8, 1500, (9000, 9000, 16000)), 12, 3,
             dict(order=[1, 2, 0], stop_on_done=False)),
    # food and mixed lose agents fast enough to fall below the threshold within a few steps
    "food": (lambda lib: populate(lib, pc.food_config(300), 6, 200, (3000, 20000, 11000)), 15, 5,
             dict(order=[2, 0, 1], stop_on_done=False)),
    "mixed": (lambda lib: populate(lib, grid_mixed_config(300), 6, 200, (3000, 22000, 9000)), 15, 6,
              dict(order=[2, 0, 1], stop_on_done=False)),
    "arrange": (lambda lib: pc.make_arrange(lib, 260, 12, n_goal=12000, n_agent=22000), 12, 12,
                dict(stop_on_done=False)),
    "sector": (lambda lib: populate(lib, pc.sector_config(300), 4, 200, (28000, 6000)), 12, 9, dict(order=[1, 0])),
    "double_attack": (lambda lib: pc.make_builtin(lib, "double_attack", 280, 4, n0=22000, n1=12000), 10, 4, {}),
    "general_rules": (lambda lib: make_grid_general_rules(lib), 12, 21, dict(stop_on_done=False)),
}


def grid_mixed_config(size):
    """mixed_config without its tank-on-tank attack rule.  That rule pays +0.3 and -0.3 to receivers that can be the same
    agent; the device adds those with float atomics in either order, so such a reward, and the last-reward feature
    that carries it, is equal only within the reward tolerance (DESIGN.md section 9).  At 34,000 agents two tanks hit
    each other within a few steps."""
    cfg = pc.mixed_config(size)
    keep = [r for r in cfg.reward_rules if r[2] != [0.3, -0.3]]
    assert len(keep) == len(cfg.reward_rules) - 1
    cfg.reward_rules = keep
    return cfg


def make_grid_general_rules(lib):
    """make_general_rules at 260x260 with 16,500 more statues and 16,500 more targets: 'all'-subject rules over a
    grid-size group.  The rovers stay few: the three-rover rule binds every ordered triple of rovers."""
    env = pc.make_general_rules(lib, 21, size=260, n_rover=60)
    S, T = env.get_handles()[:2]
    env.add_agents(S, method="random", n=16500)
    env.add_agents(T, method="random", n=16500)
    return env


# three battle arenas behind one handle, set up per arena through select_arena: two grid-size ones and a small one
GRID_BATTLE_MAP, GRID_BATTLE_SEEDS, GRID_BATTLE_AGENTS, GRID_BATTLE_STEPS = 300, (31, 32, 33), (17000, 17000, 40), 12


def make_grid_battle(lib):
    import magent_b200 as magent
    env = magent.GridWorld("battle", map_size=GRID_BATTLE_MAP, _lib=lib, _num_arenas=len(GRID_BATTLE_SEEDS))
    env.reset()
    for a, s in enumerate(GRID_BATTLE_SEEDS):
        env.select_arena(a)
        env.set_seed(s)
    for h in env.get_handles():
        for a, n in enumerate(GRID_BATTLE_AGENTS):
            env.select_arena(a)
            env.add_agents(h, method="random", n=n)
    env.select_arena(-1)
    return env


def make_grid_battle_games(lib):
    import magent_b200 as magent
    games = []
    for s, n in zip(GRID_BATTLE_SEEDS, GRID_BATTLE_AGENTS):
        env = magent.GridWorld("battle", map_size=GRID_BATTLE_MAP, _lib=lib)
        env.set_seed(s)
        env.reset()
        for h in env.get_handles():
            env.add_agents(h, method="random", n=n)
        games.append(env)
    return games


def arena_sizes(rec):
    """agents of every arena at the start of a step (run_trace or arena_trace record)"""
    return [sum(n) for n in zip(*[n if isinstance(n, tuple) else (n,) for n in rec["num"]])]


# ------------------------------------------------------------------ the child process
def play_all(lib):
    out = {}
    for name, (make, steps, seed, kw) in SCENARIOS.items():
        env = make(lib)
        log = LaunchLog(env, env)
        c0 = env.get_counters()
        trace = pc.run_trace(log, steps, seed, **kw)
        out[name] = dict(trace=trace, counters=[b - a for a, b in zip(c0, env.get_counters())], launches=log.launches)
    env = make_arena_batch(lib)
    log = LaunchLog(Batch(env), env)
    c0 = env.get_counters()
    trace = arena_trace(log, ARENA_STEPS, ARENA_SEED)
    out["arena_batch"] = dict(trace=trace, counters=[b - a for a, b in zip(c0, env.get_counters())], launches=log.launches)
    return out


def reference_traces(lib):
    """what play_all records, but the traces only, on a reference library"""
    out = {name: pc.run_trace(make(lib), steps, seed, **kw) for name, (make, steps, seed, kw) in SCENARIOS.items()}
    out["arena_batch"] = arena_trace(Games(make_arena_games(lib)), ARENA_STEPS, ARENA_SEED)
    return out


if __name__ == "__main__":
    result = play_all(pc.CUDA_LIB)
    with open(sys.argv[1], "wb") as f:
        pickle.dump(result, f)
