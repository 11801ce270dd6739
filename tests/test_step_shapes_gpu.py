"""The step and clear_dead kernels at forced CTA shapes, and as the whole-grid team in every game mode, against the
reference (tests/step_shapes_common.py).

Forced shapes: each runs in a child process with MAGENT_B200_STEP_THREADS / MAGENT_B200_CULL_THREADS /
MAGENT_B200_STEP_SMEM set (the engine reads them once per process).  The child plays every scenario on the CUDA
engine; the parent compares its traces with reference traces computed once for the module, checks from the
"step_launch" report that the forced shape really ran, and checks that the event counters do not depend on the shape.
Shapes that matter: one warp (more than 32 movers per thread: the movers past the 32 that SettledMask remembers), three
warps (a partial warp-sum row in every block scan), CTAs far wider than their arena, CTAs looping over arenas, and
the per-arena step scratch in HBM at several widths.

Whole-grid team: arenas of 34,000 to 36,000 agents in every game mode, played in this process; where an arena falls
below the grid threshold mid-episode, the later steps must run as a CTA per arena with the scratch in HBM.
"""
import math
import os
import pickle
import subprocess
import sys

import pytest

import parity_common as pc
import step_shapes_common as sc

pytestmark = pytest.mark.gpu

KNOBS = ("MAGENT_B200_STEP_THREADS", "MAGENT_B200_CULL_THREADS", "MAGENT_B200_STEP_SMEM")

# name -> (step threads, cull threads, step scratch in shared memory); None = the engine's choice
SHAPES = {
    "default": (None, None, True),
    "32_32_smem": (32, 32, True),
    "96_96_smem": (96, 96, True),
    "1024_1024_smem": (1024, 1024, True),
    "default_hbm": (None, None, False),
    "32_64_hbm": (32, 64, False),
    "608_1024_hbm": (608, 1024, False),
    "1024_32_hbm": (1024, 32, False),
}


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


def play_in_child(shape, out_dir):
    step, cull, smem = SHAPES[shape]
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    if step is not None:
        env["MAGENT_B200_STEP_THREADS"] = str(step)
    if cull is not None:
        env["MAGENT_B200_CULL_THREADS"] = str(cull)
    if not smem:
        env["MAGENT_B200_STEP_SMEM"] = "0"
    out = os.path.join(str(out_dir), shape + ".pkl")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [sc.__file__, out]
    r = subprocess.run(cmd, env=env, cwd=pc.REPO, capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, "%s child exited with %d:\n%s" % (shape, r.returncode, r.stderr[-4000:])
    with open(out, "rb") as f:
        return pickle.load(f)


@pytest.fixture(scope="module")
def reference():
    return sc.reference_traces(checker_lib())


@pytest.fixture(scope="module")
def default_run(tmp_path_factory):
    return play_in_child("default", tmp_path_factory.mktemp("default"))


def test_scenarios_show_what_they_are_there_for(reference):
    def total(rec, g):
        return sum(rec["num"][g]) if isinstance(rec["num"][g], tuple) else rec["num"][g]

    for name, group in (("battle_kills", 0), ("battle_kills", 1), ("crowd", 0), ("gather_infight", 1), ("forest", 0),
                        ("food_3", 1), ("food_5", 1), ("mixed", 1), ("multi4", 0), ("arena_batch", 0)):
        trace = reference[name]
        assert total(trace[-1], group) < total(trace[0], group), "%s: nobody of group %d died" % (name, group)
    for name in ("arrange", "arrange_goals_move"):                   # movers absorbed by goals
        trace = reference[name]
        assert total(trace[-1], 1) < total(trace[0], 1), name
    assert any((r["reward"][1] > 0.5).any() for r in reference["double_attack"]), "the two-tiger rule never fired"
    assert any(r["done"] for r in reference["general_rules"]), "the terminal rule never fired"
    # the crowd puts more movers on a thread of a 32-thread CTA than SettledMask remembers
    assert math.ceil(max(sc.arena_sizes(reference["crowd"][0])) / 32) > 32


@pytest.mark.timeout(300)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_forced_shape_matches_the_reference(shape, reference, default_run, tmp_path):
    got = default_run if shape == "default" else play_in_child(shape, tmp_path)
    step, cull, smem = SHAPES[shape]
    assert sorted(got) == sorted(reference)
    for name, want in reference.items():
        what = "%s %s" % (shape, name)
        pc.compare_traces(want, got[name]["trace"], what)
        assert got[name]["counters"] == default_run[name]["counters"], what + " event counters"
        launches = got[name]["launches"]
        arenas = len(sc.arena_sizes(want[0]))
        assert len(launches) == len(want)
        for t, (st, cu) in enumerate(launches):
            where = "%s step %d: %s / %s" % (what, t, st, cu)
            assert st["mode"] == 0 and cu["mode"] == 0 and cu["smem"] == 0 and cu["scratch_in_smem"] == 0, where
            assert st["threads"] == step if step is not None else st["threads"] in (256, 512, 1024), where
            assert cu["threads"] == cull if cull is not None else cu["threads"] in (256, 512, 1024), where
            assert st["scratch_in_smem"] == int(smem) and (st["smem"] > 0) == smem, where
            assert 0 < st["grid"] <= arenas and 0 < cu["grid"] <= arenas, where
    if step == 1024:                                                 # CTAs loop over the batch's arenas
        assert all(st["grid"] < sc.ARENAS for st, _ in got["arena_batch"]["launches"]), got["arena_batch"]["launches"][0]
    if step == 32:
        sizes = sc.arena_sizes(reference["crowd"][0])
        assert math.ceil(max(sizes) / step) > 32, sizes


def check_grid_launches(trace, launches, what):
    """the whole-grid team while an arena holds more than the threshold, then a CTA per arena with the scratch in
    HBM; returns the number of steps that ran as CTAs"""
    assert max(sc.arena_sizes(trace[0])) > sc.GRID_THRESHOLD, what
    assert len(launches) == len(trace)
    cta_steps = 0
    for t, (rec, (st, cu)) in enumerate(zip(trace, launches)):
        grid = max(sc.arena_sizes(rec)) > sc.GRID_THRESHOLD
        where = "%s step %d (%s agents): %s / %s" % (what, t, sc.arena_sizes(rec), st, cu)
        assert st["mode"] == cu["mode"] == int(grid), where
        assert st["grid"] > 0 and cu["grid"] > 0, where
        if grid:
            assert st["threads"] == cu["threads"] == 512 and st["smem"] == 0, where
        else:
            assert st["scratch_in_smem"] == 0 and st["smem"] == 0, where
            cta_steps += 1
    return cta_steps


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", list(sc.GRID_SCENARIOS))
def test_whole_grid_team_matches_the_reference(name):
    make, steps, seed, kw = sc.GRID_SCENARIOS[name]
    want = pc.run_trace(make(checker_lib()), steps, seed, **kw)
    env = make(pc.CUDA_LIB)
    log = sc.LaunchLog(env, env)
    got = pc.run_trace(log, steps, seed, **kw)
    pc.compare_traces(want, got, name)
    cta_steps = check_grid_launches(got, log.launches, name)
    if name in ("food", "mixed", "arrange", "sector"):               # the grid -> HBM-CTA switch happened
        assert cta_steps > 0, [sc.arena_sizes(r) for r in got]


@pytest.mark.timeout(300)
def test_whole_grid_team_loops_over_a_batch_of_arenas():
    """two grid-size arenas and a 2x40 one behind one handle, against three independent reference games"""
    games = sc.make_grid_battle_games(checker_lib())
    want = sc.arena_trace(sc.Games(games), sc.GRID_BATTLE_STEPS, 5)
    env = sc.make_grid_battle(pc.CUDA_LIB)
    log = sc.LaunchLog(sc.Batch(env), env)
    got = sc.arena_trace(log, sc.GRID_BATTLE_STEPS, 5)
    pc.compare_traces(want, got, "grid battle")
    check_grid_launches(got, log.launches, "grid battle")
    assert all(min(sc.arena_sizes(r)) < 100 for r in got)
