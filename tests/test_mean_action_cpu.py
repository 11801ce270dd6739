"""The mean neighbour action (magent_b200_get_mean_action) on the CPU.

The test-only host emulation (tests/emu/mean_action_emu.cc) decides every observer's neighbours with the functions the
CUDA kernel uses (nbr_phases.h).  Here the restatement of tests/mean_action_common.py is pinned to what the compiled
reference's own views show (or the oracle's C restatement where the reference is absent), and the emulation is checked
against the restatement in every game mode, under the fuzz configs and on the edge cases of the call."""
import os
import re
import subprocess

import numpy as np
import pytest

import action_mask_common as am
import arena_restore_common as arc
import fuzz_common as fz
import global_state_common as gs
import mean_action_common as ma
import parity_common as pc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
MEAN_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_mean.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation plus its restore loop (snapshots) and its mean-action loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "arena_restore_emu.cc", "mean_action_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(MEAN_EMU_LIB) or os.path.getmtime(MEAN_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(MEAN_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", MEAN_EMU_LIB], check=True, capture_output=True)
    return MEAN_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the default emulation library, which has no mean-action loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    if not os.path.exists(pc.EMU_LIB) or os.path.getmtime(pc.EMU_LIB) < newest:
        subprocess.run([os.path.join(EMU_DIR, "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


def checker():
    return pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB


# ---------------------------------------------------------------- the definition, pinned to the reference's views
LOCKSTEP_GAMES = {
    "battle": lambda lib: pc.make_battle(lib, 20, 40, 3),
    "pursuit": lambda lib: pc.make_pursuit(lib, 24, 2),
    "gather": lambda lib: pc.make_gather(lib, 20, 1, 20, 40),
    "multi4": lambda lib: pc.make_multi4(lib, 24, 8, 20),
    "sector": lambda lib: pc.make_sector(lib, 30, 4),
    "turn": lambda lib: pc.make_turn(lib, 30, 8),
    "arrange": lambda lib: pc.make_arrange(lib, 24, 12, 30, 60),
}


@pytest.mark.parametrize("name", sorted(LOCKSTEP_GAMES))
def test_neighbours_are_what_the_reference_view_shows(emu, name, tmp_path):
    """The engine on the emulation and the reference play the same actions.  Every step, for every (group, of) pair:
    the body cells of the restated neighbours that lie on in-range, on-board cells of each observer's window are
    exactly the cells where the reference's own view shows group `of` present (less the observer's own body when
    of == group), and the emulation's rows equal the rows restated from the reference's getters, bit for bit."""
    make = LOCKSTEP_GAMES[name]
    ref, eng = make(checker()), make(emu)
    cd = ref.config.config_dict
    turn = bool(cd.get("turn_mode", False))
    if turn:
        ref.set_render_dir(str(tmp_path))
    base = 1 + int(bool(cd.get("food_mode", False)))
    stride = 2 + int(bool(cd.get("minimap_mode", False)))
    hs, rhs = eng.get_handles(), ref.get_handles()
    G = len(hs)
    H, W, _C = eng.get_state_space()
    rs = np.random.RandomState(4)
    counted = shown_cells = 0
    for t in range(6):
        for h, rh in zip(hs, rhs):
            np.testing.assert_array_equal(eng.get_pos(h), ref.get_pos(rh), err_msg="step %d: engines diverged" % t)
        dirs = gs.headings(ref, str(tmp_path)) if turn else None
        views = [ref.get_observation(rh)[0].copy() for rh in rhs]
        acts = [ma.held_actions(ref, rh) for rh in rhs]
        pos = [ref.get_pos(rh).astype(np.int64) for rh in rhs]
        alive = [ref.get_alive(rh).copy() for rh in rhs]
        for of in range(G):
            _m, _x1, _y1, w, l = gs.view_geometry(ref, of)
            owner = ma.owner_grid(H, W, pos[of], alive[of], None if dirs is None else dirs[of], w, l)
            for g in range(G):
                if len(pos[g]) == 0:
                    continue
                nbrs, X, Y, on = ma.neighbour_sets(ref, g, of, pos[g], alive[g], None if dirs is None else dirs[g], owner)
                seen = np.where(on, owner[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)], -1)
                restated = np.stack([on[i] & np.isin(seen[i], nbrs[i]) for i in range(len(nbrs))])
                shown = on & (views[g][..., base + ((of - g) % G) * stride] != 0)
                if of == g:
                    shown &= seen != np.arange(len(nbrs)).reshape(-1, 1, 1)
                bad = np.argwhere(restated != shown)
                assert len(bad) == 0, "%s step %d: group %d over %d, %d cells differ, first (agent, vy, vx) %s" % (
                    name, t, g, of, len(bad), tuple(bad[0]))
                shown_cells += int(shown.sum())
                want_m, want_c = ma.rows(nbrs, acts[of], ref.get_action_space(rhs[of])[0])
                got_m, got_c = eng.get_mean_action(hs[g], hs[of])
                np.testing.assert_array_equal(got_c, want_c, err_msg="%s step %d: counts of %d over %d" % (name, t, g, of))
                np.testing.assert_array_equal(ma._bits(got_m), ma._bits(want_m),
                                              err_msg="%s step %d: means of %d over %d" % (name, t, g, of))
                counted += int(want_c.sum())
        for h, rh in zip(hs, rhs):
            act = rs.randint(0, ref.get_action_space(rh)[0], size=ref.get_num(rh)).astype(np.int32)
            eng.set_action(h, act)
            ref.set_action(rh, act)
        ref.step()
        eng.step()
        ref.clear_dead()
        eng.clear_dead()
    assert counted > 0 and shown_cells > 0
    print("views read from", os.path.relpath(checker(), pc.REPO), "-", counted, "neighbours,", shown_cells, "cells")


# ---------------------------------------------------------------- emulation against the restatement
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_mean_action_equals_the_restatement_in_every_game_mode(emu, name, tmp_path):
    env = arc.SCENARIOS[name](emu, 5)
    assert ma.play_and_check(env, 8, 3, tmp_path, uncull_every=3) > 0


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


def test_mean_action_equals_the_restatement_under_the_fuzz_configs(emu, tmp_path):
    """random configs: 1 x 3 and turning long bodies, sector views, 5-8 groups, large-map bands, empty groups"""
    long3 = sector = many = turn_long = 0
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed)
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        ma.play_and_check(env, 5, seed, d, uncull_every=3)
        hs = env.get_handles()
        geo = [gs.view_geometry(env, g) for g in range(len(hs))]
        attrs = [env.config.agent_type_dict[env.config.groups[g]] for g in range(len(hs))]
        turn = bool(env.config.config_dict.get("turn_mode", False))
        long3 += any(max(x[3], x[4]) == 3 for x in geo)
        turn_long += turn and any(x[3] != x[4] for x in geo)
        sector += any(a.get("view_range") is not None and a["view_range"].angle < 180 for a in attrs)
        many += len(hs) >= 5
    assert long3 and sector and many and turn_long, (long3, sector, many, turn_long)


# ---------------------------------------------------------------- edge cases
def test_ragged_batch_with_an_empty_group(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=4)
    hs = env.get_handles()
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        env.add_agents(hs[0], method="random", n=extra)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    for t in range(5):
        ma.check_means(env, what="step %d" % t)
        am.random_step(env, rs)
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # 9 per arena; group 1 stays empty
    ma.check_means(lone)
    h0, h1 = lone.get_handles()
    m, c = lone.get_mean_action(h1, h0)
    assert m.shape == (0, 21) and c.shape == (0,)
    m, c = lone.get_mean_action(h0, h1)
    assert m.shape == (18, 21) and not m.any() and not c.any()


def test_between_set_action_and_step_the_rows_show_the_actions_just_set(emu):
    env = pc.make_battle(emu, 14, 30, 2, _num_arenas=2)
    hs = env.get_handles()
    rs = np.random.RandomState(3)
    for t in range(4):
        acts = [rs.randint(0, 21, size=env.get_num(h)).astype(np.int32) for h in hs]
        for h, a in zip(hs, acts):
            env.set_action(h, a)
        ma.check_means(env, what="step %d after set_action" % t, acts=acts)
        env.step()
        env.clear_dead()
        ma.check_means(env, what="step %d after the step" % t)


def test_fresh_agents_and_out_of_range_actions_count_in_no_bin(emu):
    env = pc.make_battle(emu, 12, 30, 6)
    hs = env.get_handles()
    am.random_step(env, np.random.RandomState(0))
    n_old = env.get_num(hs[1])
    env.add_agents(hs[1], method="random", n=15)
    acts1 = ma.held_actions(env, hs[1])
    assert (acts1[n_old:] == -1).all() and (acts1[:n_old] >= 0).all()
    m, c = env.get_mean_action(hs[0], hs[1])
    ma.check_means(env, what="after add_agents")
    # some observer sees a fresh agent: its row sums to less than 1
    assert ((c > 0) & (m.sum(axis=1) < 1 - 1e-6)).any()
    # ids outside [0, n_action) are held as set and fall in no bin
    bad = np.full(env.get_num(hs[1]), 21, dtype=np.int32)
    bad[::3] = -4
    bad[1::3] = 5
    env.set_action(hs[1], bad)
    ma.check_means(env, what="out-of-range ids", acts=[None, np.where(bad == 5, 5, -1)], pairs=[(0, 1), (1, 1)])
    m, c = env.get_mean_action(hs[0], hs[1])
    assert (m[:, :5] == 0).all() and (m[:, 6:] == 0).all() and (m[:, 5] <= 1).all()


def test_rows_after_restore_arenas(emu):
    env = pc.make_battle(emu, 16, 24, 5, _num_arenas=3)
    snap = env.snapshot_arenas()
    want = [ma.expected(env, g, o) for g in range(2) for o in range(2)]
    rs = np.random.RandomState(2)
    for t in range(4):
        am.random_step(env, rs)
    ma.check_means(env, what="before the restore")
    env.restore_arenas(snap, np.array([0, -1, 2], dtype=np.int32))
    ma.check_means(env, what="after the restore")
    env.restore_arenas(snap, np.array([-1, 1, -1], dtype=np.int32))
    for (g, o), (wm, wc) in zip([(g, o) for g in range(2) for o in range(2)], want):
        m, c = env.get_mean_action(env.get_handles()[g], env.get_handles()[o])
        np.testing.assert_array_equal(c, wc)
        np.testing.assert_array_equal(ma._bits(m), ma._bits(wm))


# ---------------------------------------------------------------- refusals
def test_bad_group_handles_are_refused_and_change_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4)
    h = env.get_handles()[0]
    m0, c0 = (x.copy() for x in env.get_mean_action(h))
    mean = np.zeros(4096, dtype=np.float32)
    count = np.zeros(256, dtype=np.int32)
    for g, o in ((-1, 0), (2, 0), (99, 1), (0, -1), (0, 2), (1, 99)):
        assert env._lib.magent_b200_get_mean_action(env.game, g, o, mean.ctypes.data, count.ctypes.data) == -1
        assert b"invalid group handle" in env._lib.magent_b200_last_error()
    assert not mean.any() and not count.any()
    m, c = env.get_mean_action(h)
    np.testing.assert_array_equal(m, m0)
    np.testing.assert_array_equal(c, c0)
    # count may be NULL
    buf = np.zeros((env.get_num(h), 21), dtype=np.float32)
    assert env._lib.magent_b200_get_mean_action(env.game, 0, 0, buf.ctypes.data, None) == 0
    np.testing.assert_array_equal(buf, m0)


def test_a_backend_without_the_mean_action_loop_refuses_the_call(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    with pytest.raises(RuntimeError, match="no mean-action kernel"):
        env.get_mean_action(env.get_handles()[0])
    am.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernel
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


def test_mean_action_kernel_has_no_stack_or_spills():
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    kernel = "mean_action_kernel"
    m = re.search(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, open(LOG).read())
    assert m, kernel + " not in the ptxas report"
    assert tuple(int(v) for v in m.groups()[1:]) == (0, 0, 0), "%s: %s" % (kernel, m.groups()[1:])
