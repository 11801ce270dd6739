"""The nearest visible neighbours (magent_b200_get_neighbours) on the CPU.

The test-only host emulation (tests/emu/neighbours_emu.cc) keys and lists every observer's neighbours with the functions
the CUDA kernel uses (nbr_phases.h).  Here the restatement of tests/neighbours_common.py is pinned to what the compiled
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
import neighbours_common as nb
import parity_common as pc
from magent_b200 import build as b


EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
NBR_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_nbr.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation plus its restore loop (snapshots), its mean-action loop and its neighbours loop"""
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    emu_srcs = [os.path.join(EMU_DIR, f) for f in ("backend_emu.cc", "arena_restore_emu.cc", "mean_action_emu.cc",
                                                   "neighbours_emu.cc")]
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(NBR_EMU_LIB) or os.path.getmtime(NBR_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(NBR_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(src_dir, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", NBR_EMU_LIB], check=True, capture_output=True)
    return NBR_EMU_LIB


@pytest.fixture(scope="module")
def plain_emu():
    """the default emulation library, which has no neighbours loop"""
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
def test_listed_neighbours_are_where_the_reference_view_shows_them(emu, name, tmp_path):
    """The engine on the emulation and the reference play the same actions.  Every step, for every (group, of) pair
    and every listed neighbour: the reference's own view of the observer shows group `of` at `rel`, on a cell that
    neighbour covers; keys along a row do not decrease; and the emulation's rows equal the rows restated from the
    reference's getters."""
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
    K = 32
    listed = 0
    for t in range(6):
        for h, rh in zip(hs, rhs):
            np.testing.assert_array_equal(eng.get_pos(h), ref.get_pos(rh), err_msg="step %d: engines diverged" % t)
        dirs = gs.headings(ref, str(tmp_path)) if turn else None
        views = [ref.get_observation(rh)[0].copy() for rh in rhs]
        pos = [ref.get_pos(rh).astype(np.int64) for rh in rhs]
        alive = [ref.get_alive(rh).copy() for rh in rhs]
        for of in range(G):
            _m, _x1, _y1, w, l = gs.view_geometry(ref, of)
            owner = ma.owner_grid(H, W, pos[of], alive[of], None if dirs is None else dirs[of], w, l)
            for g in range(G):
                if len(pos[g]) == 0:
                    continue
                want_i, want_r, want_c, keys = nb.arena_rows(ref, g, of, K, pos[g], alive[g],
                                                             None if dirs is None else dirs[g], owner, 0)
                _n, X, Y, on = ma.neighbour_sets(ref, g, of, pos[g], alive[g], None if dirs is None else dirs[g], owner)
                seen = np.where(on, owner[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)], -1)
                ch = views[g][..., base + ((of - g) % G) * stride]
                for i, r in zip(*np.nonzero(want_i >= 0)):
                    vy, vx = want_r[i, r]
                    assert ch[i, vy, vx] != 0, "%s step %d: %d over %d, observer %d slot %d: the view shows nothing" % (
                        name, t, g, of, i, r)
                    assert seen[i, vy, vx] == want_i[i, r], "%s step %d: the cell is not the neighbour's" % (name, t)
                assert (np.diff(np.where(keys >= 0, keys, np.iinfo(np.int64).max), axis=1) >= 0).all()
                got = eng.get_neighbours(hs[g], K, hs[of])
                for x, y, what in zip(got, (want_i, want_r, want_c), ("idx", "rel", "count")):
                    np.testing.assert_array_equal(x, y, err_msg="%s step %d: %s of %d over %d" % (name, t, what, g, of))
                listed += int((want_i >= 0).sum())
        for h, rh in zip(hs, rhs):
            act = rs.randint(0, ref.get_action_space(rh)[0], size=ref.get_num(rh)).astype(np.int32)
            eng.set_action(h, act)
            ref.set_action(rh, act)
        ref.step()
        eng.step()
        ref.clear_dead()
        eng.clear_dead()
    assert listed > 0
    print("views read from", os.path.relpath(checker(), pc.REPO), "-", listed, "neighbours listed")


# ---------------------------------------------------------------- emulation against the restatement
@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_neighbours_equal_the_restatement_in_every_game_mode(emu, name, tmp_path):
    env = arc.SCENARIOS[name](emu, 5)
    assert nb.play_and_check(env, 6, 3, (1, 3, 32), tmp_path, uncull_every=3) > 0


FUZZ_SEEDS = [1, 2, 3, 5, 6, 8, 11, 13, 14, 20, 34, 41, 1004, 70001, 70005, 100002]


def test_neighbours_equal_the_restatement_under_the_fuzz_configs(emu, tmp_path):
    """random configs: 1 x 3 and turning long bodies, sector views, 5-8 groups, large-map bands, empty groups"""
    long3 = sector = many = turn_long = 0
    for seed in FUZZ_SEEDS:
        env = fz.make_env(emu, seed)
        d = tmp_path / ("s%d" % seed)
        d.mkdir()
        nb.play_and_check(env, 4, seed, (3, 32), d, uncull_every=3)
        hs = env.get_handles()
        geo = [gs.view_geometry(env, g) for g in range(len(hs))]
        attrs = [env.config.agent_type_dict[env.config.groups[g]] for g in range(len(hs))]
        turn = bool(env.config.config_dict.get("turn_mode", False))
        long3 += any(max(x[3], x[4]) == 3 for x in geo)
        turn_long += turn and any(x[3] != x[4] for x in geo)
        sector += any(a.get("view_range") is not None and a["view_range"].angle < 180 for a in attrs)
        many += len(hs) >= 5
    assert long3 and sector and many and turn_long, (long3, sector, many, turn_long)


def test_count_is_the_mean_action_count(emu):
    env = pc.make_pursuit(emu, 24, 2)
    rs = np.random.RandomState(5)
    hs = env.get_handles()
    for t in range(4):
        for g in hs:
            for o in hs:
                c = env.get_neighbours(g, 2, o)[2].copy()
                np.testing.assert_array_equal(c, env.get_mean_action(g, o)[1])
        am.random_step(env, rs)


# ---------------------------------------------------------------- edge cases
def test_ragged_batch_with_an_empty_group(emu):
    env = pc.make_battle(emu, 16, 20, 4, _num_arenas=4)
    hs = env.get_handles()
    for a, extra in enumerate((0, 7, 33, 1)):
        env.select_arena(a)
        env.add_agents(hs[0], method="random", n=extra)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    for t in range(4):
        nb.check_rows(env, 5, what="step %d" % t)
        am.random_step(env, rs)
    import magent_b200 as magent
    lone = magent.GridWorld("battle", map_size=12, _lib=emu, _num_arenas=2)
    lone.reset()
    lone.add_agents(lone.get_handles()[0], method="random", n=9)          # 9 per arena; group 1 stays empty
    nb.check_rows(lone, 4)
    h0, h1 = lone.get_handles()
    idx, rel, c = lone.get_neighbours(h1, 4, h0)
    assert idx.shape == (0, 4) and rel.shape == (0, 4, 2) and c.shape == (0,)
    idx, rel, c = lone.get_neighbours(h0, 4, h1)
    assert idx.shape == (18, 4) and (idx == -1).all() and (rel == -1).all() and not c.any()
    # rows of arena 1 point into arena 1's part of the concatenation
    idx = lone.get_neighbours(h0, 4, h0)[0]
    assert ((idx[9:] == -1) | (idx[9:] >= 9)).all() and ((idx[:9] == -1) | (idx[:9] < 9)).all()


def test_k_larger_than_every_count(emu):
    env = pc.make_battle(emu, 14, 12, 7)
    hs = env.get_handles()
    for g in hs:
        for o in hs:
            idx, rel, c = (x.copy() for x in env.get_neighbours(g, 32, o))
            assert c.max() < 32
            filled = np.arange(32).reshape(1, -1) < c.reshape(-1, 1)
            assert ((idx >= 0) == filled).all() and ((rel[..., 0] >= 0) == filled).all()
            assert ((rel[..., 1] >= 0) == filled).all()
            # the first slots are the rows at smaller k
            for k in (1, 2, 5):
                small = env.get_neighbours(g, k, o)
                np.testing.assert_array_equal(small[0], idx[:, :k])
                np.testing.assert_array_equal(small[1], rel[:, :k])
                np.testing.assert_array_equal(small[2], c)
    nb.check_rows(env, 32)


def test_rows_after_restore_arenas(emu):
    env = pc.make_battle(emu, 16, 24, 5, _num_arenas=3)
    snap = env.snapshot_arenas()
    pairs = [(g, o) for g in range(2) for o in range(2)]
    want = [nb.expected(env, g, o, 6) for g, o in pairs]
    rs = np.random.RandomState(2)
    for t in range(4):
        am.random_step(env, rs)
    nb.check_rows(env, 6, what="before the restore")
    env.restore_arenas(snap, np.array([0, -1, 2], dtype=np.int32))
    nb.check_rows(env, 6, what="after the restore")
    env.restore_arenas(snap, np.array([-1, 1, -1], dtype=np.int32))
    hs = env.get_handles()
    for (g, o), w in zip(pairs, want):
        for x, y in zip(env.get_neighbours(hs[g], 6, hs[o]), w):
            np.testing.assert_array_equal(x, y)


# ---------------------------------------------------------------- refusals
def test_refusals_change_nothing(emu):
    env = pc.make_battle(emu, 16, 20, 4)
    h = env.get_handles()[0]
    n = env.get_num(h)
    want = [x.copy() for x in env.get_neighbours(h, 3)]
    idx = np.full(4096, 7, dtype=np.int32)
    rel = np.full(8192, 7, dtype=np.int32)
    count = np.full(256, 7, dtype=np.int32)
    L = env._lib
    for g, o, k, what in ((-1, 0, 3, b"invalid group handle"), (2, 0, 3, b"invalid group handle"),
                          (0, -1, 3, b"invalid group handle"), (0, 2, 3, b"invalid group handle"),
                          (0, 0, 0, b"outside [1, 32]"), (0, 1, 33, b"outside [1, 32]"), (0, 0, -2, b"outside [1, 32]")):
        assert L.magent_b200_get_neighbours(env.game, g, o, k, idx.ctypes.data, rel.ctypes.data, count.ctypes.data) == -1
        assert what in L.magent_b200_last_error()
    assert L.magent_b200_get_neighbours(env.game, 0, 0, 3, None, rel.ctypes.data, count.ctypes.data) == -1
    assert b"needs an idx buffer" in L.magent_b200_last_error()
    assert (idx == 7).all() and (rel == 7).all() and (count == 7).all()
    with pytest.raises(ValueError):
        env.get_neighbours(h, 0)
    with pytest.raises(ValueError):
        env.get_neighbours(h, 33)
    for x, y in zip(env.get_neighbours(h, 3), want):
        np.testing.assert_array_equal(x, y)
    # rel and count may be NULL
    buf = np.zeros((n, 3), dtype=np.int32)
    assert L.magent_b200_get_neighbours(env.game, 0, 0, 3, buf.ctypes.data, None, None) == 0
    np.testing.assert_array_equal(buf, want[0])


def test_a_backend_without_the_neighbours_loop_refuses_the_call(plain_emu):
    env = pc.make_battle(plain_emu, 16, 20, 4)
    with pytest.raises(RuntimeError, match="no neighbours kernel"):
        env.get_neighbours(env.get_handles()[0], 4)
    am.random_step(env, np.random.RandomState(0))


# ---------------------------------------------------------------- the compiled kernel
LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")


def test_neighbours_kernel_has_no_stack_or_spills():
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    kernel = "neighbours_kernel"
    m = re.search(r"Function properties for (_ZN2mg2be\d+%s\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, open(LOG).read())
    assert m, kernel + " not in the ptxas report"
    assert tuple(int(v) for v in m.groups()[1:]) == (0, 0, 0), "%s: %s" % (kernel, m.groups()[1:])
