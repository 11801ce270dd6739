"""The replay recorder (magent_b200_replay_new / _record / _write / _free) on the CPU.

The test-only host emulation (tests/emu/replay_emu.cc) gathers frames with the functions the CUDA kernels use
(replay_phases.h); everything else -- episodes, event lists, the frame buffer, the writer and its files -- is the
engine's own.  Each recorded arena's files are pinned byte for byte to env_render's for the same run with
select_arena(a) (tests/replay_common.py), and, for one arena, to the reference's env_render where it is built."""
import os
import subprocess

import numpy as np
import pytest

import arena_restore_common as arc
import parity_common as pc
import replay_common as rp

EMU_DIR = os.path.join(pc.REPO, "tests", "emu")
SRC_DIR = os.path.join(pc.REPO, "magent_b200", "csrc")
REPLAY_EMU_LIB = os.path.join(pc.REPO, "tests", "_emu", "libmagent_emu_replay.so")


@pytest.fixture(scope="module")
def emu():
    """the host emulation with every emulated loop (the restore tests need the restore and slot loops)"""
    emu_srcs = [os.path.join(EMU_DIR, f) for f in sorted(os.listdir(EMU_DIR)) if f.endswith("_emu.cc")]
    assert os.path.join(EMU_DIR, "replay_emu.cc") in emu_srcs
    newest = max(os.path.getmtime(os.path.join(SRC_DIR, f)) for f in os.listdir(SRC_DIR))
    newest = max([newest] + [os.path.getmtime(f) for f in emu_srcs])
    if not os.path.exists(REPLAY_EMU_LIB) or os.path.getmtime(REPLAY_EMU_LIB) < newest:
        os.makedirs(os.path.dirname(REPLAY_EMU_LIB), exist_ok=True)
        srcs = [os.path.join(SRC_DIR, f) for f in ("engine.cc", "shim.cc", "host_expand.cc")] + emu_srcs
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall",
                        "-Wno-unused-function"] + srcs + ["-pthread", "-o", REPLAY_EMU_LIB], check=True,
                       capture_output=True)
    return REPLAY_EMU_LIB


# every game mode: battle, absorbers (arrange), turn_mode, food_mode, sector views, the 4-group game
GAMES = {
    "battle": arc.SCENARIOS["battle"],
    "arrange": arc.SCENARIOS["arrange"],
    "turn": arc.SCENARIOS["turn"],
    "food": arc.SCENARIOS["food"],
    "multi4": arc.SCENARIOS["multi4"],
    "gather": arc.SCENARIOS["gather"],
    "sector": lambda lib, seed, **kw: pc.make_sector(lib, 30, seed, **kw),
}


def reset_and_place(env):
    """an env_reset mid-run with new placement in every arena"""
    env.select_arena(-1)
    env.reset()
    for h in env.get_handles():
        env.add_agents(h, method="random", n=8)


@pytest.mark.parametrize("name", sorted(GAMES))
def test_files_equal_env_render_in_every_game_mode(emu, name, tmp_path):
    rp.check_against_render(GAMES[name], emu, 3, 4, [0, 2, 3], 6, tmp_path)


@pytest.mark.parametrize("name", ["battle", "turn"])
def test_one_arena_equals_the_reference_render(emu, name, tmp_path):
    """with a single arena the recorder's files equal the reference's own env_render"""
    if not os.path.exists(pc.REF_LIB):
        pytest.skip("the reference build is not present")
    rec = str(tmp_path / "replay")
    rp.record_run(GAMES[name], emu, 5, 1, [0], 5, rec)
    rp.render_run(GAMES[name], pc.REF_LIB, 5, 1, 0, 5, str(tmp_path / "ref"))
    rp.assert_same_files(str(tmp_path / "ref"), os.path.join(rec, "arena_0"))


def test_env_reset_opens_a_new_file_with_walls(emu, tmp_path):
    rp.check_against_render(arc.make_duel, emu, 11, 3, [0, 1, 2], 6, tmp_path, ops={2: reset_and_place})
    d = tmp_path / "replay" / "arena_1"
    assert sorted(os.listdir(d)) == ["config.json", "video_1.txt", "video_2.txt"]
    assert rp.has_wall_block(d / "video_2.txt")


def _restore_run(emu, tmp_path, src_at, steps=8):
    """a duel batch recording every arena, with restore_arenas(pool, src_at[t]) after the clear_dead of step t"""
    env = arc.make_duel(emu, 21, _num_arenas=4)
    pool = env.snapshot_arenas()
    rid = env.new_replay([0, 1, 2, 3], 200)
    ops = {t: (lambda e, s=s: e.restore_arenas(pool, None if s is None else np.array(s, np.int32)))
           for t, s in src_at.items()}
    rp.drive(env, steps, 3, lambda: env.record_replay(rid), ops)
    env.write_replay(rid, str(tmp_path))
    return env


def test_host_src_restores_open_files_and_minus_one_does_not(emu, tmp_path):
    _restore_run(emu, tmp_path, {1: [-1, 1, 0, -1], 4: [-1, -1, 2, -1]})
    files = {a: sorted(f for f in os.listdir(tmp_path / ("arena_%d" % a)) if f.startswith("video")) for a in range(4)}
    assert files == {0: ["video_1.txt"], 1: ["video_1.txt", "video_2.txt"],
                     2: ["video_1.txt", "video_2.txt", "video_3.txt"], 3: ["video_1.txt"]}, files
    for a in (1, 2):
        for f in files[a][1:]:
            path = tmp_path / ("arena_%d" % a) / f
            assert rp.has_wall_block(path)
            first = rp.frames_of(path)[0]
            n_attack = int(first[0].split()[2])
            assert n_attack == 0, "a restored arena has no attack events until its next step"


def test_null_src_restores_exactly_the_done_arenas(emu, tmp_path):
    env = arc.make_duel(emu, 5, _num_arenas=4)
    pool = env.snapshot_arenas()
    rid = env.new_replay([0, 1, 2, 3], 400)
    rs = np.random.RandomState(0)
    hs = env.get_handles()
    env.record_replay(rid)
    restored = np.zeros(4, int)
    for _ in range(60):
        for h in hs:
            env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=env.get_num(h)).astype(np.int32))
        env.step()
        env.clear_dead()
        done = env.get_arena_done().copy()
        env.record_replay(rid)
        env.restore_arenas(pool)
        restored += done
        env.record_replay(rid)
    assert restored.sum() > 0, "no duel finished"
    env.write_replay(rid, str(tmp_path))
    for a in range(4):
        files = [f for f in os.listdir(tmp_path / ("arena_%d" % a)) if f.startswith("video")]
        assert len(files) == 1 + restored[a], (a, files, restored)


def test_restored_twin_replays_the_snapshot_arena(emu, tmp_path):
    """arena 1 restored from snapshot arena 0 and fed arena 0's slot actions writes arena 0's file from the snapshot"""
    env = arc.make_duel(emu, 9, _num_arenas=2)
    hs = env.get_handles()
    pool = env.snapshot_arenas()
    rid = env.new_replay([0, 1], 100)
    rs = np.random.RandomState(4)
    hist = []

    def play(acts_of):
        env.record_replay(rid)
        for t in range(6):
            acts = [acts_of(t, g, h) for g, h in enumerate(hs)]
            for h, x in zip(hs, acts):
                env.set_action_slots(h, x)
            env.step()
            env.record_replay(rid)
            env.clear_dead()
            env.record_replay(rid)
            hist.append(acts)

    def fresh(t, g, h):
        S = env.get_slot_space(h)
        return rs.randint(0, env.get_action_space(h)[0], size=(2, S)).astype(np.int32)
    play(fresh)
    env.restore_arenas(pool, np.array([-1, 0], np.int32))
    first = list(hist)

    def twin(t, g, h):
        x = fresh(t, g, h)
        x[1] = first[t][g][0]
        return x
    play(twin)
    env.write_replay(rid, str(tmp_path))
    a0 = open(tmp_path / "arena_0" / "video_1.txt").read()
    a1 = open(tmp_path / "arena_1" / "video_2.txt").read()
    # arena 0 played on after the restore: its file from the snapshot on is the twin's, followed by more frames
    assert len(rp.frames_of(tmp_path / "arena_1" / "video_2.txt")) == 13
    assert a0.startswith(a1) and len(a0) > len(a1)


def test_overflow_drops_and_counts_frames(emu, tmp_path):
    env = arc.make_duel(emu, 2, _num_arenas=2)
    rid = env.new_replay([1], 3)
    for _ in range(5):
        env.record_replay(rid)
    assert env.write_replay(rid, str(tmp_path)) == (3, 2)
    assert len(rp.frames_of(tmp_path / "arena_1" / "video_1.txt")) == 3
    env.record_replay(rid)
    assert env.write_replay(rid, str(tmp_path)) == (1, 0)
    assert len(rp.frames_of(tmp_path / "arena_1" / "video_1.txt")) == 4


def test_two_writes_equal_one(emu, tmp_path):
    ops = {3: reset_and_place}
    rp.record_run(arc.make_duel, emu, 13, 3, [0, 2], 7, str(tmp_path / "one"), ops=ops)
    rp.record_run(arc.make_duel, emu, 13, 3, [0, 2], 7, str(tmp_path / "many"), ops=ops, writes=4)
    for a in (0, 2):
        rp.assert_same_files(str(tmp_path / "one" / ("arena_%d" % a)), str(tmp_path / "many" / ("arena_%d" % a)))


def test_ten_thousand_frame_split_matches_env_render(emu, tmp_path):
    n = 10010
    env = arc.make_duel(emu, 1, n=2)
    rid = env.new_replay([0], n)
    for _ in range(n):
        env.record_replay(rid)
    assert env.write_replay(rid, str(tmp_path / "replay")) == (n, 0)
    ren = arc.make_duel(emu, 1, n=2)
    ren.set_render_dir(str(tmp_path / "render"))
    for _ in range(n):
        ren.render()
    rp.assert_same_files(str(tmp_path / "render"), str(tmp_path / "replay" / "arena_0"))
    assert sorted(os.listdir(tmp_path / "render")) == ["config.json", "video_1.txt", "video_2.txt"]


def _state(env):
    hs = env.get_handles()
    out = [env.get_counters().copy(), env.get_global_state().copy()]
    for h in hs:
        out += [env.get_agent_id(h).copy(), env.get_pos(h).copy(), env.get_alive(h).copy(),
                env.get_reward(h).copy()]
        if env.get_num(h):
            out += [x.copy() for x in env.get_observation(h)]
    return out


def test_a_live_recorder_changes_no_other_output(emu):
    runs = []
    for with_rec in (False, True):
        env = arc.SCENARIOS["battle"](emu, 4, _num_arenas=3)
        rid = env.new_replay([1], 64) if with_rec else None
        log = []
        rp.drive(env, 5, 2, lambda: log.append(_state(env)) or (with_rec and env.record_replay(rid)))
        runs.append(log)
    for a, b in zip(*runs):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


def _refused(fn):
    with pytest.raises(RuntimeError, match="refused"):
        fn()


def test_refusals_change_nothing(emu, tmp_path):
    env = arc.make_duel(emu, 3, _num_arenas=3)
    before = _state(env)
    for bad in ([], [3], [-1], [0, 0], [1, 2, 1]):
        _refused(lambda: env.new_replay(bad, 4))
    _refused(lambda: env.new_replay([0], 0))
    for fn in (env.record_replay, env.free_replay, lambda i: env.write_replay(i, str(tmp_path))):
        _refused(lambda: fn(0))
    rid = env.new_replay([0, 2], 4)
    env.free_replay(rid)
    for fn in (env.record_replay, env.free_replay, lambda i: env.write_replay(i, str(tmp_path))):
        _refused(lambda: fn(rid))
    rid = env.new_replay([1], 4)
    env.record_replay(rid)
    for s, t in zip(before, _state(env)):
        np.testing.assert_array_equal(s, t)
    # more agents than the frames were sized for: the per-arena capacity grows past 64
    grown = pc.make_battle(emu, 20, 8, 1, _num_arenas=2)
    rid = grown.new_replay([1], 4)
    grown.add_agents(grown.get_handles()[0], method="random", n=70)
    _refused(lambda: grown.record_replay(rid))
    assert grown.write_replay(rid, str(tmp_path / "grown")) == (0, 0)
