"""The replay recorder on the CUDA library: the record and event kernels against env_render, in every game mode, inside
a replayed CUDA graph with device-side restores, and at bench.py's sizes (tests/replay_common.py drives the runs)."""
import os

import numpy as np
import pytest

import arena_restore_common as arc
import parity_common as pc
import replay_common as rp
from test_replay_cpu import GAMES, reset_and_place

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


@pytest.mark.parametrize("name", sorted(GAMES))
def test_cuda_files_equal_env_render_in_every_game_mode(name, tmp_path):
    rp.check_against_render(GAMES[name], pc.CUDA_LIB, 3, 4, [0, 2, 3], 6, tmp_path)


def test_cuda_episodes_and_two_writes(tmp_path):
    rp.check_against_render(arc.make_duel, pc.CUDA_LIB, 11, 3, [0, 1, 2], 8, tmp_path, ops={2: reset_and_place},
                            writes=3)
    assert sorted(os.listdir(tmp_path / "replay" / "arena_1")) == ["config.json", "video_1.txt", "video_2.txt"]


@pytest.mark.parametrize("name", ["battle", "turn", "arrange"])
def test_cuda_one_arena_equals_the_compiled_reference(name, tmp_path):
    if not os.path.exists(pc.REF_LIB):
        pytest.skip("build() made no reference under oracle/_ref")
    rec = str(tmp_path / "replay")
    rp.record_run(GAMES[name], pc.CUDA_LIB, 5, 1, [0], 5, rec)
    rp.render_run(GAMES[name], pc.REF_LIB, 5, 1, 0, 5, str(tmp_path / "ref"))
    rp.assert_same_files(str(tmp_path / "ref"), os.path.join(rec, "arena_0"))


def _slot_loop(out_dir, graph):
    """a slot-ordered duel loop on the device: actions, step, two culls, restore_arenas(src=None), records"""
    import torch
    env = arc.make_duel(pc.CUDA_LIB, 17, _num_arenas=8)
    hs = env.get_handles()
    pool = env.snapshot_arenas()
    rid = env.new_replay(list(range(8)), 400)
    env.record_replay(rid)
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    shapes = [(8, env.get_slot_space(h)) for h in hs]
    acts = [torch.zeros(s, dtype=torch.int32, device="cuda") for s in shapes]
    gen = np.random.RandomState(5)

    def body():
        for _ in range(2):
            for h, x in zip(hs, acts):
                env.set_action_slots(h, x)
            env.step_device_done(done.data_ptr())
            env.record_replay(rid)
            env.clear_dead()
            env.record_replay(rid)
            env.restore_arenas(pool)
            env.record_replay(rid)
    gid = env.capture_graph(body) if graph else None
    for _ in range(50):
        for h, x, s in zip(hs, acts, shapes):
            x.copy_(torch.from_numpy(gen.randint(0, env.get_action_space(h)[0], size=s).astype(np.int32)))
        if graph:
            env.launch_graph(gid)
        else:
            body()
    n, dropped = env.write_replay(rid, out_dir)
    assert (n, dropped) == (1 + 50 * 6, 0)
    if graph:
        with pytest.raises(RuntimeError, match="refused"):
            env.free_replay(rid)
        with pytest.raises(RuntimeError, match="create recorders before capturing"):
            env.new_replay([1], 4)
    return env


def test_graph_replayed_loop_writes_the_eager_files(tmp_path):
    _slot_loop(str(tmp_path / "eager"), False)
    _slot_loop(str(tmp_path / "graph"), True)
    files = 0
    for a in range(8):
        rp.assert_same_files(str(tmp_path / "eager" / ("arena_%d" % a)), str(tmp_path / "graph" / ("arena_%d" % a)))
        files += len(os.listdir(tmp_path / "eager" / ("arena_%d" % a))) - 1
    assert files > 8, "no duel was restored"


def test_step_launch_report_is_unchanged_by_a_recorder():
    reports = []
    for with_rec in (False, True):
        env = arc.SCENARIOS["battle"](pc.CUDA_LIB, 4, _num_arenas=3)
        if with_rec:
            env.new_replay([1], 8)
        rp.drive(env, 2, 1, lambda: None)
        buf = np.zeros(10, np.int32)
        env._lib.env_get_info(env.game, -1, b"step_launch", buf.ctypes.data)
        reports.append(buf)
    np.testing.assert_array_equal(reports[0], reports[1])


def _bench_runs(workload, arenas, recorded, steps, tmp):
    """bench.py's workload with device-drawn legal actions: the recorder's files against env_render's"""
    import bench
    wl = bench.WORKLOADS[workload]

    def make(lib, seed, **kw):
        return bench.build_env(wl, lib, arenas, seed0=seed)[0]

    def run(frame, env):
        hs = env.get_handles()
        frame()
        for t in range(steps):
            for g, h in enumerate(hs):
                env.set_random_legal_actions(h, 1000 * t + g)
            env.step()
            frame()
            env.clear_dead()
            frame()
    rec = os.path.join(str(tmp), "replay")
    env = make(pc.CUDA_LIB, 3)
    rid = env.new_replay(recorded, 2 * steps + 1)
    run(lambda: env.record_replay(rid), env)
    assert env.write_replay(rid, rec) == (2 * steps + 1, 0)
    del env
    for a in recorded:
        env = make(pc.CUDA_LIB, 3)
        env.select_arena(a)
        d = os.path.join(str(tmp), "render_%d" % a)
        os.makedirs(d)
        env.set_render_dir(d)
        run(env.render, env)
        rp.assert_same_files(d, os.path.join(rec, "arena_%d" % a), "%s arena %d" % (workload, a))
        del env


def test_battle512_recording_four_arenas(tmp_path):
    _bench_runs("battle512", 512, [0, 1, 255, 511], 50, tmp_path)


def test_battle1m_recording_its_arena(tmp_path):
    _bench_runs("battle1m", 1, [0], 2, tmp_path)
