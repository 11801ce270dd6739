"""Checks of the replay recorder (magent_b200_replay_*) against env_render.

The recorder's files for arena a must equal, byte for byte, the files env_render writes for the same run with
select_arena(a) in force, frame for frame at the same points.  `drive` plays a batch with seeded random actions and
calls frame() after placement, after every env_step (attack events, dead agents still listed) and after every
clear_dead; `ops[t]` runs after the clear_dead of step t (an env_reset with new placement, say) in both runs alike.
"""
import os

import numpy as np


def drive(env, steps, seed, frame, ops=None):
    rs = np.random.RandomState(seed)
    hs = env.get_handles()
    frame()
    for t in range(steps):
        for h in hs:
            n = env.get_num(h)
            env.set_action(h, rs.randint(0, env.get_action_space(h)[0], size=n).astype(np.int32))
        env.step()
        frame()
        env.clear_dead()
        frame()
        if ops and t in ops:
            ops[t](env)
            frame()


def render_run(make, lib, seed, arenas, arena, steps, out_dir, ops=None, **kw):
    """env_render's files of one arena of the batch"""
    env = make(lib, seed, _num_arenas=arenas, **kw) if arenas > 1 else make(lib, seed, **kw)
    if arenas > 1:
        env.select_arena(arena)
    os.makedirs(out_dir, exist_ok=True)
    env.set_render_dir(out_dir)
    # an op may route setup calls to every arena: the render follows `arena` again after it
    if arenas > 1:
        ops = {t: (lambda e, f=f: (f(e), e.select_arena(arena))) for t, f in (ops or {}).items()}
    drive(env, steps, seed + 7, env.render, ops)
    return env


def record_run(make, lib, seed, arenas, recorded, steps, out_dir, ops=None, max_frames=None, writes=1, **kw):
    """the recorder's files of the recorded arenas (out_dir/arena_<a>), written `writes` times along the run"""
    env = make(lib, seed, _num_arenas=arenas, **kw) if arenas > 1 else make(lib, seed, **kw)
    frames = 3 + 2 * steps + 2 * len(ops or {})
    rid = env.new_replay(recorded, max_frames or frames)
    count = [0]
    every = max(1, frames // writes)

    def frame():
        env.record_replay(rid)
        count[0] += 1
        if writes > 1 and count[0] % every == 0:
            env.write_replay(rid, out_dir)
    drive(env, steps, seed + 7, frame, ops)
    written, dropped = env.write_replay(rid, out_dir)
    return env, rid, written, dropped


def read_dir(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def assert_same_files(want_dir, got_dir, what=""):
    want, got = read_dir(want_dir), read_dir(got_dir)
    assert sorted(want) == sorted(got), "%s: files %s, env_render wrote %s" % (what, sorted(got), sorted(want))
    for f in want:
        if want[f] != got[f]:
            a, b = want[f].split(b"\n"), got[f].split(b"\n")
            i = next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))
            raise AssertionError("%s %s: line %d differs: env_render %r, replay %r (%d and %d lines)"
                                 % (what, f, i, a[i] if i < len(a) else None, b[i] if i < len(b) else None,
                                    len(a), len(b)))


def check_against_render(make, lib, seed, arenas, recorded, steps, tmp, ops=None, writes=1, **kw):
    """record `recorded` in one run and render each of them in a run of its own; every file must match"""
    rec_dir = os.path.join(str(tmp), "replay")
    env, _rid, written, dropped = record_run(make, lib, seed, arenas, recorded, steps, rec_dir, ops=ops, writes=writes,
                                             **kw)
    assert dropped == 0
    for a in recorded:
        ren_dir = os.path.join(str(tmp), "render_%d" % a)
        render_run(make, lib, seed, arenas, a, steps, ren_dir, ops=ops, **kw)
        assert_same_files(ren_dir, os.path.join(rec_dir, "arena_%d" % a), "arena %d" % a)
    return env


def frames_of(path):
    """the frames of a video file, each a list of lines starting with its F line (the W block dropped)"""
    lines = open(path).read().split("\n")
    out, cur = [], None
    for ln in lines:
        if ln.startswith("F "):
            cur = [ln]
            out.append(cur)
        elif cur is not None and ln:
            cur.append(ln)
    return out


def has_wall_block(path):
    return open(path).read().startswith("W ")
