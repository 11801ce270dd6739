"""Measure the replay recorder on the battle512 workload (512 arenas of 2 x 1000 agents, device-drawn legal actions).

    python profiles/replay_bw.py [--steps 50] [--runs 3] [--out DIR]

Per configuration, `steps` steps between two CUDA events after a warm-up, `runs` rounds: the loop (legal actions drawn
on the device for both groups, env_step with a device `done`, clear_dead) with no recorder, and with a recorder of 1, 8
and 64 arenas calling record_replay after every step, both eager and replayed as a CUDA graph of two steps.  Also ms
per record_replay call alone and bytes per recorded frame, and, for contrast, ms per step of the eager loop with
env_render of one arena after every step (a host clock around synchronised steps: env_render synchronises).  Prints
the card, its power limit and SM clocks beside the numbers, and one JSON document.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def window(fn, calls):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    import torch
    import bench
    import parity_common as pc
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("replay_bw.py measures on a CUDA device; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    wl = bench.WORKLOADS["battle512"]
    A = wl["arenas"]
    doc = {"card": card, "steps": args.steps, "runs": args.runs, "step_ms": {}, "record_ms": {}, "frame_bytes": {}}
    tmp = tempfile.mkdtemp()
    for k in (0, 1, 8, 64):
        for graph in (False, True):
            env = bench.build_env(wl, pc.CUDA_LIB, A, seed0=1)[0]
            hs = env.get_handles()
            done = torch.zeros(1, dtype=torch.int32, device="cuda")
            rid = env.new_replay(list(range(0, A, A // k))[:k], 2 * args.steps + 8) if k else None

            def step(t=[0]):
                t[0] += 1
                for g, h in enumerate(hs):
                    env.set_random_legal_actions(h, 2 * t[0] + g)
                env.step_device_done(done.data_ptr())
                env.clear_dead()
                if k:
                    env.record_replay(rid)
            fn = step
            if graph:
                gid = env.capture_graph(lambda: (step(), step()))
                fn = lambda: env.launch_graph(gid)      # noqa: E731
            per = 2 if graph else 1
            for _ in range(4):
                fn()
            ms = []
            for _ in range(args.runs):
                if k:
                    env.write_replay(rid, tmp)
                ms.append(round(window(fn, max(1, args.steps // per)) / per, 4))
            key = "%s_%d_arenas" % ("graph" if graph else "eager", k)
            doc["step_ms"][key] = ms
            print("%s: battle512 step with a recorder of %2d arenas, %s: %s ms" % (card, k, "graph" if graph else "eager", ms))
            if k and not graph:
                env.write_replay(rid, tmp)
                rec = [round(window(lambda: env.record_replay(rid), args.steps), 4) for _ in range(args.runs)]
                env.write_replay(rid, tmp)
                doc["record_ms"]["%d_arenas" % k] = rec
                print("%s: record_replay of %2d arenas: %s ms per call" % (card, k, rec))
            del env
            torch.cuda.synchronize()
    # bytes per frame of one arena: header, cap_total agent rows (20 B) and event rows (16 B), the wall bitmap
    env = bench.build_env(wl, pc.CUDA_LIB, A, seed0=1)[0]
    cap = sum(max(64, (int(env.get_arena_nums(h).max()) + 63) // 64 * 64) for h in env.get_handles())
    words = (wl["map_size"] ** 2 + 127) // 128 * 4
    doc["frame_bytes"] = {"per_arena": 128 + 36 * cap + 4 * words, "cap_total": cap}
    print("%s: one recorded frame of one arena: %d bytes (cap_total %d)" % (card, doc["frame_bytes"]["per_arena"], cap))
    hs = env.get_handles()
    env.select_arena(0)
    env.set_render_dir(os.path.join(tmp, "render"))
    render_steps = max(3, args.steps // 10)
    ms = []
    for _ in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(render_steps):
            for g, h in enumerate(hs):
                env.set_random_legal_actions(h, 7 * t + g)
            env.step()
            env.clear_dead()
            env.render()
        torch.cuda.synchronize()
        ms.append(round((time.perf_counter() - t0) * 1e3 / render_steps, 3))
    doc["step_ms"]["eager_env_render_1_arena"] = ms
    print("%s: battle512 step with env_render of one arena: %s ms" % (card, ms))
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "replay_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
