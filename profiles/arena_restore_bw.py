"""Measure restore_arenas (the reset pool) on the battle512 workload against the host route of a new episode.

    python profiles/arena_restore_bw.py [--calls 50] [--runs 2] [--out DIR]

512 arenas of battle 200x200 with 2 x 1000 agents, snapshotted right after placement, then 20 random steps so that the
live arenas differ from the snapshot.  Three restores from a device src (a CUDA tensor), each timed as `calls`
back-to-back calls between two CUDA events, after a warm-up:
  none   src = -1 everywhere: the cost of a call that restores nothing;
  5%     26 arenas;
  all    every arena from itself.
Bytes moved by one restored arena (read + written): occ (read, written) and claim_head (written) planes of
4 * 200 * 200 bytes, the padded kind (1 byte per cell) and hp_norm (4 bytes) planes of 212 * 212 cells (battle's view
radius 6 pads the map by 6 cells), and 35 bytes per agent record (8 four-byte and 3 one-byte fields) read and written.
The effective rate of the full restore is set against `zero_()` of the same number of bytes.  The host route is
env_reset + add_agents of 2 x 1000 agents into every arena + the first env_step (which uploads the whole image).
Prints the card name and power limit beside the numbers and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
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
    import numpy as np
    import torch
    import parity_common as pc
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    A, size, n, pad = 512, 200, 1000, 6
    env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=A)
    hs = env.get_handles()
    pool = env.snapshot_arenas()
    for t in range(20):
        for h in hs:
            env.set_random_actions(h, t)
        env.step()
        env.clear_dead()
    torch.cuda.synchronize()
    cells, kcells = size * size, (size + 2 * pad) ** 2
    arena_bytes = 2 * 4 * cells + 4 * cells + 2 * kcells + 2 * 4 * kcells + 2 * 2 * n * 35
    rs = np.random.RandomState(0)
    five = np.full((A,), -1, np.int32)
    pick = rs.choice(A, 26, replace=False)
    five[pick] = pick
    cases = {"none": (np.full((A,), -1, np.int32), 0), "5%": (five, 26), "all": (np.arange(A, dtype=np.int32), A)}
    res = {"card": card, "arenas": A, "arena_bytes": arena_bytes, "calls": args.calls, "runs": args.runs}
    for name, (src, k) in cases.items():
        d = torch.from_numpy(src).cuda()
        call = lambda: env.restore_arenas(pool, d)
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        ts = [window(call, args.calls) for _ in range(args.runs)]
        ms = min(ts)
        res[name] = {"arenas": k, "ms": [round(x, 4) for x in ts], "gbs": round(k * arena_bytes / ms / 1e6, 1)}
        print("%s: restore %-4s (%3d arenas)  %.4f ms/call  %.1f GB/s" % (card, name, k, ms, res[name]["gbs"]))
    z = torch.empty((A * arena_bytes,), dtype=torch.uint8, device="cuda")
    for _ in range(5):
        z.zero_()
    ms0 = min(window(z.zero_, args.calls) for _ in range(args.runs))
    res["zero_ms"] = round(ms0, 4)
    res["zero_gbs"] = round(A * arena_bytes / ms0 / 1e6, 1)
    res["all_ratio_to_zero"] = round(ms0 / min(res["all"]["ms"]), 3)
    print("%s: zero_() of the same %.1f MB  %.4f ms  %.1f GB/s  (full restore at %.3f of it)" % (
        card, A * arena_bytes / 1e6, ms0, res["zero_gbs"], res["all_ratio_to_zero"]))
    # the host route: a new episode for every arena through reset, host placement and the upload of the first step
    host = []
    for r in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        env.reset()
        for h in hs:
            env.add_agents(h, method="random", n=n)
        for h in hs:
            env.set_random_actions(h, 100 + r)
        env.step()
        env.sync()
        host.append((time.perf_counter() - t0) * 1e3)
        env.clear_dead()
    res["host_route_ms"] = [round(x, 1) for x in host]
    print("%s: reset + add_agents + first step  %.1f ms  (%.0fx the full restore)" % (
        card, min(host), min(host) / min(res["all"]["ms"])))
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "arena_restore_bw.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
