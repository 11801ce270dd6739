"""Measure the mean neighbour action on the battle512 workload (512 arenas of 2 x 1000 agents).

    python profiles/mean_action_bw.py [--calls 200] [--runs 3] [--out DIR]

After 5 steps of uniform random actions, per group: windows of `calls` back-to-back calls between two CUDA events,
after a warm-up, alternating between get_mean_action_torch(of=own group, out=...), get_mean_action_torch(of=the enemy,
out=...), zero_() of the same mean and count tensors (a pure write of the same bytes) and get_observation_torch of the
same group (the render, for scale); `runs` rounds, every round's figure reported.  Also the neighbours counted per
observer.  Prints the card, its power limit and SM clocks beside the numbers, and one JSON document.
"""
import argparse
import json
import os
import subprocess
import sys

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
    import parity_common as pc
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mean_action_bw.py measures on a CUDA device; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    A, size, n = 512, 200, 1000
    env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=A)
    hs = env.get_handles()
    for t in range(5):                                   # a few steps: armies have met, some agents are dead
        for h in hs:
            env.set_random_actions(h, t)
        env.step()
        env.clear_dead()
    doc = {"card": card, "calls": args.calls, "runs": args.runs, "groups": []}
    for g, h in enumerate(hs):
        enemy = hs[1 - g]
        rows, na = env.get_num_bound(h), env.get_action_space(h)[0]
        mean = torch.empty((rows, na), dtype=torch.float32, device="cuda")
        count = torch.empty((rows,), dtype=torch.int32, device="cuda")
        view = torch.empty((rows,) + env.view_space[g], dtype=torch.float32, device="cuda")
        feat = torch.empty((rows,) + env.feature_space[g], dtype=torch.float32, device="cuda")

        def zero():
            mean.zero_()
            count.zero_()
        variants = {"mean_own": lambda: env.get_mean_action_torch(h, h, out=(mean, count)),
                    "mean_enemy": lambda: env.get_mean_action_torch(h, enemy, out=(mean, count)),
                    "zero": zero,
                    "observation": lambda: env.get_observation_torch(h, out=(view, feat))}
        for fn in variants.values():
            for _ in range(20):
                fn()
        torch.cuda.synchronize()
        calls_ms = {k: [] for k in variants}
        for _ in range(args.runs):
            for k, fn in variants.items():
                calls_ms[k].append(round(window(fn, args.calls), 5))
        agents = env.get_num(h)
        nbrs = {}
        for k, of in (("own", h), ("enemy", enemy)):
            _m, c = env.get_mean_action_torch(h, of)
            nbrs[k] = round(float(c.double().mean()), 3)
        for k, v in calls_ms.items():
            print("%s: group %d %-12s ms per call, rounds %s  (%d agents, %d mean + count bytes)" % (
                card, g, k, v, agents, agents * (na + 1) * 4))
        print("%s: group %d neighbours per observer %s" % (card, g, nbrs))
        doc["groups"].append({"group": g, "agents": agents, "n_action": na, "call_ms": calls_ms,
                              "neighbours_per_observer": nbrs})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mean_action_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
