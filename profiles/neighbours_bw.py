"""Measure the nearest visible neighbours on the battle512 workload (512 arenas of 2 x 1000 agents).

    python profiles/neighbours_bw.py [--calls 200] [--runs 3] [--out DIR]

After 5 steps of uniform random actions, per group: windows of `calls` back-to-back calls between two CUDA events,
after a warm-up, alternating between get_neighbours_torch(k=3, own group, out=(idx, rel, count)), the same without
count (the kernel stops at the third neighbour), get_neighbours_torch(k=32, of=the enemy, out=(idx, rel, count)),
get_mean_action_torch of the same group (for scale) and zero_() of the k = 32 outputs (a pure write of the same bytes);
`runs` rounds, every round's figure reported.  Also the neighbours per observer.  Prints the card, its power limit and
SM clocks beside the numbers, and one JSON document.
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
        sys.exit("neighbours_bw.py measures on a CUDA device; none is visible")
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
        i3 = torch.empty((rows, 3), dtype=torch.int32, device="cuda")
        r3 = torch.empty((rows, 3, 2), dtype=torch.int32, device="cuda")
        i32 = torch.empty((rows, 32), dtype=torch.int32, device="cuda")
        r32 = torch.empty((rows, 32, 2), dtype=torch.int32, device="cuda")
        count = torch.empty((rows,), dtype=torch.int32, device="cuda")
        mean = torch.empty((rows, na), dtype=torch.float32, device="cuda")

        def zero():
            i32.zero_()
            r32.zero_()
            count.zero_()
        variants = {"k3_own": lambda: env.get_neighbours_torch(h, 3, h, out=(i3, r3, count)),
                    "k3_own_no_count": lambda: env.get_neighbours_torch(h, 3, h, out=(i3, r3, None)),
                    "k32_enemy": lambda: env.get_neighbours_torch(h, 32, enemy, out=(i32, r32, count)),
                    "mean_action_own": lambda: env.get_mean_action_torch(h, h, out=(mean, count)),
                    "zero_k32": zero}
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
            c = env.get_neighbours_torch(h, 1, of)[2]
            nbrs[k] = round(float(c.double().mean()), 3)
        for k, v in calls_ms.items():
            print("%s: group %d %-16s ms per call, rounds %s  (%d agents)" % (card, g, k, v, agents))
        print("%s: group %d neighbours per observer %s; k = 32 writes %d bytes" % (card, g, nbrs, agents * (3 * 32 + 1) * 4))
        doc["groups"].append({"group": g, "agents": agents, "call_ms": calls_ms, "neighbours_per_observer": nbrs})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "neighbours_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
