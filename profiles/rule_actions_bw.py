"""Measure the built-in scripted opponents on the battle512 workload (512 arenas of 2 x 1000 agents).

    python profiles/rule_actions_bw.py [--calls 200] [--runs 3] [--out DIR]

After 5 steps of uniform random actions, per group against the other: windows of `calls` back-to-back calls between two
CUDA events, after a warm-up, alternating between set_rule_actions (in place) and get_rule_actions_slots_torch (into a
fixed (A, S) tensor) for rush and for flee, and, for scale, set_random_legal_actions and get_neighbours_torch(k=1, of=the
enemy, out=(idx, None, None)); `runs` rounds, every round's figure reported.  Also the share of agents that see an enemy and the
mean number of legal actions.  Prints the card, its power limit and SM clocks beside the numbers, and one
JSON document.
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
        sys.exit("rule_actions_bw.py measures on a CUDA device; none is visible")
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
        rows, S = env.get_num_bound(h), env.get_slot_space(h)
        slots = torch.empty((A, S), dtype=torch.int32, device="cuda")
        idx = torch.empty((rows, 1), dtype=torch.int32, device="cuda")
        variants = {"rush_in_place": lambda: env.set_rule_actions(h, enemy, "rush", 1),
                    "rush_slots": lambda: env.get_rule_actions_slots_torch(h, enemy, "rush", 1, out=slots),
                    "flee_in_place": lambda: env.set_rule_actions(h, enemy, "flee", 1),
                    "flee_slots": lambda: env.get_rule_actions_slots_torch(h, enemy, "flee", 1, out=slots),
                    "random_legal_actions": lambda: env.set_random_legal_actions(h, 1),
                    "neighbours_k1_enemy": lambda: env.get_neighbours_torch(h, 1, enemy, out=(idx, None, None))}
        for fn in variants.values():
            for _ in range(20):
                fn()
        torch.cuda.synchronize()
        calls_ms = {k: [] for k in variants}
        for _ in range(args.runs):
            for k, fn in variants.items():
                calls_ms[k].append(round(window(fn, args.calls), 5))
        agents = env.get_num(h)
        mask = env.get_action_mask_torch(h)
        seen = env.get_neighbours_torch(h, 1, enemy, out=(idx, None, None))[0][:, 0] >= 0
        share = {"sees_an_enemy": round(float(seen.double().mean()), 4),
                 "legal_actions_per_agent": round(float(mask.double().sum(1).mean()), 3)}
        for k, v in calls_ms.items():
            print("%s: group %d %-22s ms per call, rounds %s  (%d agents, S = %d)" % (card, g, k, v, agents, S))
        print("%s: group %d %s" % (card, g, share))
        doc["groups"].append({"group": g, "agents": agents, "slot_space": S, "call_ms": calls_ms, "state": share})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rule_actions_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
