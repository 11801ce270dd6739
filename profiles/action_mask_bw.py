"""Measure the legal-action mask and the legal draws on the battle512 workload (512 arenas of 2 x 1000 agents).

    python profiles/action_mask_bw.py [--calls 200] [--runs 3] [--steps 60] [--out DIR]

Part 1, the calls themselves, per group: windows of `calls` back-to-back calls between two CUDA events, after a warm-up,
alternating between get_action_mask_torch(out=...), zero_() of the same output tensor (a pure write of the same 21 MB),
set_random_legal_actions and set_random_actions; `runs` rounds, every round's figure reported.
Part 2, the step loop: `steps` steps driven by set_random_actions against `steps` steps driven by
set_random_legal_actions, alternating in rounds on two games that start from the same placement: ms per step (set
actions + step + clear_dead between CUDA events) and hits / kills per step from get_counters.  Legal draws make the
fight denser, so the step itself does more work: that is the workload changing, reported apart from part 1.
Prints the card, its power limit and SM clocks beside the numbers, and one JSON document.
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
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("action_mask_bw.py measures on a CUDA device; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    A, size, n = 512, 200, 1000
    make = lambda: pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=A)
    env = make()
    hs = env.get_handles()
    for t in range(5):                                   # a few steps: armies have met, some agents are dead
        for h in hs:
            env.set_random_actions(h, t)
        env.step()
        env.clear_dead()
    h = hs[0]
    rows, na = env.get_num_bound(h), env.get_action_space(h)[0]
    out = torch.empty((rows, na), dtype=torch.uint8, device="cuda")
    variants = {"mask": lambda: env.get_action_mask_torch(h, out=out), "zero": out.zero_,
                "legal_draw": lambda: env.set_random_legal_actions(h, 3), "uniform_draw": lambda: env.set_random_actions(h, 3)}
    for fn in variants.values():
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    calls_ms = {k: [] for k in variants}
    for _ in range(args.runs):
        for k, fn in variants.items():
            calls_ms[k].append(round(window(fn, args.calls), 5))
    agents = env.get_num(h)
    for k, v in calls_ms.items():
        print("%s: %-12s ms per call and group, rounds %s  (%d agents, %d mask bytes)" % (card, k, v, agents, agents * na))
    del env

    loops = {"uniform": (make(), "set_random_actions"), "legal": (make(), "set_random_legal_actions")}
    step_ms = {k: [] for k in loops}
    per_step = {k: [] for k in loops}
    t0 = 0
    for r in range(args.runs + 1):                       # round 0 warms up and is dropped
        for k, (e, setter) in loops.items():
            c0 = e.get_counters()

            def one(e=e, setter=setter):
                nonlocal t0
                t0 += 1
                for hh in e.get_handles():
                    getattr(e, setter)(hh, t0)
                e.step()
                e.clear_dead()
            ms = window(one, args.steps)
            c1 = e.get_counters()
            if r:
                step_ms[k].append(round(ms, 4))
                per_step[k].append({"hits": round((c1[2] - c0[2]) / args.steps, 1), "kills": round((c1[3] - c0[3]) / args.steps, 1),
                                    "agents_left": sum(e.get_num(hh) for hh in e.get_handles())})
    for k in loops:
        print("%s: step loop with %-8s draws  ms per step, rounds %s  %s" % (card, k, step_ms[k], per_step[k]))
    doc = {"card": card, "agents_per_group": agents, "n_action": na, "calls": args.calls, "runs": args.runs,
           "call_ms": calls_ms, "steps": args.steps, "step_ms": step_ms, "per_step": per_step}
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "action_mask_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
