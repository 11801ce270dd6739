"""Measure the stable agent slots on the battle512 workload (512 arenas of 2 x 1000 agents).

    python profiles/slots_bw.py [--calls 200] [--runs 3] [--out DIR]

After 5 steps of uniform random actions, per group: windows of `calls` back-to-back calls between two CUDA events,
after a warm-up, alternating between get_slots_torch(out=(row_slot, slot_row)), zero_() of the same two tensors (a pure
write of the same bytes) and the torch scatter of the group's float32 observations into [A, S] that INTEGRATION.md §4
does with them (view only: obs[slot_row.clamp(min=0).view(-1)] * (slot_row >= 0)); `runs` rounds, every round's figure
reported.  Prints the card, its power limit and SM clocks beside the numbers, and one JSON document.
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
        sys.exit("slots_bw.py measures on a CUDA device; none is visible")
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
        rows, S = env.get_num_bound(h), env.get_slot_space(h)
        row_slot = torch.empty((rows,), dtype=torch.int32, device="cuda")
        slot_row = torch.empty((A, S), dtype=torch.int32, device="cuda")
        env.get_slots_torch(h, out=(row_slot, slot_row))
        obs = env.get_observation_torch(h)[0]
        keep = (slot_row >= 0).view(-1, 1, 1, 1)
        index = slot_row.clamp(min=0).view(-1)

        def zero():
            row_slot.zero_()
            slot_row.zero_()
        variants = {"get_slots": lambda: env.get_slots_torch(h, out=(row_slot, slot_row)),
                    "zero_same_bytes": zero,
                    "scatter_obs_f32": lambda: obs[index] * keep}
        for fn in variants.values():
            for _ in range(20):
                fn()
        torch.cuda.synchronize()
        calls_ms = {k: [] for k in variants}
        for _ in range(args.runs):
            for k, fn in variants.items():
                calls_ms[k].append(round(window(fn, args.calls), 5))
        agents = env.get_num(h)
        out_bytes = (rows + A * S) * 4
        obs_bytes = A * S * obs[0].numel() * 4
        for k, v in calls_ms.items():
            print("%s: group %d %-16s ms per call, rounds %s  (%d agents)" % (card, g, k, v, agents))
        print("%s: group %d get_slots writes %d bytes; the observation scatter writes %d" % (card, g, out_bytes, obs_bytes))
        doc["groups"].append({"group": g, "agents": agents, "slot_space": S, "num_bound": rows, "call_ms": calls_ms,
                              "slots_bytes": out_bytes, "scatter_bytes": obs_bytes})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "slots_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
