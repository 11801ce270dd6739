"""Measure the slot-ordered observation on battle512 (512 arenas of 200 x 200, 2 x 1000 agents).

    python profiles/obs_slots_bw.py [--calls 5] [--runs 3] [--states fresh,ragged,blocks] [--out DIR]

Three calls per group, timed in windows of `calls` back-to-back calls between two CUDA events after a warm-up, and
alternated in one process, `runs` rounds each:
  * slots   get_observation_slots_torch(out=...): the [A, S] records rendered in slot order;
  * rows    get_observation_torch(out=...): the same group's row-ordered observation;
  * recipe  INTEGRATION.md's gather: the row-ordered observation, get_slots_torch, then the view and the feature rows
            gathered with slot_row and multiplied by the vacancy mask.
In three states of the batch, float32 and float16:
  (a) fresh   battle512 right after placement: every slot occupied;
  (b) ragged  arena 0 holds 1000 agents per group and every other arena 500 (select_arena): half of their slots are
              vacant, in one run at the end of the arena;
  (c) blocks  battle512_blocks after 200 steps of random legal actions, each followed by clear_dead: the vacant
              slots of the dead lie scattered between live ones (a render CTA meets vacant <-> live changes, which
              rebuild its tile).
Prints the card, its power limit and SM clocks beside the numbers, and one JSON document.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

A = 512


def window(fn, calls):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def fresh():
    import parity_common as pc
    return pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=A)


def ragged():
    import magent_b200 as magent
    import parity_common as pc
    env = magent.GridWorld("battle", map_size=200, _lib=pc.CUDA_LIB, _num_arenas=A)
    env.set_seed(100)
    env.reset()
    for a in range(A):
        env.select_arena(a)
        for h in env.get_handles():
            env.add_agents(h, method="random", n=1000 if a == 0 else 500)
    env.select_arena(-1)
    return env


def blocks():
    import parity_common as pc
    env = pc.make_battle_blocks(pc.CUDA_LIB, 200, _num_arenas=A)
    for t in range(200):
        for h in env.get_handles():
            env.set_random_legal_actions(h, t)
        env.step()
        env.clear_dead()
    return env


def measure(env, state, card, calls, runs):
    import torch
    out = []
    for g, h in enumerate(env.get_handles()):
        S = env.get_slot_space(h)
        rs, slot_row = env.get_slots_torch(h)
        n = env.get_num(h)
        vacant = int((slot_row < 0).sum())
        for dt in (torch.float32, torch.float16):
            sv, sf = env.get_observation_slots_torch(h, dtype=dt)
            rv, rf = env.get_observation_torch(h, dtype=dt)

            def recipe():
                env.get_observation_torch(h, out=(rv, rf))
                env.get_slots_torch(h, out=(rs, slot_row))
                idx = slot_row.clamp(min=0).view(-1)
                keep = (slot_row >= 0).unsqueeze(-1).to(dt)
                gv = rv[idx].view((A, S, -1)) * keep
                gf = rf[idx].view((A, S, -1)) * keep
                return gv, gf
            variants = {"slots": lambda: env.get_observation_slots_torch(h, out=(sv, sf)),
                        "rows": lambda: env.get_observation_torch(h, out=(rv, rf)),
                        "recipe": recipe}
            for fn in variants.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            ms = {k: [] for k in variants}
            for _ in range(runs):
                for k, fn in variants.items():
                    ms[k].append(round(window(fn, calls), 4))
            esz = 2 if dt == torch.float16 else 4
            slot_bytes = (sv.numel() + sf.numel()) * esz
            row_bytes = (rv.numel() + rf.numel()) * esz
            name = "f16" if dt == torch.float16 else "f32"
            for k, v in ms.items():
                print("%s: %-6s group %d %s %-6s ms per call, rounds %s  (%d agents, %d of %d slots vacant)" % (
                    card, state, g, name, k, v, n, vacant, A * S))
            out.append({"state": state, "group": g, "dtype": name, "agents": n, "slot_space": S, "vacant_slots": vacant,
                        "slot_bytes": slot_bytes, "row_bytes": row_bytes, "call_ms": ms})
            del sv, sf, rv, rf
            gc.collect()
            torch.cuda.empty_cache()
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--states", default="fresh,ragged,blocks")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("obs_slots_bw.py measures on a CUDA device; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    doc = {"card": card, "calls": args.calls, "runs": args.runs, "results": []}
    makers = {"fresh": fresh, "ragged": ragged, "blocks": blocks}
    for state in args.states.split(","):
        make = makers[state]
        env = make()
        doc["results"] += measure(env, state, card, args.calls, args.runs)
        del env
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "obs_slots_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
