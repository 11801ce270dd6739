"""Measure the slot-ordered mean action and neighbours on battle512 (512 arenas of 200 x 200, 2 x 1000 agents, S = 1000).

    python profiles/nbr_slots_bw.py [--calls 20] [--runs 3] [--steps 5] [--out DIR]

After `steps` steps of random legal actions, each followed by clear_dead, every call below is timed per group, for
`of` = its own group and the enemy and (neighbours) k = 3 and 32, in windows of `calls` back-to-back calls between two
CUDA events after a warm-up, the variants alternated in one process, `runs` rounds each:
  * slots   get_mean_action_slots / get_neighbours_slots into device buffers;
  * rows    the row-ordered call into device buffers (the raw ABI call, which never waits for the counts);
  * recipe  what the slot call replaces: the row call, get_slots_torch of the group (and, for neighbours, of `of`) and
            the torch gathers that bring the rows into slot order and the neighbour rows to flat slots;
  * zero    zero_() of the bytes the slot call writes.
Prints the card, its power limit and SM clocks beside the numbers, and one JSON document.
"""
import argparse
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


def variants(env, h, o, k):
    """{call: {variant: fn}} for group h over group o, and the bytes each slot call writes"""
    import torch
    L, game, g, of = env._lib, env.game, env._hv(h), env._hv(o)
    S, na, bound, bound_of = env.get_slot_space(h), env.get_action_space(o)[0], env.get_num_bound(h), env.get_num_bound(o)
    i32 = torch.int32
    dev = dict(device="cuda")
    mean, count = torch.empty((A, S, na), **dev), torch.empty((A, S), dtype=i32, **dev)
    idx, rel, ncount = (torch.empty((A, S) + t, dtype=i32, **dev) for t in ((k,), (k, 2), ()))
    mrow, crow = torch.empty((bound, na), **dev), torch.empty((bound,), dtype=i32, **dev)
    irow, rrow, nrow = (torch.empty((bound,) + t, dtype=i32, **dev) for t in ((k,), (k, 2), ()))
    row_slot_of = torch.empty((bound_of,), dtype=i32, **dev)
    slot_row = torch.empty((A, S), dtype=i32, **dev)
    zero_mean = torch.empty((A * S * (na + 1) * 4,), dtype=torch.uint8, **dev)
    zero_nbr = torch.empty((A * S * (3 * k + 1) * 4,), dtype=torch.uint8, **dev)

    def row_mean():
        L.magent_b200_get_mean_action(game, g, of, mrow.data_ptr(), crow.data_ptr())

    def row_nbr():
        L.magent_b200_get_neighbours(game, g, of, k, irow.data_ptr(), rrow.data_ptr(), nrow.data_ptr())

    def recipe_mean():
        row_mean()
        env.get_slots_torch(h, out=(None, slot_row))
        occ, rows = slot_row >= 0, slot_row.clamp(min=0)
        return torch.where(occ.unsqueeze(-1), mrow[rows], 0.0), torch.where(occ, crow[rows], 0)

    def recipe_nbr():
        row_nbr()
        env.get_slots_torch(h, out=(None, slot_row))
        env.get_slots_torch(o, out=(row_slot_of, None))
        occ, rows = slot_row >= 0, slot_row.clamp(min=0)
        ir = irow[rows]
        i = torch.where(occ.unsqueeze(-1) & (ir >= 0), row_slot_of[ir.clamp(min=0)], -1)
        return i, torch.where(occ[..., None, None], rrow[rows], -1), torch.where(occ, nrow[rows], 0)

    calls = {
        "mean": {"slots": lambda: env.get_mean_action_slots_torch(h, o, out=(mean, count)), "rows": row_mean,
                 "recipe": recipe_mean, "zero": zero_mean.zero_},
        "neighbours": {"slots": lambda: env.get_neighbours_slots_torch(h, k, o, out=(idx, rel, ncount)), "rows": row_nbr,
                       "recipe": recipe_nbr, "zero": zero_nbr.zero_},
    }
    return calls, {"mean": zero_mean.numel(), "neighbours": zero_nbr.numel()}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nbr_slots_bw.py measures on a CUDA device; none is visible")
    import parity_common as pc
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    env = pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=A)
    for t in range(args.steps):
        for h in env.get_handles():
            env.set_random_legal_actions(h, t)
        env.step()
        env.clear_dead()
    hs = env.get_handles()
    doc = {"card": card, "calls": args.calls, "runs": args.runs, "steps": args.steps, "results": []}
    for g, h in enumerate(hs):
        for which, o in (("own", h), ("enemy", hs[1 - g])):
            for k in (3, 32):
                S, n = env.get_slot_space(h), env.get_num(h)
                calls, nbytes = variants(env, h, o, k)
                if k == 32:
                    del calls["mean"]                  # the mean action has no k: measured once, with k = 3
                for call, fns in calls.items():
                    for fn in fns.values():
                        for _ in range(3):
                            fn()
                    torch.cuda.synchronize()
                    ms = {v: [] for v in fns}
                    for _ in range(args.runs):
                        for v, fn in fns.items():
                            ms[v].append(round(window(fn, args.calls) * 1000.0, 1))
                    for v, t in ms.items():
                        print("%s: group %d of %-5s %-10s k %2s %-6s us per call, rounds %s  (%d agents, S = %d, %d bytes)"
                              % (card, g, which, call, k if call == "neighbours" else "-", v, t, n, S, nbytes[call]))
                    doc["results"].append({"group": g, "of": which, "call": call, "k": k if call == "neighbours" else None,
                                           "agents": n, "slot_space": S, "bytes": nbytes[call], "call_us": ms})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "nbr_slots_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
