"""Measure the slot-ordered step-loop calls on battle512 (512 arenas of 200 x 200, 2 x 1000 agents, S = 1000).

    python profiles/slot_loop_bw.py [--calls 20] [--runs 3] [--steps 5] [--out DIR]

After `steps` steps of random legal actions, each followed by clear_dead, every call below is timed per group in windows
of `calls` back-to-back calls between two CUDA events after a warm-up, the variants alternated in one process, `runs`
rounds each.  Each new call against the recipe of INTEGRATION.md it replaces, and against zero_() of the bytes it writes:
  * actions  set_action_slots(act [A, S])  vs  get_slots_torch + act.view(-1)[row_slot.clamp(min=0)] + env_set_action
             with the device pointer;
  * reward   get_reward_slots_torch(out=(reward, status))  vs  env_get_reward and env_get_info("alive") into device
             buffers + get_slots_torch + two torch.where gathers;
  * mask     get_action_mask_slots_torch(out=...)  vs  get_action_mask_torch(out=...) + get_slots_torch + a torch.where
             gather.
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


def variants(env, h):
    """{call: {variant: fn}} for one group, and the bytes each call writes"""
    import torch
    L, game, g = env._lib, env.game, env._hv(h)
    S, na, bound = env.get_slot_space(h), env.get_action_space(h)[0], env.get_num_bound(h)
    row_slot = torch.empty((bound,), dtype=torch.int32, device="cuda")
    slot_row = torch.empty((A, S), dtype=torch.int32, device="cuda")
    mask = env.get_action_mask_slots_torch(h)
    act = (torch.rand(mask.shape, device="cuda") * mask).argmax(-1).to(torch.int32)
    reward = torch.empty((A, S), dtype=torch.float32, device="cuda")
    status = torch.empty((A, S), dtype=torch.uint8, device="cuda")
    rrow = torch.empty((bound,), dtype=torch.float32, device="cuda")
    arow = torch.empty((bound,), dtype=torch.uint8, device="cuda")
    mrow = torch.empty((bound, na), dtype=torch.uint8, device="cuda")
    zero_act, zero_rs, zero_mask = (torch.empty((A * S * k,), dtype=torch.uint8, device="cuda") for k in (4, 5, na))

    def recipe_act():
        env.get_slots_torch(h, out=(row_slot, None))
        rows = act.view(-1)[row_slot.clamp(min=0)]
        L.env_set_action(game, g, rows.data_ptr())

    def recipe_reward():
        L.env_get_reward(game, g, rrow.data_ptr())
        L.env_get_info(game, g, b"alive", arow.data_ptr())
        env.get_slots_torch(h, out=(None, slot_row))
        occ, idx = slot_row >= 0, slot_row.clamp(min=0)
        return torch.where(occ, rrow[idx], 0.0), torch.where(occ, 2 - arow[idx], 0)

    def recipe_mask():
        env.get_action_mask_torch(h, out=mrow)
        env.get_slots_torch(h, out=(None, slot_row))
        return torch.where((slot_row >= 0).unsqueeze(-1), mrow[slot_row.clamp(min=0)], 0)

    calls = {
        "actions": {"slots": lambda: env.set_action_slots(h, act), "recipe": recipe_act, "zero": zero_act.zero_},
        "reward": {"slots": lambda: env.get_reward_slots_torch(h, out=(reward, status)), "recipe": recipe_reward,
                   "zero": zero_rs.zero_},
        "mask": {"slots": lambda: env.get_action_mask_slots_torch(h, out=mask), "recipe": recipe_mask,
                 "zero": zero_mask.zero_},
    }
    return calls, {"actions": A * S * 4, "reward": A * S * 5, "mask": A * S * na}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("slot_loop_bw.py measures on a CUDA device; none is visible")
    import parity_common as pc
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    env = pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=A)
    for t in range(args.steps):
        for h in env.get_handles():
            env.set_random_legal_actions(h, t)
        env.step()
        env.clear_dead()
    doc = {"card": card, "calls": args.calls, "runs": args.runs, "steps": args.steps, "results": []}
    for g, h in enumerate(env.get_handles()):
        S, n = env.get_slot_space(h), env.get_num(h)
        calls, nbytes = variants(env, h)
        for call, fns in calls.items():
            for fn in fns.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            ms = {k: [] for k in fns}
            for _ in range(args.runs):
                for k, fn in fns.items():
                    ms[k].append(round(window(fn, args.calls) * 1000.0, 1))
            for k, v in ms.items():
                print("%s: group %d %-7s %-6s us per call, rounds %s  (%d agents, S = %d, %d bytes)" % (
                    card, g, call, k, v, n, S, nbytes[call]))
            doc["results"].append({"group": g, "call": call, "agents": n, "slot_space": S, "bytes": nbytes[call],
                                   "call_us": ms})
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "slot_loop_bw.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
