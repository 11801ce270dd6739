"""Measure the global-state kernel (magent_b200_get_global_state into a device tensor) on the battle512 workload.

    python profiles/global_state_bw.py [--calls 200] [--runs 2] [--out DIR]

Output per call: 512 * 200 * 200 * 5 elements (409.6 MB float32, 204.8 MB float16), plus the 512 * 200 * 200 kind bytes
(20.5 MB) the kernel reads.  Every timed window is `calls` back-to-back calls between two CUDA events, after a warm-up;
windows of the state kernel alternate with windows of `zero_()` on the same output tensor (a pure write stream of the
same bytes), `runs` times.  Prints the card name and power limit beside the numbers and one JSON line per dtype.
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
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    A, size, n = 512, 200, 1000
    env = pc.make_battle(pc.CUDA_LIB, size, n, 100, _num_arenas=A)
    for h in env.get_handles():                       # one step: agents below max hp load the hp_norm plane
        env.set_random_actions(h, 1)
    env.step()
    env.clear_dead()
    H, W, C = env.get_state_space()
    results = []
    for dtype in (torch.float32, torch.float16):
        out = torch.empty((A, H, W, C), dtype=dtype, device="cuda")
        state = lambda: env.get_global_state_torch(out=out)
        for _ in range(20):
            state()
            out.zero_()
        torch.cuda.synchronize()
        t_state, t_zero = [], []
        for _ in range(args.runs):
            t_state.append(window(state, args.calls))
            t_zero.append(window(out.zero_, args.calls))
        nbytes = out.numel() * out.element_size()
        ms, ms0 = min(t_state), min(t_zero)
        r = {"dtype": str(dtype).replace("torch.", ""), "card": card, "out_bytes": nbytes, "kind_bytes": A * H * W,
             "calls": args.calls, "runs": args.runs, "state_ms": [round(x, 4) for x in t_state],
             "zero_ms": [round(x, 4) for x in t_zero], "state_write_gbs": round(nbytes / ms / 1e6, 1),
             "state_gbs": round((nbytes + A * H * W) / ms / 1e6, 1),
             "zero_gbs": round(nbytes / ms0 / 1e6, 1), "ratio_to_zero": round(ms0 / ms, 3)}
        print("%s: %s  %.4f ms/call  %.1f GB/s  zero_() %.4f ms  %.1f GB/s  ratio %.3f" % (
            card, r["dtype"], ms, r["state_gbs"], ms0, r["zero_gbs"], r["ratio_to_zero"]))
        results.append(r)
    for r in results:
        print(json.dumps(r))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "global_state_bw.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
