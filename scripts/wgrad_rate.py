#!/usr/bin/env python
"""Before / after of the 32-channel weight-gradient convolution, in one run on one GPU.

    python scripts/wgrad_rate.py --before DIR [--reps 3] [--skip-bench] [--skip-timeline]

DIR is a second, already built copy of this repository inside the working tree (for example the parent commit exported
with `git archive` into a git-ignored directory and built there with `python disentangling-vae_b200/build.py`); "after"
is the tree this script lies in.  Absolute times move by several percent between sessions, so only the comparisons
inside one run count.  Steps:

1. the card's name, power limit and maximum SM clock (read-only nvidia-smi query);
2. per build, in child processes, alternating before / after --reps times: CUDA events around 50 back-to-back
   ops.conv_wgrad calls (kernel + split-K reduce) after 5 warm-up calls, 5 repeats, at B = 1024 and lo 16, 8, 4, and at
   B = 512 and 256 for lo 16; min-max over all repeats in us per call, and the algorithmic TFLOP/s
   (2 * B * H^2 * 32 * 16 * 32 FLOP per call) at the fastest repeat;
3. per build, alternating --reps times: bench.py --steps 200 --warmup 20 at c2, then once each at c1, c3 and c5:
   ms_per_step and parity.ok;
4. once for the after build: the per-stream timeline of one replayed c2 step (scripts/step_timeline.py).

One JSON line with everything, then Markdown tables.  Exits non-zero without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1024, 16), (1024, 8), (1024, 4), (512, 16), (256, 16)]
CALLS, WARMUP, REPEATS = 50, 5, 5


def flop(B, H):
    return 2 * B * H * H * 32 * 16 * 32


def time_kernels(root):
    """Child: us per ops.conv_wgrad call of the build at `root`, REPEATS times per shape."""
    sys.path[:0] = [root, os.path.join(root, "disentangling-vae_b200")]
    import torch
    from disvae import ops
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    out = {}
    for B, H in SHAPES:
        hi = torch.randn(B, 2 * H, 2 * H, 32, device=dev)
        lo = torch.randn(B, H, H, 32, device=dev)
        for _ in range(WARMUP):
            ops.conv_wgrad(lo, hi, B, H, H, 32, 0, True)
        us = []
        for _ in range(REPEATS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(CALLS):
                ops.conv_wgrad(lo, hi, B, H, H, 32, 0, True)
            e1.record()
            torch.cuda.synchronize()
            us.append(e0.elapsed_time(e1) / CALLS * 1e3)
        out["B%d_lo%d" % (B, H)] = us
    print(json.dumps(out), flush=True)


def child(cmd, cwd):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        sys.exit("%s failed in %s:\n%s%s" % (" ".join(cmd), cwd, r.stdout[-2000:], r.stderr[-4000:]))
    return r.stdout


def last_json(text):
    return json.loads([ln for ln in text.splitlines() if ln.startswith("{")][-1])


def bench(root, workload):
    out = last_json(child([sys.executable, "bench.py", "--gpus", "1", "--steps", "200", "--warmup", "20", "--workload", workload,
                           "--no-cpu-baseline", "--no-eager-baseline"], root))
    return {"ms_per_step": out["ms_per_step"], "parity_ok": out["parity"]["ok"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--before", help="root of the built copy to compare against")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-bench", action="store_true")
    ap.add_argument("--skip-timeline", action="store_true")
    ap.add_argument("--time-kernels", metavar="ROOT", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("wgrad_rate.py needs a GPU")
    if args.time_kernels:
        return time_kernels(args.time_kernels)
    if not args.before:
        ap.error("--before is required")
    builds = [("before", os.path.abspath(args.before)), ("after", ROOT)]
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    res = {"card": q, "calls": CALLS, "repeats": REPEATS, "reps": args.reps, "kernel_us": {}, "bench": {}}
    print("card (name, power limit, max SM clock):", q, flush=True)

    kernel = {name: {} for name, _ in builds}
    for _ in range(args.reps):
        for name, root in builds:
            got = last_json(child([sys.executable, os.path.abspath(__file__), "--time-kernels", root], root))
            for k, us in got.items():
                kernel[name].setdefault(k, []).extend(us)
    res["kernel_us"] = kernel
    print("\n| B, lo | before us / call (min-max) | after us / call (min-max) | after / before (min) | after TFLOP/s |")
    print("|---|---|---|---|---|")
    for B, H in SHAPES:
        k = "B%d_lo%d" % (B, H)
        b, a = kernel["before"][k], kernel["after"][k]
        print("| %d, %d | %.1f-%.1f | %.1f-%.1f | %.3f | %.1f |" % (B, H, min(b), max(b), min(a), max(a), min(a) / min(b),
                                                                 flop(B, H) / min(a) * 1e-6), flush=True)

    if not args.skip_bench:
        runs = {name: {"c2": []} for name, _ in builds}
        for _ in range(args.reps):
            for name, root in builds:
                runs[name]["c2"].append(bench(root, "c2"))
        for w in ("c1", "c3", "c5"):
            for name, root in builds:
                runs[name][w] = [bench(root, w)]
        res["bench"] = runs
        print("\n| workload | before ms/step | after ms/step | parity.ok (before, after) |")
        print("|---|---|---|---|")
        for w in ("c2", "c1", "c3", "c5"):
            b, a = runs["before"][w], runs["after"][w]
            print("| %s | %s | %s | %s, %s |" % (w, ", ".join("%.4f" % r["ms_per_step"] for r in b),
                                                ", ".join("%.4f" % r["ms_per_step"] for r in a),
                                                all(r["parity_ok"] for r in b), all(r["parity_ok"] for r in a)), flush=True)
    print("\n" + json.dumps(res), flush=True)
    if not args.skip_timeline:
        print("\ntimeline of one replayed c2 step, after build:")
        print(child([sys.executable, os.path.join("scripts", "step_timeline.py")], ROOT), flush=True)


if __name__ == "__main__":
    main()
