#!/usr/bin/env python
"""Before / after of the 32-channel down and up convolutions (dv_conv_down / dv_conv_up at CH = 32), in one run on one GPU.

    python scripts/conv_epilogue_rate.py --before DIR [--reps 3] [--skip-identity] [--skip-bench] [--skip-timeline]

DIR is a second, already built copy of this repository inside the working tree (for example the parent commit exported
with `git archive` into a git-ignored directory and built there with `python disentangling-vae_b200/build.py`); "after"
is the tree this script lies in.  Absolute times move by several percent between sessions, so only the comparisons
inside one run count.  Steps:

1. the card's name, power limit and maximum SM clock (read-only nvidia-smi query);
2. bit-identity: per build, in a child process, ops.conv_down and ops.conv_up on the same seeded inputs at lo 16, 8 and
   4 and B = 1024, 512, 256, 37, without a mask, with the float mask alone and with the float mask and its mask words,
   with bias + ReLU and without either (every output: lo / hi, the [x > 0] words, the channel sums of down); then bench.py --dump-outputs
   for c2 and c5.  Every array must be bitwise equal between the builds;
3. per build, in child processes, alternating before / after --reps times: CUDA events around 50 back-to-back calls
   after 5 warm-up calls, 5 repeats, for the four 32 -> 32 calls of a training step (down forward, down with mask
   words + channel sums = decoder dgrad, up forward, up with mask words = encoder dgrad) at B = 1024, lo 16 and 8;
   min-max in us per call;
4. per build, alternating --reps times: bench.py --steps 200 --warmup 20 at c2, then once each at c1, c3 and c5:
   ms_per_step and parity.ok;
5. per build: scripts/step_timeline.py on one replayed c2 step, summed time of the down and up kernels and step span.

One JSON line with everything, then Markdown tables.  Exits non-zero without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS, WARMUP, REPEATS = 50, 5, 5
TIMED = [(1024, 16), (1024, 8)]
IDENT_B = [1024, 512, 256, 37]
IDENT_H = [16, 8, 4]
KERNELS = {"conv_down32_mma_kernel": "down", "conv_up_halo_mma_kernel": "up"}


def _import(root):
    sys.path[:0] = [root, os.path.join(root, "disentangling-vae_b200")]
    import torch
    from disvae import ops
    return torch, ops


def _inputs(torch, B, H, seed):
    """Seeded on the host, so both builds see the same bits."""
    g = torch.Generator().manual_seed(seed)
    dev = torch.device("cuda", 0)
    hi = torch.randn(B, 2 * H, 2 * H, 32, generator=g).to(dev)
    lo = torch.randn(B, H, H, 32, generator=g).to(dev)
    w = (torch.randn(32, 32, 4, 4, generator=g) * 0.1).to(dev)
    bias = (torch.randn(32, generator=g) * 0.1).to(dev)
    bits_lo = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, H, H), generator=g, dtype=torch.int32).to(dev)
    bits_hi = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, 2 * H, 2 * H), generator=g, dtype=torch.int32).to(dev)
    mask_lo = torch.randn(B, H, H, 32, generator=g).to(dev)
    mask_hi = torch.randn(B, 2 * H, 2 * H, 32, generator=g).to(dev)
    return hi, lo, w, bias, bits_lo, bits_hi, mask_lo, mask_hi


def identity_outputs(root, out_path):
    """Child: every output of the seeded conv calls of the build at `root`, saved to out_path."""
    torch, ops = _import(root)
    out = {}
    for H in IDENT_H:
        for B in IDENT_B:
            hi, lo, w, bias, bits_lo, bits_hi, mask_lo, mask_hi = _inputs(torch, B, H, 1000 * H + B)
            wp = ops.conv_pack(w, 32)
            for relu in (0, 1):
                act, b = (ops.N.ACT_RELU, bias) if relu else (ops.N.ACT_NONE, None)
                for use_mask, use_bits in ((0, 0), (1, 0), (1, 1)):    # the words come with the float mask only
                    key = "H%d_B%d_relu%d_bits%d_mask%d" % (H, B, relu, use_bits, use_mask)
                    d = ops.conv_down(hi, wp, b, mask_lo if use_mask else None, B, H, H, 32, 0, act, want_colsum=True,
                                      mask_bits=bits_lo if use_bits else None, want_bits=True)
                    u = ops.conv_up(lo, wp, b, mask_hi if use_mask else None, B, H, H, 32, 0, act,
                                    mask_bits=bits_hi if use_bits else None, want_bits=True)
                    for name, t in zip(("down_lo", "down_colsum", "down_bits", "up_hi", "up_bits"), d + u):
                        out[key + "." + name] = t.cpu()
    torch.cuda.synchronize()
    torch.save(out, out_path)


def time_kernels(root):
    """Child: us per call of the four 32 -> 32 calls of a training step, REPEATS times per shape."""
    torch, ops = _import(root)
    out = {}
    for B, H in TIMED:
        hi, lo, w, bias, bits_lo, bits_hi, mask_lo, mask_hi = _inputs(torch, B, H, 7)
        wp = ops.conv_pack(w, 32)
        R, NONE = ops.N.ACT_RELU, ops.N.ACT_NONE
        calls = {   # as disvae/ops.py issues them in a training step
            "down": lambda: ops.conv_down(hi, wp, bias, None, B, H, H, 32, 0, R, want_bits=True),
            "down+mask": lambda: ops.conv_down(hi, wp, None, mask_lo, B, H, H, 32, 0, NONE, want_colsum=True,
                                               mask_bits=bits_lo),
            "up": lambda: ops.conv_up(lo, wp, bias, None, B, H, H, 32, 0, R, want_bits=True),
            "up+mask": lambda: ops.conv_up(lo, wp, None, mask_hi, B, H, H, 32, 0, NONE, mask_bits=bits_hi),
        }
        for name, fn in calls.items():
            for _ in range(WARMUP):
                fn()
            us = []
            for _ in range(REPEATS):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(CALLS):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                us.append(e0.elapsed_time(e1) / CALLS * 1e3)
            out["%s lo%d" % (name, H)] = us
    print(json.dumps(out), flush=True)


def child(cmd, cwd, env=None):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=1800, env=env)
    if r.returncode != 0:
        sys.exit("%s failed in %s:\n%s%s" % (" ".join(cmd), cwd, r.stdout[-2000:], r.stderr[-4000:]))
    return r.stdout


def last_json(text):
    return json.loads([ln for ln in text.splitlines() if ln.startswith("{")][-1])


def bench(root, workload, extra=(), steps=200, warmup=20):
    out = last_json(child([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
                           "--workload", workload, "--no-cpu-baseline", "--no-eager-baseline"] + list(extra), root))
    return {"ms_per_step": out["ms_per_step"], "parity_ok": out["parity"]["ok"]}


def check_identity(builds, tmp):
    import numpy as np
    import torch
    got = {}
    for name, root in builds:
        path = os.path.join(tmp, name + ".pt")
        child([sys.executable, os.path.abspath(__file__), "--identity", root, path], root)
        got[name] = torch.load(path)
    b, a = got["before"], got["after"]
    bad = sorted(k for k in b if k not in a or b[k].shape != a[k].shape or not torch.equal(b[k].view(torch.int32) if
              b[k].dtype == torch.float32 else b[k], a[k].view(torch.int32) if a[k].dtype == torch.float32 else a[k]))
    res = {"conv_arrays": len(b), "conv_differ": bad}
    for w in ("c2", "c5"):
        dirs = {}
        for name, root in builds:
            dirs[name] = os.path.join(tmp, "%s_%s" % (name, w))
            bench(root, w, ["--dump-outputs", dirs[name]], steps=3, warmup=1)
        files = sorted(os.listdir(dirs["before"]))
        differ = [f for f in files if not os.path.exists(os.path.join(dirs["after"], f)) or
                  np.load(os.path.join(dirs["before"], f)).tobytes() != np.load(os.path.join(dirs["after"], f)).tobytes()]
        res["bench_" + w] = {"arrays": len(files), "differ": differ}
    return res


def timeline(root):
    """Step span and summed down / up kernel time of one replayed c2 step."""
    text = child([sys.executable, os.path.join("scripts", "step_timeline.py")], root)
    tot = {v: 0.0 for v in KERNELS.values()}
    span = None
    for ln in text.splitlines():
        for k, v in KERNELS.items():
            if k in ln[:58]:
                tot[v] += float(ln.split()[-2])
        if ln.startswith("step span"):
            span = float(ln.split()[2])
    return {"span_us": span, "down_us": round(tot["down"], 1), "up_us": round(tot["up"], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--before", help="root of the built copy to compare against")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-identity", action="store_true")
    ap.add_argument("--skip-bench", action="store_true")
    ap.add_argument("--skip-timeline", action="store_true")
    ap.add_argument("--time-kernels", metavar="ROOT", help=argparse.SUPPRESS)
    ap.add_argument("--identity", nargs=2, metavar=("ROOT", "OUT"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("conv_epilogue_rate.py needs a GPU")
    if args.time_kernels:
        return time_kernels(args.time_kernels)
    if args.identity:
        return identity_outputs(*args.identity)
    if not args.before:
        ap.error("--before is required")
    builds = [("before", os.path.abspath(args.before)), ("after", ROOT)]
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    res = {"card": q, "calls": CALLS, "repeats": REPEATS, "reps": args.reps}
    print("card (name, power limit, max SM clock):", q, flush=True)
    ok = True

    if not args.skip_identity:
        with tempfile.TemporaryDirectory() as tmp:
            res["identity"] = ident = check_identity(builds, tmp)
        ok = not ident["conv_differ"] and not ident["bench_c2"]["differ"] and not ident["bench_c5"]["differ"]
        print("\nbit-identity: %d conv arrays, %d differ; bench c2 %d arrays, %d differ; bench c5 %d arrays, %d differ"
              % (ident["conv_arrays"], len(ident["conv_differ"]), ident["bench_c2"]["arrays"],
                 len(ident["bench_c2"]["differ"]), ident["bench_c5"]["arrays"], len(ident["bench_c5"]["differ"])), flush=True)
        for k in ident["conv_differ"][:20]:
            print("  differs:", k)

    kernel = {name: {} for name, _ in builds}
    for _ in range(args.reps):
        for name, root in builds:
            got = last_json(child([sys.executable, os.path.abspath(__file__), "--time-kernels", root], root))
            for k, us in got.items():
                kernel[name].setdefault(k, []).extend(us)
    res["kernel_us"] = kernel
    print("\n| call | before us / call (min-max) | after us / call (min-max) | after / before (min) |")
    print("|---|---|---|---|")
    for k in kernel["before"]:
        b, a = kernel["before"][k], kernel["after"][k]
        print("| %s | %.1f-%.1f | %.1f-%.1f | %.3f |" % (k, min(b), max(b), min(a), max(a), min(a) / min(b)), flush=True)

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

    if not args.skip_timeline:
        res["timeline"] = {name: timeline(root) for name, root in builds}
        print("\n| one replayed c2 step | before | after |")
        print("|---|---|---|")
        for k in ("down_us", "up_us", "span_us"):
            print("| %s | %s | %s |" % (k, res["timeline"]["before"][k], res["timeline"]["after"][k]), flush=True)
    print("\n" + json.dumps(res), flush=True)
    if not ok:
        sys.exit("outputs differ between the builds")


if __name__ == "__main__":
    main()
