"""CUDA-event microbenchmark of the weight-gradient launches of the `hier` train step against their floors.

usage: python tools/bench_wgrad.py [--baseline TREE] [--rounds N]

Cases: the grouped launch of one path-level transformer block (d_model 256, feed-forward 512: in_proj, out_proj, linear1 and
linear2 gradients in one dsvg_outer_group call) at the encoder and decoder row counts, and the args head gradient (M 126976,
P 2827 with ld 2832, Q 256, device-side alpha).  L2 is flushed by a 512 MB fill before every launch.

The floor of a case is the larger of its FLOPs at 989 TFLOP/s and its operand bytes (each operand read once) at 3.35 TB/s,
the H100 SXM data-sheet rates; "frac" is floor / measured time.  With --baseline TREE, TREE is another built checkout of this
project (the parent commit, say): its kernels are timed on the same cases in a subprocess, alternating with this tree's.
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
D, FF = 256, 512


def block(M):
    return [(D, FF), (FF, D), (D, D), (3 * D, D)]   # (P, Q) of linear2, linear1, out_proj, in_proj


CASES = [("block M=131072", "group", 131072, block(131072)),
         ("block M=126976", "group", 126976, block(126976)),
         ("args head M=126976", "head", 126976, [(2827, 256)])]


def floor_us(M, pq):
    flops = sum(2.0 * M * p * q for p, q in pq)
    nbytes = sum(2.0 * M * (p + q) for p, q in pq)
    return 1e6 * max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES)


def measure(tree, reps):
    sys.path.insert(0, tree)
    import torch
    from deepsvg_b200 import ops
    dev = torch.device("cuda:0")
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    out = {}
    for name, kind, M, pq in CASES:
        g = torch.Generator(device=dev).manual_seed(0)
        probs = []
        for p, q in pq:
            A = ops.Act(M, p, 1, dev, ld=(p + 7) // 8 * 8, zero=True)
            A.t[0, :, :p] = torch.randn(M, p, device=dev, generator=g).to(torch.bfloat16)
            B = ops.Act(M, q, 1, dev, zero=True)
            B.t[0] = torch.randn(M, q, device=dev, generator=g).to(torch.bfloat16)
            probs.append((A, B, p, q, torch.zeros(p, q, device=dev), torch.zeros(p, device=dev)))
        alpha = torch.full((1,), 0.5, device=dev)

        def launch():
            if kind == "group":
                ops.outer_group(probs, M)
            else:
                A, B, p, q, Cw, cs = probs[0]
                ops.outer(A, B, M, p, q, Cw, alpha_dev=alpha, colsum=cs)
        ts = []
        for it in range(reps + 2):
            flush.fill_(it)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts = sorted(ts[2:])
        out[name] = ts[len(ts) // 2]
        del probs
    return out


def run_tree(tree, reps):
    cmd = [sys.executable, os.path.abspath(__file__), "--tree", tree, "--reps", str(reps), "--json"]
    res = subprocess.run(cmd, check=True, stdout=subprocess.PIPE, text=True)
    return json.loads(res.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default="", help="another built checkout of this project to time alongside this one")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds per tree")
    ap.add_argument("--reps", type=int, default=10, help="timed launches per case and round (median)")
    ap.add_argument("--tree", default="", help=argparse.SUPPRESS)
    ap.add_argument("--json", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.json:
        print(json.dumps(measure(a.tree, a.reps)))
        return
    import torch
    print("device: %s" % torch.cuda.get_device_name(0), flush=True)
    trees = [("this", HERE)] + ([("baseline", os.path.abspath(a.baseline))] if a.baseline else [])
    runs = {t: [] for t, _ in trees}
    for _ in range(a.rounds):
        for t, path in trees:
            runs[t].append(run_tree(path, a.reps))
    summary = {}
    for name, _, M, pq in CASES:
        fl = floor_us(M, pq)
        row = {"floor_us": fl}
        for t, _ in trees:
            us = sorted(r[name] for r in runs[t])
            row[t] = {"us": us[len(us) // 2], "all_us": us, "frac": fl / us[len(us) // 2]}
        summary[name] = row
        line = "%-20s floor %6.1f us" % (name, fl)
        for t, _ in trees:
            line += "   %s %7.1f us (%.2f of floor)" % (t, row[t]["us"], row[t]["frac"])
        if a.baseline:
            line += "   speed-up %.2fx" % (row["baseline"]["us"] / row["this"]["us"])
        print(line, flush=True)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
