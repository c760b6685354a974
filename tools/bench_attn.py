"""CUDA-event microbenchmark of the 32 x 32 tensor-core attention (attn_mma_fwd_kernel / attn_mma_bwd_kernel) at the shapes
of the `hier` train step, against the HBM floor.

usage: python tools/bench_attn.py [--baseline TREE] [--rounds N] [--reps N]

Cases: the path-level launches (4096 sequences of L = 32, H = 8, head_dim 32) and the group-level ones (512 sequences of
L = 8), forward and backward, single-plane bf16, key mask from seeded lengths, dropout 0.1 as in training.  L2 is flushed
by a 512 MB fill before every launch; the median over --reps launches is reported.

The floor of a case is its bytes as ops.attn_fwd / ops.attn_bwd count them (q, k, v in and o out; q, k, v, dO in and dq,
dk, dv out) at 3.35 TB/s, the H100 SXM data-sheet rate; "frac" is floor / measured time.  With --baseline TREE, TREE is
another built checkout of this project (the parent commit, say): its kernels are timed on the same cases in a subprocess,
alternating with this tree's, and the SHA-256 of every output (o, dq, dk, dv) on the same seeded inputs and dropout seed
tells whether the two builds compute bit-identical results.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_BYTES = 3.35e12
HD, DROP = 32, 0.1

# (name, nseq, L, H)
CASES = [("path L=32", 4096, 32, 8), ("group L=8", 512, 8, 8)]


def nbytes(nseq, L, H, bwd):
    return 2.0 * nseq * L * H * HD * (7 if bwd else 4)


def floor_us(nseq, L, H, bwd):
    return 1e6 * nbytes(nseq, L, H, bwd) / PEAK_BYTES


def _digest(t):
    import torch
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def measure(tree, reps):
    sys.path.insert(0, tree)
    import torch
    from deepsvg_b200 import ops
    dev = torch.device("cuda:0")
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    out = {}
    for name, nseq, L, H in CASES:
        d, M = H * HD, nseq * L
        g = torch.Generator(device=dev).manual_seed(0)
        qkv = ops.Act(M, 3 * d, 1, dev)
        qkv.t[0] = (torch.randn(M, 3 * d, device=dev, generator=g) * 0.7).to(torch.bfloat16)
        dout = ops.Act(M, d, 1, dev)
        dout.t[0] = torch.randn(M, d, device=dev, generator=g).to(torch.bfloat16)
        lens = torch.randint(1, L + 1, (nseq,), device=dev, generator=g)
        valid = (torch.arange(L, device=dev)[None, :] < lens[:, None]).to(torch.uint8).reshape(-1).contiguous()
        o = ops.Act(M, d, 1, dev, zero=True)
        dqkv = ops.Act(M, 3 * d, 1, dev, zero=True)
        drop = (DROP, 7, 1234)
        launches = {"fwd": lambda: ops.attn_fwd(qkv, valid, o, nseq, L, H, HD, drop),
                    "bwd": lambda: ops.attn_bwd(qkv, valid, dout, dqkv, nseq, L, H, HD, HD ** -0.5, drop)}
        for kind, launch in launches.items():
            ts = []
            for it in range(reps + 3):
                flush.fill_(it)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                launch()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            ts = sorted(ts[3:])
            out["%s %s" % (name, kind)] = ts[len(ts) // 2]
        out["%s digest" % name] = {"o": _digest(o.t), "dq": _digest(dqkv.t[0, :, :d]),
                                   "dk": _digest(dqkv.t[0, :, d:2 * d]), "dv": _digest(dqkv.t[0, :, 2 * d:])}
        del qkv, dout, o, dqkv
    return out


def run_tree(tree, reps):
    cmd = [sys.executable, os.path.abspath(__file__), "--tree", tree, "--reps", str(reps), "--json"]
    res = subprocess.run(cmd, check=True, stdout=subprocess.PIPE, text=True)
    return json.loads(res.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default="", help="another built checkout of this project to time alongside this one")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds per tree")
    ap.add_argument("--reps", type=int, default=50, help="timed launches per case and round (median)")
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
    for name, nseq, L, H in CASES:
        for kind in ("fwd", "bwd"):
            key = "%s %s" % (name, kind)
            fl = floor_us(nseq, L, H, kind == "bwd")
            row = {"floor_us": fl, "bytes": nbytes(nseq, L, H, kind == "bwd")}
            for t, _ in trees:
                us = sorted(r[key] for r in runs[t])
                med = us[len(us) // 2]
                row[t] = {"us": med, "all_us": us, "frac": fl / med, "gbs": row["bytes"] / med / 1e3}
            summary[key] = row
            line = "%-16s floor %6.1f us" % (key, fl)
            for t, _ in trees:
                line += "   %s %7.1f us (%.2f of floor)" % (t, row[t]["us"], row[t]["frac"])
            if a.baseline:
                line += "   speed-up %.2fx" % (row["baseline"]["us"] / row["this"]["us"])
            print(line, flush=True)
        dkey = "%s digest" % name
        digests = [r[dkey] for t, _ in trees for r in runs[t]]
        same = all(dg == digests[0] for dg in digests)
        summary[dkey] = {"bit_identical": same, "this": runs["this"][0][dkey]}
        print("%-16s outputs (o, dq, dk, dv) %s across %s" % (name, "bit-identical" if same else "DIFFER",
                                                             "runs and trees" if a.baseline else "runs"), flush=True)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
