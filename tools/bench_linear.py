"""Microbenchmark of the path-level GEMM roles of the `hier` workload (M = 131072 rows, d_model = 256, ff = 512),
CUDA-event timed over many launches, plus the fused GEMM + LayerNorm forward against its two-kernel equivalent.

For each role it prints the time per launch, the algorithmic bytes over that time (and as a fraction of the H100 SXM
data-sheet HBM3 bandwidth, 3.35 TB/s) and the achieved TFLOP/s, with the card's name and power limit.  Outputs alternate
between two buffers so that no launch reads a warm L2 copy of the previous launch's output.

    python tools/bench_linear.py [--iters 100] [--json FILE]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from deepsvg_b200 import ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
M, D, FF = 131072, 256, 512


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timeit(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3   # us per launch


def roles(dev):
    """(name, N, K, bytes, launch(k)) for every path-level GEMM role; launch(k) writes output buffer k (0 / 1)."""
    def act(r, c, std=1.0):
        a = ops.Act(r, c, 1, dev, zero=True)
        a.t.normal_(std=std)
        return a

    def w(n, k):
        return act(n, k, k ** -0.5)

    def bias(n):
        return torch.randn(n, device=dev) * 0.1

    x_d, x_ff, x_3d = act(M, D), act(M, FF), act(M, 3 * D)
    mask = act(M, FF)
    res = torch.randn(M, D, device=dev)
    g, b = torch.ones(D, device=dev), torch.zeros(D, device=dev)
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    out_a = {n: [ops.Act(M, n, 1, dev) for _ in range(2)] for n in (D, FF, 3 * D)}
    out_f = [torch.empty(M, D, device=dev) for _ in range(2)]
    y = [ops.Act(M, D, 1, dev) for _ in range(2)]
    wq, wo, w1, w2 = w(3 * D, D), w(D, D), w(FF, D), w(D, FF)
    w2t, w1t, wot, wqt = w(FF, D), w(D, FF), w(D, D), w(D, 3 * D)
    bq, bo, b1, b2 = bias(3 * D), bias(D), bias(FF), bias(D)
    drop = (0.1, 4, 7)
    act_b, f32_b = 2, 4
    ln_b = M * (f32_b * D + act_b * D + 2 * 4)      # x1 out, LayerNorm out, mean and rstd
    return [
        ("qkv", 3 * D, D, M * (D + 3 * D) * act_b,
         lambda k: ops.linear(x_d, wq, M, 3 * D, D, bias=bq, scale_cols=D, scale=0.125, out_act=out_a[3 * D][k])),
        ("out_proj+res+ln", D, D, M * (D * act_b + D * f32_b) + ln_b,
         lambda k: ops.linear(x_d, wo, M, D, D, bias=bo, drop=drop, residual=res, out_f32=out_f[k],
                              ln=(g, b, y[k], mean, rstd))),
        ("ffn1+relu+drop", FF, D, M * (D + FF) * act_b,
         lambda k: ops.linear(x_d, w1, M, FF, D, bias=b1, relu=True, drop=drop, out_act=out_a[FF][k])),
        ("ffn2+res+ln", D, FF, M * (FF * act_b + D * f32_b) + ln_b,
         lambda k: ops.linear(x_ff, w2, M, D, FF, bias=b2, drop=drop, residual=res, out_f32=out_f[k],
                              ln=(g, b, y[k], mean, rstd))),
        ("ffn2_dgrad_mask", FF, D, M * (D + 2 * FF) * act_b,
         lambda k: ops.linear(x_d, w2t, M, FF, D, mask=mask, mask_scale=1.0 / 0.9, out_act=out_a[FF][k])),
        ("ffn1_dgrad", D, FF, M * (FF + D) * act_b,
         lambda k: ops.linear(x_ff, w1t, M, D, FF, out_act=out_a[D][k])),
        ("out_proj_dgrad", D, D, M * (D + D) * act_b,
         lambda k: ops.linear(x_d, wot, M, D, D, out_act=out_a[D][k])),
        ("qkv_dgrad", D, 3 * D, M * (3 * D + D) * act_b,
         lambda k: ops.linear(x_3d, wqt, M, D, 3 * D, out_act=out_a[D][k])),
        # the fused LayerNorm against the same GEMM into the residual stream followed by the LayerNorm kernel
        ("out_proj+res (mode 4)", D, D, M * (D * act_b + 2 * D * f32_b),
         lambda k: ops.linear(x_d, wo, M, D, D, bias=bo, drop=drop, residual=res, out_f32=out_f[k])),
        ("out_proj+res, ln_fwd", D, D, M * (D * act_b + 2 * D * f32_b) + ln_b,
         lambda k: (ops.linear(x_d, wo, M, D, D, bias=bo, drop=drop, residual=res, out_f32=out_f[k]),
                    ops.ln_fwd(out_f[k], g, b, y[k], mean, rstd, M, D))),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_linear: needs a CUDA GPU")
    dev = torch.device("cuda:0")
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl))
    print("%-24s %6s %6s %9s %9s %7s %8s" % ("role (M = 131072)", "N", "K", "us", "GB/s", "HBM%", "TFLOP/s"))
    rows = []
    for role, N, K, nbytes, fn in roles(dev):
        k = [0]

        def step():
            fn(k[0])
            k[0] ^= 1

        us = timeit(step, a.iters)
        gbs = nbytes / us * 1e-3
        tf = 2.0 * M * N * K / us * 1e-6
        print("%-24s %6d %6d %9.1f %9.0f %6.1f%% %8.1f" % (role, N, K, us, gbs, 100 * gbs * 1e9 / HBM_BYTES_PER_S, tf),
              flush=True)
        rows.append(dict(role=role, N=N, K=K, us=us, bytes=nbytes, gb_s=gbs, hbm_frac=gbs * 1e9 / HBM_BYTES_PER_S,
                         tflops=tf))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=name, power_limit=pl, M=M, roles=rows), f, indent=1)


if __name__ == "__main__":
    main()
