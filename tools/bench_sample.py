"""Times autoregressive sampling (`SVGTransformer.greedy_sample` of a Sketchformer in eval mode): the cached engine
(csrc/decode.cu, one decoder row per sequence per step, the step replayed as a CUDA graph) against the teacher-forced loop
it replaces, written out below: every step runs `model.forward` on the whole prefix and keeps the last position.

Configuration: Sketchformer, d_model 256, 8 heads, 4 + 4 layers, random weights, random latents; max_total_len 50 and 139;
N = 1, 64 and 512 sequences; both precisions.  Per point the two are alternated, three timed runs each after one warm-up
run, host clock ending in a synchronise (median reported).  Also reported: the fraction of decoded positions on which the
two agree (command and all 11 arguments), and, from a separate torch.profiler run of the engine without graphs,
decode_attn_kernel's algorithmic bytes (the valid cached K and V rows it must read) over its kernel time, against the
H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Prints a table to stderr and one JSON line with the card's name and
power limit to stdout.

    python tools/bench_sample.py [--T 50,139] [--N 1,64,512] [--precision bf16,bf16x3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from deepsvg_b200 import Sketchformer, SVGTransformer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def forward_loop(model, z):
    """The pre-cache decoding: T forward passes over the growing prefix, argmax of the last position, _make_valid."""
    N, T = z.shape[0], model.cfg.max_total_len
    cy = torch.full((N, 1, 1), 5, dtype=torch.long, device=z.device)
    ay = torch.full((N, 1, 1, 11), -1, dtype=torch.long, device=z.device)
    with torch.no_grad():
        for _ in range(T):
            res = model(None, None, cy.float(), ay.float(), z=z, return_tgt=False)
            cn, an = res["command_logits"][..., -1:, :].argmax(-1), res["args_logits"][..., -1:, :, :].argmax(-1) - 1
            _, an = model._make_valid(cn, an)
            cy, ay = torch.cat([cy, cn], -1), torch.cat([ay, an], -2)
    return cy[:, 0, 1:], ay[:, 0, 1:]


def engine(model, z):
    model.greedy_sample(z=z, concat_groups=False)
    return model._ds.out_cmd, model._ds.out_args          # the decoded classes, before _make_absolute


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def attn_bandwidth(model, z):
    """decode_attn_kernel over one eager engine run: (algorithmic bytes, kernel seconds)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    cfg = model.cfg
    graphs, model.graphs = model.graphs, False
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine(model, z)
        torch.cuda.synchronize()
    model.graphs = graphs
    us = [e.time_range.elapsed_us() for e in prof.events()
          if e.device_type == DeviceType.CUDA and "decode_attn_kernel" in e.name]
    assert len(us) == cfg.max_total_len * cfg.n_layers_decode, len(us)
    kv = model._ds.key_valid.long()                                 # [N, T]: keys the kernel reads at each step
    keys = kv.cumsum(1).sum(0).double()                             # valid keys <= t, summed over sequences
    row = 2 * cfg.d_model * 2 * model.planes                        # K and V, bf16, per plane
    nbytes = float(keys.sum()) * row * cfg.n_layers_decode
    return nbytes, sum(us) * 1e-6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", default="50,139")
    ap.add_argument("--N", default="1,64,512")
    ap.add_argument("--precision", default="bf16,bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sample: needs a CUDA GPU")
    dev = torch.device("cuda:0")
    name, pl = card()
    sys.stderr.write("card: %s, power limit %s\n" % (name, pl))
    sys.stderr.write("%6s %4s %4s %11s %11s %8s %7s %9s %6s\n" % ("prec", "T", "N", "loop ms", "cached ms", "speedup",
                                                                   "agree", "attn GB/s", "HBM%"))
    points = []
    for T in map(int, a.T.split(",")):
        for prec in a.precision.split(","):
            torch.manual_seed(0)
            cfg = Sketchformer(d_model=256, n_heads=8, n_layers=4, n_layers_decode=4, max_total_len=T)
            model = SVGTransformer(cfg, precision=prec).to(dev).eval()
            for N in map(int, a.N.split(",")):
                z = torch.randn(N, 1, 1, cfg.dim_z, device=dev)
                timed(lambda: forward_loop(model, z))
                timed(lambda: engine(model, z))
                t_loop, t_eng = [], []
                for _ in range(3):
                    t, (lc, la) = timed(lambda: forward_loop(model, z))
                    t_loop.append(t)
                    t, (ec, ea) = timed(lambda: engine(model, z))
                    t_eng.append(t)
                agree = ((lc == ec) & (la == ea).all(-1)).float().mean().item()
                nbytes, secs = attn_bandwidth(model, z)
                ml, me = sorted(t_loop)[1] * 1e3, sorted(t_eng)[1] * 1e3
                bw = nbytes / secs
                points.append(dict(precision=prec, T=T, N=N, loop_ms=ml, cached_ms=me, speedup=ml / me, agreement=agree,
                                   attn_bytes=nbytes, attn_s=secs, attn_gb_s=bw * 1e-9, attn_hbm_frac=bw / HBM_BYTES_PER_S,
                                   loop_runs_ms=[t * 1e3 for t in t_loop], cached_runs_ms=[t * 1e3 for t in t_eng]))
                sys.stderr.write("%6s %4d %4d %11.1f %11.2f %7.1fx %7.4f %9.0f %5.1f%%\n" % (
                    prec, T, N, ml, me, ml / me, agree, bw * 1e-9, 100 * bw / HBM_BYTES_PER_S))
            del model
            torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit=pl, points=points)))


if __name__ == "__main__":
    main()
