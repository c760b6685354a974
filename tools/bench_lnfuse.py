"""Development microbenchmark: the fused GEMM+LayerNorm forward kernel against its two-kernel equivalent at the path-level
shape (M = 131072 rows, d_model = 256), CUDA-event timed.  `python tools/bench_lnfuse.py`"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deepsvg_b200 import ops

dev = torch.device("cuda:0")
M, N = 131072, 256


def act(r, c, std=1.0):
    a = ops.Act(r, c, 1, dev, zero=True)
    a.t.normal_(std=std)
    return a


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


g, b = torch.ones(N, device=dev), torch.zeros(N, device=dev)
mean, rstd = torch.zeros(M, device=dev), torch.ones(M, device=dev)
res = torch.randn(M, N, device=dev)
bias = torch.zeros(N, device=dev)
# two output buffers per tensor so that consecutive launches do not hit a warm L2 copy of the previous output
x1 = [torch.empty(M, N, device=dev) for _ in range(2)]
y = [ops.Act(M, N, 1, dev) for _ in range(2)]

for K in (256, 512):
    X, W = act(M, K), act(N, K, K ** -0.5)
    i = [0]

    def fused():
        j = i[0] = i[0] ^ 1
        ops.linear(X, W, M, N, K, bias=bias, drop=(0.1, 4, 7), residual=res, out_f32=x1[j], ln=(g, b, y[j], mean, rstd))

    def split():
        j = i[0] = i[0] ^ 1
        ops.linear(X, W, M, N, K, bias=bias, drop=(0.1, 4, 7), residual=res, out_f32=x1[j])
        ops.ln_fwd(x1[j], g, b, y[j], mean, rstd, M, N)

    print("fwd  K=%d  fused %.1f us   linear+ln_fwd %.1f us" % (K, timeit(fused), timeit(split)), flush=True)
