"""Development tool: launch one hot linear shape / epilogue mode a few times (to time it under torch.profiler)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deepsvg_b200 import ops

dev = torch.device("cuda:0")
which = sys.argv[1]
M = 131072
PL = int(os.environ.get("DSVG_PLANES", "1"))     # 2: parity-mode (bf16x3) operands for the linear roles


def go(M, N, K, **kw):
    X = ops.Act(M, K, PL, dev, zero=True)
    X.t.normal_()
    W = ops.Act(N, K, PL, dev, zero=True)
    W.t.normal_(std=K ** -0.5)
    if PL == 2:
        X.t[1] *= 2.0 ** -9
        W.t[1] *= 2.0 ** -9
    for _ in range(4):
        ops.linear(X, W, M, N, K, **kw)
    torch.cuda.synchronize()


if which == "ffn1":
    go(M, 512, 256, bias=torch.zeros(512, device=dev), relu=True, drop=(0.1, 3, 7), out_act=ops.Act(M, 512, PL, dev))
elif which == "qkv":
    go(M, 768, 256, bias=torch.zeros(768, device=dev), scale_cols=256, scale=0.17, out_act=ops.Act(M, 768, PL, dev))
elif which == "proj":
    x = torch.zeros(M, 256, device=dev)
    go(M, 256, 256, bias=torch.zeros(256, device=dev), drop=(0.1, 4, 7), residual=x, out_f32=x)
elif which == "ffn2":
    x = torch.zeros(M, 256, device=dev)
    go(M, 256, 512, bias=torch.zeros(256, device=dev), drop=(0.1, 4, 7), residual=x, out_f32=x)
elif which == "mask":
    mk = ops.Act(M, 512, 1, dev, zero=True)
    mk.t.normal_()
    go(M, 512, 256, mask=mk, mask_scale=1.1, out_act=ops.Act(M, 512, 1, dev))
elif which == "dgrad":
    go(M, 256, 512, out_act=ops.Act(M, 256, 1, dev))
elif which == "lnfwd":        # mode 8: out-proj / FFN2 with the following LayerNorm in the epilogue
    x = torch.zeros(M, 256, device=dev)
    g = torch.ones(256, device=dev)
    go(M, 256, 512, bias=torch.zeros(256, device=dev), drop=(0.1, 4, 7), residual=x, out_f32=torch.empty(M, 256, device=dev),
       ln=(g, g, ops.Act(M, 256, 1, dev), torch.empty(M, device=dev), torch.empty(M, device=dev)))
elif which == "logits":       # mode 7: the 2827-wide fp32 args head
    Ml = 126976
    go(Ml, 2827, 256, bias=torch.zeros(2827, device=dev), out_f32=torch.empty(Ml, 2827, device=dev))
elif which == "head_dgrad":   # mode 6: dgrad of the args head, accumulated in fp32
    Ml = 126976
    acc = torch.zeros(Ml, 256, device=dev)
    X = ops.Act(Ml, 2827, 1, dev, ld=2832, zero=True)
    X.t.normal_()
    W = ops.Act(256, 2827, 1, dev, ld=2832, zero=True)
    W.t.normal_(std=0.02)
    sc = torch.ones(1, device=dev)
    for _ in range(4):
        ops.linear(X, W, Ml, 256, 2827, acc_scale=sc, residual=acc, out_f32=acc)
    torch.cuda.synchronize()
elif which == "outer":
    A = ops.Act(M, 768, 1, dev, zero=True)
    A.t.normal_()
    B = ops.Act(M, 256, 1, dev, zero=True)
    B.t.normal_()
    Cw = torch.zeros(768, 256, device=dev)
    cs = torch.zeros(768, device=dev)
    for _ in range(4):
        ops.outer(A, B, M, 768, 256, Cw, colsum=cs)
    torch.cuda.synchronize()
elif which == "attn":
    nseq, L, H, hd = 4096, 32, 8, 32
    qkv = ops.Act(M, 768, PL, dev, zero=True)
    qkv.t.normal_(std=0.5)
    o, do, dq = ops.Act(M, 256, PL, dev), ops.Act(M, 256, PL, dev, zero=True), ops.Act(M, 768, PL, dev)
    for _ in range(3):
        ops.attn_fwd(qkv, None, o, nseq, L, H, hd, (0.1, 2, 9))
        ops.attn_bwd(qkv, None, do, dq, nseq, L, H, hd, 0.17, (0.1, 2, 9))
    torch.cuda.synchronize()
elif which == "gattn":        # general tensor-core attention at the scaled config's path-level shape
    nseq, L, H, hd = 2048, 66, 8, 64
    Mg = nseq * L
    qkv = ops.Act(Mg, 1536, PL, dev, zero=True)
    qkv.t.normal_(std=0.5)
    o, do, dq = ops.Act(Mg, 512, PL, dev), ops.Act(Mg, 512, PL, dev, zero=True), ops.Act(Mg, 1536, PL, dev)
    for _ in range(3):
        ops.attn_fwd(qkv, None, o, nseq, L, H, hd, (0.1, 2, 9))
        ops.attn_bwd(qkv, None, do, dq, nseq, L, H, hd, 0.125, (0.1, 2, 9))
    torch.cuda.synchronize()
elif which == "ln_bwd":
    x, dxin = torch.randn(M, 256, device=dev), torch.randn(M, 256, device=dev)
    g = torch.ones(256, device=dev)
    mean, rstd = torch.zeros(M, device=dev), torch.ones(M, device=dev)
    dy = ops.Act(M, 256, 1, dev, zero=True)
    dg, db = torch.zeros(256, device=dev), torch.zeros(256, device=dev)
    for _ in range(3):
        ops.ln_bwd(x, mean, rstd, g, M, 256, dy=dy, dx_in=dxin, dx_out=torch.empty(M, 256, device=dev),
                   dact=ops.Act(M, 256, 1, dev), drop=(0.1, 3, 5), dgamma=dg, dbeta=db)
    torch.cuda.synchronize()
elif which == "small_outer":
    Ms = 4096
    A = ops.Act(Ms, 768, 1, dev, zero=True)
    A.t.normal_()
    B = ops.Act(Ms, 256, 1, dev, zero=True)
    B.t.normal_()
    Cw = torch.zeros(768, 256, device=dev)
    cs = torch.zeros(768, device=dev)
    for _ in range(4):
        ops.outer(A, B, Ms, 768, 256, Cw, colsum=cs)
    torch.cuda.synchronize()
elif which == "small_generic":
    g2 = torch.zeros(512, 256, device=dev)
    go(512, 256, 256, bias=torch.zeros(256, device=dev), drop=(0.1, 4, 7), rowvec=g2, rows_per_group=1,
       out_f32=torch.zeros(512, 256, device=dev))
elif which == "small_lean":
    x = torch.zeros(4096, 256, device=dev)
    go(4096, 256, 256, bias=torch.zeros(256, device=dev), drop=(0.1, 4, 7), residual=x, out_f32=x)
