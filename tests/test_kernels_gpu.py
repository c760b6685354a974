"""Per-kernel parity on the GPU: every C-ABI entry point against a plain fp32 / fp64 PyTorch restatement of the same op
(teacher-forced: identical inputs, so only accumulation order / operand rounding differ).

Every `*_CASES` table below is a list of pytest.param whose last value names the kernel(s) the case must launch, as
`family<template arguments>` (e.g. "linear_kernel<256, 1, 0>"); the test asserts them with `expect_kernels`, and
tests/test_kernel_coverage.py checks that together the tables name every compiled instantiation."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

# the longest sequence config.check_supported accepts per head_dim: the SIMT attention backward keeps Q, K, V, dO and two
# L x L fp32 tiles of one (sequence, head) pair in at most 227 KB of shared memory
ATTN_MAX_L = {16: 155, 32: 141, 64: 117}


def kernel_key(name):
    """'void dsvg::linear_kernel<256, 1, 0>(CUtensorMap_st, ...)' -> 'linear_kernel<256, 1, 0>'; None outside dsvg::."""
    m = re.match(r"(?:void )?dsvg::(\w+(?:<[^>]*>)?)", name)
    return m.group(1).replace("(bool)1", "true").replace("(bool)0", "false") if m else None


def kernel_family(key):
    """Variants of one family compete for the same call: every attention kernel is one family."""
    base = key.split("<")[0]
    return "attn" if base.startswith("attn_") else base


def launched_kernels(fn):
    """Runs fn() under torch.profiler (CUDA activity only) and returns the demangled names of the kernels it launched."""
    import time
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # a capture window barely longer than the call sometimes came back without its kernels: keep a margin around it
        time.sleep(0.005)
        fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    assert names, "torch.profiler recorded no CUDA kernels"
    return names


def expect_kernels(expect, fn):
    """fn() must launch the kernel(s) `expect` names and no other variant of their families."""
    expect = {expect} if isinstance(expect, str) else set(expect)
    got = {k for k in map(kernel_key, launched_kernels(fn)) if k is not None}
    fams = {kernel_family(k) for k in expect}
    assert {k for k in got if kernel_family(k) in fams} == expect, (sorted(expect), sorted(got))


def _ops():
    from deepsvg_b200 import ops
    return ops


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _rel(a, b):
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def _lin(bn, planes, mode):
    return "linear_kernel<%d, %d, %d>" % (bn, planes, mode)


def _attn(kind, hd=None, nt=None):
    """(forward, backward) kernels of one attention family: "simt" <hd>, "mma" / "x3" (32 x 32), "gmma" / "gx3" <hd, nt>."""
    if kind == "simt":
        return ("attn_fwd_kernel<%d>" % hd, "attn_bwd_kernel<%d>" % hd)
    if kind in ("mma", "x3"):
        return ("attn_%s_fwd_kernel" % kind, "attn_%s_bwd_kernel" % kind)
    fwd = "attn_gmma_fwd_kernel<%d, %d, true>" if kind == "gmma" else "attn_gx3_fwd_kernel<%d, %d>"
    return (fwd % (hd, nt), "attn_%s_bwd_kernel<%d, %d>" % (kind, hd, nt))


# ------------------------------------------------------------------------------------------------ GEMMs
def _linear_case(M, N, K, planes, kernel):
    return pytest.param(M, N, K, planes, kernel, id="%d-%d-%d-%d" % (M, N, K, planes))


# bias -> fp32 is lean mode 4; rows whose fp32 output is not 16-byte aligned (N = 7, 2827) take mode 7
LINEAR_CASES = [_linear_case(M, N, K, p, _lin(bn if p == 1 else 128, p, mode))
                for M, N, K, bn, mode in [(512, 256, 256, 128, 4), (300, 768, 256, 128, 4), (496, 7, 256, 128, 7),
                                          (992, 2827, 256, 128, 7), (1024, 256, 512, 128, 4), (64, 256, 64, 128, 4),
                                          (16650, 2827, 256, 256, 7), (16650, 7, 256, 128, 7)]   # last two: wide / unaligned rows
                for p in (1, 2)]


@pytest.mark.parametrize("M,N,K,planes,kernel", LINEAR_CASES)
def test_linear_matches_fp32(M, N, K, planes, kernel):
    ops = _ops()
    X, W, b = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5), _rand(N, seed=3)
    xa, wa = ops.act_from_float(X, planes), ops.act_from_float(W, planes)
    out = torch.empty(M, N, device=DEV)
    expect_kernels(kernel, lambda: ops.linear(xa, wa, M, N, K, bias=b, out_f32=out))
    ref = (xa.float().double() @ wa.float().double().t()).float() + b
    assert _rel(out, ref) < 2e-5
    if planes == 2:  # bf16x3 must track the un-rounded fp32 product
        full = (X.double() @ W.double().t()).float() + b
        assert _rel(out, full) < 3e-5


# (M, operand planes, act-output planes): every step at once has no lean epilogue, so all of these run mode 0
FULL_EPILOGUE_CASES = [pytest.param(M, p, op, kernel, id="%d-%d-%d" % (M, p, op)) for M, p, op, kernel in [
    (620, 1, 2, _lin(128, 1, 0)),           # single-plane operands, two-plane act output
    (16650, 1, 2, _lin(256, 1, 0)),
    (16650, 1, 1, _lin(256, 1, 0)),
    (16650, 2, 2, _lin(128, 2, 0)),         # parity mode
    (1, 1, 1, _lin(128, 1, 0)), (33, 1, 1, _lin(128, 1, 0)),          # fewer rows than one warp's 32
    (16384, 1, 1, _lin(128, 1, 0)), (16385, 1, 1, _lin(256, 1, 0)),  # the tile-width switch
]]


@pytest.mark.parametrize("M,planes,out_planes,kernel", FULL_EPILOGUE_CASES)
def test_linear_full_epilogue(M, planes, out_planes, kernel):
    """The generic run-time epilogue (mode 0) with every step enabled, against an fp64 restatement."""
    ops = _ops()
    N, K, rpg = 512, 256, 31
    X, W, b = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5), _rand(N, seed=3)
    res, rv = _rand(M, N, seed=4), _rand((M + rpg - 1) // rpg, N, seed=5)
    msk = (_rand(M, N, seed=6) > 0).float()
    sc = torch.tensor([0.75], device=DEV)
    xa, wa, ma = ops.act_from_float(X, planes), ops.act_from_float(W, planes), ops.act_from_float(msk, planes)
    out = torch.empty(M, N, device=DEV)
    oa = ops.Act(M, N, out_planes, DEV)
    expect_kernels(kernel, lambda: ops.linear(xa, wa, M, N, K, bias=b, scale_cols=100, scale=0.5, relu=True, rowvec=rv,
                                              rows_per_group=rpg, mask=ma, mask_scale=1.25, residual=res, out_f32=out,
                                              out_act=oa, acc_scale=sc))
    ref = (xa.float().double() @ wa.float().double().t()) * 0.75 + b.double()
    ref[:, :100] *= 0.5
    ref = torch.relu(ref) + rv.double().repeat_interleave(rpg, 0)[:M]
    ref = ref * msk.double() * 1.25 + res.double()
    assert _rel(out, ref) < 2e-5
    assert _rel(oa.float(), ref) < (2e-4 if out_planes == 2 else 6e-3)


_LEAN_MODE = {"dgrad": 1, "qkv": 2, "ffn1": 3, "resid": 4, "mask": 5, "head_dgrad": 6, "bias_f32": 4, "res_f32": 4}


def _lean_case(mode, M, N, planes, bn, K=256, ld=None, scale_cols=None, id=None):
    """ld > K: the operands' K padding is filled with NaN, which the result must not see (the TMA boxes clip at K)."""
    return pytest.param(mode, M, N, planes, K, ld or K, scale_cols, _lin(bn, planes, _LEAN_MODE[mode]),
                        id=id or "%d-%d-%d-%s" % (M, N, planes, mode) + ("" if K == 256 else "-K%d" % K))


LEAN_CASES = (
    # 128-wide (M <= 16384) and 256-wide (single plane, M > 16384, N > 128) tiles; parity mode is always 128 wide
    [_lean_case(mode, M, N, p, bn) for M, N, p, bn in [(1000, 256, 1, 128), (1000, 768, 1, 128), (1000, 128, 1, 128),
                                                      (16650, 256, 1, 256), (16650, 768, 1, 256), (33000, 512, 1, 256),
                                                      (1000, 256, 2, 128), (16650, 768, 2, 128), (33000, 512, 2, 128)]
     for mode in _LEAN_MODE]
    # the head dgrads at the model's contraction lengths: K = 2827 (ld 2880, the argument logits), 7 and 2 (ld 8)
    + [_lean_case("head_dgrad", 16650, 256, p, 256 if p == 1 else 128, K, ld)
       for p in (1, 2) for K, ld in ((2827, 2880), (7, 8), (2, 8))]
    # ragged N on the TMA-store modes: QKV of d_model 128 (N = 384: half a 256-wide tile) and ff = 520 (8 columns in the
    # last tile); M = 1000 stages the ReLU mask by TMA, M = 16650 loads it per thread
    + [_lean_case(mode, M, N, 1, bn, scale_cols=sc, id="%d-%d-1-%s" % (M, N, mode))
       for M, bn in ((1000, 128), (16650, 256)) for N, sc in ((384, 128), (520, 256))
       for mode in ("dgrad", "qkv", "ffn1", "mask")]
    # ragged K = ff = 520: the FFN second linear (residual stream) and its dgrad
    + [_lean_case(mode, M, 256, 1, bn, K=520, ld=520) for M, bn in ((1000, 128), (16650, 256)) for mode in ("resid", "dgrad")]
    # fewer rows than one warp's 32, and the tile-width switch
    + [_lean_case("dgrad", M, 256, 1, bn) for M, bn in ((1, 128), (33, 128), (16384, 128), (16385, 256))]
)


@pytest.mark.parametrize("mode,M,N,planes,K,ld,scale_cols,kernel", LEAN_CASES)
def test_linear_lean_epilogues(mode, M, N, planes, K, ld, scale_cols, kernel):
    """The compile-time specialised epilogues (one per GEMM role of the model) against the same fp64 restatement.
    M = 1000: the 128-wide kernels (8 consumer warps); M > 16384: the 256-wide persistent kernels (streamed bulk stores
    with 8 consumer warps for the bf16-output modes, 16 consumer warps for the fp32-output modes), with a ragged last row
    tile and several tiles per CTA.
    planes = 2: the parity-mode (bf16x3) kernels <128, 2, mode> with the same feature sets and hi + lo act outputs."""
    ops = _ops()
    rpg = 25
    X, W = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5)
    b, res, rv = _rand(N, seed=3), _rand(M, N, seed=4), _rand((M + rpg - 1) // rpg, N, seed=5)
    msk = torch.relu(_rand(M, N, seed=6))
    xa, wa = ops.act_from_float(X, planes, ld=ld), ops.act_from_float(W, planes, ld=ld)
    ma = ops.act_from_float(msk, planes)
    acc = (xa.float().double() @ wa.float().double().t()).float()
    if ld > K:
        xa.t[:, :, K:] = float("nan")
        wa.t[:, :, K:] = float("nan")
    of, oa = torch.zeros(M, N, device=DEV), ops.Act(M, N, planes, DEV)
    sc = torch.tensor([0.37], device=DEV)
    if scale_cols is None:
        scale_cols = N // 4 * 2
    run = lambda **kw: expect_kernels(kernel, lambda: ops.linear(xa, wa, M, N, K, **kw))   # noqa: E731
    if mode == "dgrad":
        run(out_act=oa)
        ref, got = acc, oa.float()
    elif mode == "qkv":
        run(bias=b, scale_cols=scale_cols, scale=0.25, out_act=oa)
        ref = acc + b
        ref[:, :scale_cols] *= 0.25
        got = oa.float()
    elif mode == "ffn1":
        run(bias=b, relu=True, drop=(0.2, 5, 77), out_act=oa)
        ka = ops.Act(M, N, 1, DEV)
        ops.cast_act(torch.ones(M, N, device=DEV), M, N, out=ka, drop=(0.2, 5, 77))
        ref, got = torch.relu(acc + b) * ka.float(), oa.float()
    elif mode == "resid":
        run(bias=b, drop=(0.2, 6, 77), rowvec=rv, rows_per_group=rpg, residual=res, out_f32=of)
        ka = ops.Act(M, N, 1, DEV)
        ops.cast_act(torch.ones(M, N, device=DEV), M, N, out=ka, drop=(0.2, 6, 77))
        got = of
        ref = (acc + b) * (ka.float() != 0) / (1 - 13107 / 65536.0) + rv.repeat_interleave(rpg, 0)[:M] + res
    elif mode == "mask":
        run(mask=ma, mask_scale=1.25, out_act=oa)
        ref, got = acc * (ma.float() != 0) * 1.25, oa.float()
    elif mode == "bias_f32":     # linear_global / VAE heads: bias only, fp32 out (lean mode 4 without residual)
        run(bias=b, out_f32=of)
        ref, got = acc + b, of
    elif mode == "res_f32":      # dgrad accumulated into an fp32 gradient (lean mode 4 without bias)
        of.copy_(res)
        run(residual=of, out_f32=of)
        ref, got = acc + res, of
    else:
        run(acc_scale=sc, residual=res, out_f32=of)
        ref, got = acc * 0.37 + res, of
    tol = 2e-5 if got is of else (6e-3 if planes == 1 else 4e-5)   # bf16 output rounding (one plane) / hi + lo planes
    if mode == "ffn1":
        ref = torch.relu(acc + b) * (ka.float() != 0) / (1 - 13107 / 65536.0)
    assert _rel(got, ref) < tol, mode


def test_linear_dropout_statistics_and_determinism():
    ops = _ops()
    M, N, K = 1024, 256, 64
    X = torch.ones(M, K, device=DEV)
    W = torch.ones(N, K, device=DEV) / K
    xa, wa = ops.act_from_float(X, 1), ops.act_from_float(W, 1)
    o1, o2, o3 = (torch.empty(M, N, device=DEV) for _ in range(3))
    ops.linear(xa, wa, M, N, K, drop=(0.1, 7, 1234), out_f32=o1)
    ops.linear(xa, wa, M, N, K, drop=(0.1, 7, 1234), out_f32=o2)
    ops.linear(xa, wa, M, N, K, drop=(0.1, 8, 1234), out_f32=o3)
    assert torch.equal(o1, o2) and not torch.equal(o1, o3)
    keep = (o1 != 0).float().mean().item()
    assert abs(keep - 0.9) < 0.005
    assert torch.allclose(o1[o1 != 0], torch.tensor(1 / 0.9, device=DEV), rtol=1e-5)
    # cast_act regenerates the same mask from (seed, site, row*N+col)
    ca = ops.Act(M, N, 1, DEV)
    ops.cast_act(torch.ones(M, N, device=DEV), M, N, out=ca, drop=(0.1, 7, 1234))
    assert torch.equal(ca.float() != 0, o1 != 0)


OUTER_CASES = [pytest.param(M, P, Q, p, "outer_kernel<%d, %d>" % (bq, p), id="%d-%d-%d-%d" % (M, P, Q, p))
               for M, P, Q, bq in [(4096, 768, 256, 256), (1000, 300, 200, 256), (2048, 2827, 64, 128), (992, 7, 256, 256),
                                   (130, 256, 512, 256),
                                   (640, 100, 30, 128), (20000, 512, 256, 256),    # Q % 4 != 0: scalar reductions; many row blocks
                                   # M >= 16384, the path-level weight gradients: many 128 x 256 tiles (2827 x 256,
                                   # 1536 x 512 with bias sums only from the first Q tile, 512 x 512), ragged P with
                                   # Q % 4 != 0 (scalar reductions), ragged P and Q
                                   (16500, 2827, 256, 256), (20000, 1536, 512, 256), (16500, 512, 512, 256),
                                   (17000, 1000, 250, 256), (33000, 600, 300, 256),
                                   # few tiles at the same row counts; M = 131072: splits capped at 48 row blocks
                                   (20000, 768, 256, 256), (17000, 256, 512, 256), (33000, 300, 200, 256),
                                   (131072, 768, 256, 256)]
               for p in (1, 2)]


@pytest.mark.parametrize("M,P,Q,planes,kernel", OUTER_CASES)
def test_outer_matches_fp32(M, P, Q, planes, kernel):
    """128-row tiles, 256 (Q > 128) or 128 columns wide; planes = 2 is parity mode (three products per K step)."""
    ops = _ops()
    A, B = _rand(M, P, seed=1), _rand(M, Q, seed=2)
    lda, ldb = (P + 7) // 8 * 8, (Q + 7) // 8 * 8
    aa, ba = ops.act_from_float(A, planes, ld=lda), ops.act_from_float(B, planes, ld=ldb)
    Cout = torch.ones(P, Q, device=DEV)
    cs = torch.ones(P, device=DEV)
    sc = torch.tensor([2.0], device=DEV)
    expect_kernels(kernel, lambda: ops.outer(aa, ba, M, P, Q, Cout, alpha=0.5, alpha_dev=sc, colsum=cs))
    ref = (aa.float().double().t() @ ba.float().double()).float() + 1.0
    assert _rel(Cout, ref) < 2e-5
    assert _rel(cs, aa.float().double().sum(0).float() + 1.0) < 2e-5   # fused bias-gradient column sums
    if planes == 2:
        assert _rel(Cout, (A.double().t() @ B.double()).float() + 1.0) < 3e-5


@pytest.mark.parametrize("M,d,ff", [(20000, 256, 512), (131072, 256, 512), (16500, 128, 256), (17000, 512, 512), (16400, 200, 300)])
def test_outer_group_matches_fp32(M, d, ff):
    """dsvg_outer_group: the four weight gradients of one block (in_proj, out_proj, linear1, linear2) in one launch, every
    problem with its bias column sums, accumulating into non-zero buffers; ragged tile edges at d = 128 / 200."""
    ops = _ops()
    shapes = [(3 * d, d), (d, d), (ff, d), (d, ff)]
    probs, refs = [], []
    for i, (P, Q) in enumerate(shapes):
        A, B = _rand(M, P, seed=10 + i), _rand(M, Q, seed=20 + i)
        aa = ops.act_from_float(A, 1, ld=(P + 7) // 8 * 8)
        ba = ops.act_from_float(B, 1, ld=(Q + 7) // 8 * 8)
        Cout = torch.full((P, Q), 0.5, device=DEV)
        cs = torch.full((P,), -1.0, device=DEV)
        probs.append((aa, ba, P, Q, Cout, cs))
        refs.append(((aa.float().double().t() @ ba.float().double()).float() + 0.5, aa.float().double().sum(0).float() - 1.0))
    ops.outer_group(probs, M)
    for (aa, ba, P, Q, Cout, cs), (rc, rs) in zip(probs, refs):
        assert _rel(Cout, rc) < 2e-5, (P, Q)
        assert _rel(cs, rs) < 2e-5, (P, Q)


# ------------------------------------------------------------------------------------------------ LayerNorm
LAYERNORM_CASES = [pytest.param(D, p, ("ln_fwd_kernel<%d>" % (D // 128), "ln_bwd_kernel<%d>" % (D // 128)),
                                id="%d" % D if p == 0 else "%d-drop%g" % (D, p))
                   for p in (0.0, 0.1) for D in (128, 256, 512)]


@pytest.mark.parametrize("D,drop_p,kernels", LAYERNORM_CASES)
def test_layernorm_fwd_bwd(D, drop_p, kernels):
    ops = _ops()
    M = 777
    x, g, b = _rand(M, D, seed=1), 1 + 0.1 * _rand(D, seed=2), 0.1 * _rand(D, seed=3)
    y = ops.Act(M, D, 2, DEV)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    expect_kernels(kernels[0], lambda: ops.ln_fwd(x, g, b, y, mean, rstd, M, D))
    xr = x.clone().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref = F.layer_norm(xr, (D,), gr, br, 1e-5)
    assert _rel(y.float(), ref.detach()) < 1e-4
    dy, dx_in = _rand(M, D, seed=4), _rand(M, D, seed=5)
    dya = ops.act_from_float(dy, 2)
    ref.backward(dya.float())
    dx = torch.empty(M, D, device=DEV)
    dact = ops.Act(M, D, 2, DEV)
    dg, db = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV)
    drop = (drop_p, 9, 77) if drop_p > 0 else (0.0, 0, 0)
    expect_kernels(kernels[1], lambda: ops.ln_bwd(x, mean, rstd, g, M, D, dy=dya, dx_in=dx_in, dx_out=dx, dact=dact,
                                                  drop=drop, dgamma=dg, dbeta=db))
    want = xr.grad + dx_in
    assert _rel(dx, want) < 2e-5
    if drop_p > 0:      # dact = dropout(dx_out): zeros at rate p, kept entries scaled by 1 / (1 - p)
        zero = dact.float() == 0
        assert abs(zero.float().mean().item() - drop_p) < 0.01
        assert _rel(dact.float()[~zero], (want / (1 - drop_p))[~zero]) < 1e-4
    else:
        assert _rel(dact.float(), want) < 1e-4
    assert _rel(dg, gr.grad) < 2e-5 and _rel(db, br.grad) < 2e-5


LN_FUSED_CASES = [pytest.param(M, K, rv, p, _lin(256, 1, 8), id="%d-%d-%s-%s" % (M, K, rv, p))
                  for M, K, rv, p in [(16500, 256, False, 0.0), (16500, 512, True, 0.1), (33000, 256, True, 0.1),
                                      (20000, 512, False, 0.2)]]


@pytest.mark.parametrize("M,K,rowvec,drop_p,kernel", LN_FUSED_CASES)
def test_linear_layernorm_fused_forward(M, K, rowvec, drop_p, kernel):
    """dsvg_linear_ln_fwd == dsvg_linear (residual-stream epilogue) followed by dsvg_ln_fwd: same fp32 residual stream bit
    for bit (same arithmetic, same dropout draws), LayerNorm output and statistics to rounding; and against plain fp32
    torch when dropout is off."""
    ops = _ops()
    N = 256
    assert ops.ln_fusable(M, N, 1) and not ops.ln_fusable(M, N, 2) and not ops.ln_fusable(4096, N, 1)
    X = ops.act_from_float(_rand(M, K, seed=1, scale=0.5), 1)
    W = ops.act_from_float(_rand(N, K, seed=2, scale=0.1), 1)
    bias, res = _rand(N, seed=3), _rand(M, N, seed=4, scale=2.0) + 1.5      # a non-zero row mean (variance by E[x^2]-m^2)
    g, b = 1 + 0.1 * _rand(N, seed=5), 0.1 * _rand(N, seed=6)
    L = 31
    rv = _rand((M + L - 1) // L, N, seed=7) if rowvec else None
    drop = (drop_p, 5, 1234) if drop_p > 0 else (0.0, 0, 0)
    kw = dict(bias=bias, drop=drop, rowvec=rv, rows_per_group=L if rowvec else 1, residual=res)
    x_a, x_b = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
    y_a, y_b = ops.Act(M, N, 1, DEV), ops.Act(M, N, 1, DEV)
    m_a, r_a, m_b, r_b = (torch.empty(M, device=DEV) for _ in range(4))
    ops.linear(X, W, M, N, K, out_f32=x_a, **kw)
    ops.ln_fwd(x_a, g, b, y_a, m_a, r_a, M, N)
    expect_kernels(kernel, lambda: ops.linear(X, W, M, N, K, out_f32=x_b, ln=(g, b, y_b, m_b, r_b), **kw))
    assert (x_a - x_b).abs().max().item() <= 2e-6 * x_a.abs().max().item()      # same arithmetic up to FMA contraction
    assert _rel(m_b, m_a) < 1e-5 and _rel(r_b, r_a) < 1e-4
    # the two outputs are bf16 roundings of values that agree to ~1e-6: at most one bf16 ulp apart
    assert ((y_a.float() - y_b.float()).abs() <= 2.0 ** -7 * y_a.float().abs() + 1e-6).all()
    assert (y_a.t != y_b.t).float().mean().item() < 0.02
    if drop_p == 0:
        ref = X.float() @ W.float().t() + bias + res
        if rowvec:
            ref = ref + rv[torch.arange(M, device=DEV) // L]
        assert _rel(x_b, ref) < 1e-5
        assert _rel(y_b.float(), F.layer_norm(ref, (N,), g, b, 1e-5)) < 1e-2


LN_POOL_CASES = [pytest.param(D, "ln_pool_fwd_kernel<%d>" % (D // 128), id=str(D)) for D in (128, 256, 512)]


@pytest.mark.parametrize("D,kernel", LN_POOL_CASES)
def test_layernorm_pool_fwd_bwd(D, kernel):
    ops = _ops()
    nseq, L = 96, 31
    M = nseq * L
    x, g, b = _rand(M, D, seed=1), 1 + 0.1 * _rand(D, seed=2), 0.1 * _rand(D, seed=3)
    lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(9))
    valid = (torch.arange(L)[None, :] < lens[:, None]).to(torch.uint8).to(DEV).reshape(-1).contiguous()
    z = torch.empty(nseq, D, device=DEV)
    mean, rstd, ic = torch.empty(M, device=DEV), torch.empty(M, device=DEV), torch.empty(nseq, device=DEV)
    expect_kernels(kernel, lambda: ops.ln_pool_fwd(x, g, b, valid, z, mean, rstd, ic, nseq, L, D))
    xr = x.clone().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    w = valid.float().reshape(nseq, L, 1)
    ref = (F.layer_norm(xr, (D,), gr, br, 1e-5).reshape(nseq, L, D) * w).sum(1) / w.sum(1)
    assert _rel(z, ref.detach()) < 2e-5
    dz = _rand(nseq, D, seed=4)
    ref.backward(dz)
    dx = torch.empty(M, D, device=DEV)
    dg, db = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV)
    ops.ln_bwd(x, mean, rstd, g, M, D, dz=dz, valid=valid, inv_cnt=ic, L=L, dx_out=dx, dgamma=dg, dbeta=db)
    assert _rel(dx, xr.grad) < 2e-5
    assert _rel(dg, gr.grad) < 2e-5 and _rel(db, br.grad) < 2e-5


# ------------------------------------------------------------------------------------------------ attention
def _attn_fwd_bwd_case(L, H, hd, masked, nseq, planes, kernels, new=True):
    ident = "%d-%d-%d-%s-%d" % (L, H, hd, masked, nseq)
    return pytest.param(L, H, hd, masked, nseq, planes, kernels, id=ident + ("-p%d" % planes if new else ""))


ATTN_FWD_BWD_CASES = (
    [_attn_fwd_bwd_case(*c, 2, k, new=False) for *c, k in [
        (32, 8, 32, True, 37, _attn("x3")), (31, 8, 32, False, 37, _attn("x3")), (8, 8, 32, True, 37, _attn("x3")),
        (52, 4, 64, True, 37, _attn("gx3", 64, 4)), (66, 8, 64, False, 37, _attn("gx3", 64, 5)),
        (8, 4, 16, False, 37, _attn("simt", 16)), (31, 8, 32, True, 1500, _attn("x3")),
        (66, 8, 64, True, 300, _attn("gx3", 64, 5)), (52, 8, 32, True, 300, _attn("gx3", 32, 4)),
        (16, 8, 64, True, 300, _attn("gx3", 64, 1))]]
    # every parity-mode general kernel <head_dim, 16-row tiles>, at one past the previous tile count and at the top of its own
    + [_attn_fwd_bwd_case(L, 4, hd, L % 2 == 1, 40, 2, _attn("gx3", hd, nt))
       for hd, L, nt in ((32, 33, 3), (32, 48, 3), (32, 49, 4), (32, 64, 4), (32, 65, 5), (32, 80, 5),
                         (64, 1, 1), (64, 17, 2), (64, 32, 2), (64, 33, 3), (64, 48, 3), (64, 49, 4), (64, 64, 4),
                         (64, 80, 5))]
    # fp32 SIMT (head_dim 16 at any length, every head_dim above 80 positions), one and two planes: L = 33 runs the row
    # loops twice, L = 81 on two warps per block, the longest accepted length on one warp per block
    + [_attn_fwd_bwd_case(L, 128 // hd, hd, masked, nseq, p, _attn("simt", hd))
       for hd, L, masked, nseq in ((16, 33, True, 20), (16, 81, False, 8), (16, ATTN_MAX_L[16], True, 3),
                                   (32, 81, True, 8), (32, ATTN_MAX_L[32], False, 3),
                                   (64, 81, False, 8), (64, ATTN_MAX_L[64], True, 3))
       for p in (1, 2)]
)


@pytest.mark.parametrize("L,H,hd,masked,nseq,planes,kernels", ATTN_FWD_BWD_CASES)
def test_attention_fwd_bwd(L, H, hd, masked, nseq, planes, kernels):
    """Two-plane (parity mode) operands: 32 x 32 bf16x3 mma kernels (head_dim 32, L <= 32), general bf16x3 kernels
    (head_dim 32 / 64, L <= 80), fp32 SIMT for the rest (head_dim 16, L > 80), against an fp64 restatement.  Single-plane
    operands on the SIMT kernels: P and dS stay fp32 there, so the bf16 rounding of the outputs is the only error."""
    ops = _ops()
    d = H * hd
    M = nseq * L
    qkv = _rand(M, 3 * d, seed=1, scale=0.7)
    qa = ops.act_from_float(qkv, planes)
    qv = qa.float().double().requires_grad_(True)
    valid = None
    vmask = None
    if masked:
        lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(3))
        vmask = (torch.arange(L)[None, :] < lens[:, None]).to(DEV)
        valid = vmask.to(torch.uint8).reshape(-1).contiguous()
    out = ops.Act(M, d, planes, DEV)
    expect_kernels(kernels[0], lambda: ops.attn_fwd(qa, valid, out, nseq, L, H, hd, (0.0, 0, 0)))
    q, k, v = (t.reshape(nseq, L, H, hd).transpose(1, 2) for t in qv.split(d, dim=-1))
    s = q @ k.transpose(-1, -2)
    if masked:
        s = s.masked_fill(~vmask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(M, d)
    tol = 1e-4 if planes == 2 else 5e-3
    assert _rel(out.float(), ref.detach()) < tol
    do = _rand(M, d, seed=5)
    da = ops.act_from_float(do, planes)
    ref.backward(da.float().double())
    dqkv = ops.Act(M, 3 * d, planes, DEV)
    expect_kernels(kernels[1], lambda: ops.attn_bwd(qa, valid, da, dqkv, nseq, L, H, hd, 0.5, (0.0, 0, 0)))
    g = qv.grad.clone()
    g[:, :d] *= 0.5     # dq carries the folded query scaling
    assert _rel(dqkv.float(), g) < tol


@pytest.mark.parametrize("hd", [16, 32, 64])
def test_attention_backward_past_the_length_limit_is_refused(hd):
    """One position past the longest accepted sequence the backward's tiles exceed shared memory: dsvg_attn_bwd must
    return the host-side error instead of launching."""
    from deepsvg_b200 import _lib
    ops = _ops()
    L, H, nseq = ATTN_MAX_L[hd] + 1, 128 // hd, 2
    M = nseq * L
    qa, da = ops.act_from_float(_rand(M, 384, seed=1), 1), ops.act_from_float(_rand(M, 128, seed=2), 1)
    dqkv = ops.Act(M, 384, 1, DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="sequence length %d too long for shared memory" % L):
        ops.attn_bwd(qa, None, da, dqkv, nseq, L, H, hd, 1.0, (0.0, 0, 0))
    assert _lib.launch_count() == n0


ATTN_MMA_CASES = [pytest.param(L, m, n, _attn("mma"), id="%d-%s-%d" % (L, m, n))
                  for L, m, n in [(32, True, 61), (31, False, 61), (8, True, 61), (17, True, 61), (31, True, 1500),
                                  (8, True, 2600)]]


@pytest.mark.parametrize("L,masked,nseq,kernels", ATTN_MMA_CASES)
def test_attention_mma_fast_path(L, masked, nseq, kernels):
    """Single-plane bf16, head_dim 32, L <= 32 -> the mma.sync kernels; P and dS are rounded to bf16 inside.
    The large nseq cases make every CTA of the block-per-sequence kernels loop over several sequences."""
    ops = _ops()
    H, hd = 8, 32
    d, M = H * hd, nseq * L
    qa = ops.act_from_float(_rand(M, 3 * d, seed=1, scale=0.7), 1)
    qv = qa.float().clone().requires_grad_(True)
    valid = vmask = None
    if masked:
        lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(3))
        vmask = (torch.arange(L)[None, :] < lens[:, None]).to(DEV)
        valid = vmask.to(torch.uint8).reshape(-1).contiguous()
    out = ops.Act(M, d, 1, DEV)
    expect_kernels(kernels[0], lambda: ops.attn_fwd(qa, valid, out, nseq, L, H, hd, (0.0, 0, 0)))
    q, k, v = (t.reshape(nseq, L, H, hd).transpose(1, 2) for t in qv.split(d, dim=-1))
    s = q @ k.transpose(-1, -2)
    if masked:
        s = s.masked_fill(~vmask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(M, d)
    assert _rel(out.float(), ref.detach()) < 1.5e-2
    da = ops.act_from_float(_rand(M, d, seed=5), 1)
    ref.backward(da.float())
    dqkv = ops.Act(M, 3 * d, 1, DEV)
    expect_kernels(kernels[1], lambda: ops.attn_bwd(qa, valid, da, dqkv, nseq, L, H, hd, 0.5, (0.0, 0, 0)))
    g = qv.grad.clone()
    g[:, :d] *= 0.5
    for lo, hi, nm in ((0, d, "dq"), (d, 2 * d, "dk"), (2 * d, 3 * d, "dv")):
        e = (dqkv.float()[:, lo:hi] - g[:, lo:hi]).norm() / g[:, lo:hi].norm()
        assert e.item() < 1.5e-2, (nm, e.item())


ATTN_GMMA_CASES = (
    [pytest.param(*c, _attn("gmma", c[2], nt), id="%d-%d-%d-%s-%d" % tuple(c)) for *c, nt in [
        (52, 8, 32, True, 40, 4), (51, 8, 32, False, 40, 4), (66, 8, 64, True, 33, 5), (65, 8, 64, False, 33, 5),
        (16, 8, 64, True, 50, 1), (33, 4, 32, True, 3000, 3), (80, 2, 64, True, 7, 5), (8, 8, 64, True, 64, 1)]]
    # every reachable <head_dim, 16-row tiles> at one past the previous tile count and at the top of its own
    # (head_dim 32 with L <= 32 runs the 32 x 32 kernels)
    + [pytest.param(L, 4, hd, L % 2 == 1, 40, _attn("gmma", hd, nt), id="%d-4-%d-%s-40" % (L, hd, L % 2 == 1))
       for hd, L, nt in ((32, 48, 3), (32, 49, 4), (32, 64, 4), (32, 65, 5), (32, 80, 5),
                         (64, 2, 1), (64, 17, 2), (64, 32, 2), (64, 33, 3), (64, 48, 3), (64, 49, 4), (64, 64, 4))]
)


@pytest.mark.parametrize("L,H,hd,masked,nseq,kernels", ATTN_GMMA_CASES)
def test_attention_general_tensor_core_path(L, H, hd, masked, nseq, kernels):
    """Single-plane bf16, head_dim 32 / 64, L <= 80 (one-stage fonts L = 52 / 51, scaled hierarchical L = 66 / 65 and
    16 group-level) -> attn_gmma kernels (CTA per (sequence, head), warp per 16-row query tile).  Same bound as the
    32 x 32 fast path: P and dS are rounded to bf16 inside."""
    ops = _ops()
    d, M = H * hd, nseq * L
    qa = ops.act_from_float(_rand(M, 3 * d, seed=1, scale=0.7), 1)
    qv = qa.float().double().requires_grad_(True)
    valid = vmask = None
    if masked:
        lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(3))
        vmask = (torch.arange(L)[None, :] < lens[:, None]).to(DEV)
        valid = vmask.to(torch.uint8).reshape(-1).contiguous()
    out = ops.Act(M, d, 1, DEV)
    expect_kernels(kernels[0], lambda: ops.attn_fwd(qa, valid, out, nseq, L, H, hd, (0.0, 0, 0)))
    q, k, v = (t.reshape(nseq, L, H, hd).transpose(1, 2) for t in qv.split(d, dim=-1))
    s = q @ k.transpose(-1, -2)
    if masked:
        s = s.masked_fill(~vmask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(M, d)
    assert _rel(out.float(), ref.detach()) < 1.5e-2
    da = ops.act_from_float(_rand(M, d, seed=5), 1)
    ref.backward(da.float().double())
    dqkv = ops.Act(M, 3 * d, 1, DEV)
    expect_kernels(kernels[1], lambda: ops.attn_bwd(qa, valid, da, dqkv, nseq, L, H, hd, 0.5, (0.0, 0, 0)))
    g = qv.grad.clone()
    g[:, :d] *= 0.5
    for lo, hi, nm in ((0, d, "dq"), (d, 2 * d, "dk"), (2 * d, 3 * d, "dv")):
        e = (dqkv.float()[:, lo:hi] - g[:, lo:hi]).norm() / g[:, lo:hi].norm()
        assert e.item() < 1.5e-2, (nm, e.item())


ATTN_DROPOUT_CASES = (
    [pytest.param(p, n, 66, 8, 64, _attn("gmma" if p == 1 else "gx3", 64, 5), id="%d-%d" % (p, n))
     for p, n in [(1, 9), (2, 9), (2, 700)]]
    # the SIMT kernels above 32 positions (several row / column chunks per lane).  Two planes only: one bf16 plane rounds
    # out and dv independently, and that noise alone reaches the 2e-2 bound of this cancelling sum
    + [pytest.param(2, n, L, 128 // hd, hd, _attn("simt", hd), id="2-%d-L%d-hd%d" % (n, L, hd))
       for n, L, hd in [(200, 81, 16), (200, ATTN_MAX_L[64], 64), (100, ATTN_MAX_L[32], 32)]]
)


@pytest.mark.parametrize("planes,nseq,L,H,hd,kernels", ATTN_DROPOUT_CASES)
def test_attention_general_path_dropout_consistent(planes, nseq, L, H, hd, kernels):
    """planes = 2: the parity-mode (bf16x3) variant of the general kernels; nseq = 700: every CTA strides over several pairs.
    With dropout, out is linear in v for the fixed probabilities and mask: out(v) . g == v . dv(g)."""
    ops = _ops()
    d, M = H * hd, nseq * L
    qa = ops.act_from_float(_rand(M, 3 * d, seed=1, scale=0.5), planes)
    drop = (0.3, 11, 99)
    o1, o2, o0 = ops.Act(M, d, planes, DEV), ops.Act(M, d, planes, DEV), ops.Act(M, d, planes, DEV)
    expect_kernels(kernels[0], lambda: ops.attn_fwd(qa, None, o1, nseq, L, H, hd, drop))
    ops.attn_fwd(qa, None, o2, nseq, L, H, hd, drop)
    ops.attn_fwd(qa, None, o0, nseq, L, H, hd, (0.0, 0, 0))
    assert torch.equal(o1.t, o2.t) and not torch.equal(o1.t, o0.t)
    ga = ops.act_from_float(_rand(M, d, seed=2), planes)
    dqkv = ops.Act(M, 3 * d, planes, DEV)
    expect_kernels(kernels[1], lambda: ops.attn_bwd(qa, None, ga, dqkv, nseq, L, H, hd, 1.0, drop))
    lhs = (o1.float().double() * ga.float().double()).sum().item()
    rhs = (qa.float()[:, 2 * d:].double() * dqkv.float()[:, 2 * d:].double()).sum().item()
    assert abs(lhs - rhs) < (2e-3 if planes == 2 else 2e-2) * abs(lhs)
    # dropout keeps the mean: E[out] = out(no dropout)
    assert abs(o1.float().mean().item() - o0.float().mean().item()) < 5e-3 * o0.float().abs().mean().item() + 1e-4


@pytest.mark.parametrize("planes", [1, 2])
def test_attention_dropout_consistent_fwd_bwd(planes):
    """With dropout the backward must use the forward's mask: check d(out . w)/dv against finite structure."""
    ops = _ops()
    nseq, L, H, hd = 5, 32, 8, 32
    d, M = H * hd, nseq * L
    qkv = _rand(M, 3 * d, seed=1, scale=0.5)
    qa = ops.act_from_float(qkv, planes)
    drop = (0.3, 11, 99)
    o1, o2 = ops.Act(M, d, planes, DEV), ops.Act(M, d, planes, DEV)
    ops.attn_fwd(qa, None, o1, nseq, L, H, hd, drop)
    ops.attn_fwd(qa, None, o2, nseq, L, H, hd, drop)
    assert torch.equal(o1.t, o2.t)
    # out is linear in v for fixed probabilities+mask: out(v) . g == v . dv(g)
    g = _rand(M, d, seed=2)
    ga = ops.act_from_float(g, planes)
    dqkv = ops.Act(M, 3 * d, planes, DEV)
    ops.attn_bwd(qa, None, ga, dqkv, nseq, L, H, hd, 1.0, drop)
    lhs = (o1.float() * ga.float()).sum().item()
    rhs = (qa.float()[:, 2 * d:] * dqkv.float()[:, 2 * d:]).sum().item()
    assert abs(lhs - rhs) < (2e-3 if planes == 2 else 2e-2) * abs(lhs)
    keep = (o1.float().abs() > 0).float().mean().item()   # dropped probabilities thin the output but never zero a row
    assert keep > 0.99


# ------------------------------------------------------------------------------------------------ embedding
EMBED_CASES = [pytest.param(g, d, "embed_fwd_kernel<%d>" % (d // 128), id=str(g) if d == 256 else "%s-d%d" % (g, d))
               for g, d in [(False, 256), (True, 256), (False, 128), (True, 512)]]


@pytest.mark.parametrize("use_grp,d,kernel", EMBED_CASES)
def test_embedding_fwd_bwd(use_grp, d, kernel):
    ops = _ops()
    from oracle import svg_oracle as O
    cfg = O.make_cfg("one_stage" if use_grp else "hierarchical", max_total_len=30)
    n = 6
    cmd, arg = O.synth_batch(cfg, n, seed=5)
    G, L = cmd.shape[1], cmd.shape[2]
    nseq, T, V, na = n * G, n * G * L, 257, 11
    cmd, arg = cmd.to(DEV).contiguous(), arg.to(DEV).contiguous()
    Ec, Ea = _rand(7, d, seed=1), _rand(V, 64, seed=2)
    W, b = _rand(d, 64 * na, seed=3, scale=0.05), _rand(d, seed=4)
    Pt, Gt = _rand(L, d, seed=5), _rand(10, d, seed=6)
    grp = torch.empty(T, dtype=torch.uint8, device=DEV)
    ops.seq_prep(cmd, nseq, L, None, None, None, grp, None)
    table, base = torch.empty(na * V, d, device=DEV), torch.empty(d, device=DEV)
    ops.embed_fold(Ea, W, b, table, base, V, na, d)
    x = torch.empty(T, d, device=DEV)
    expect_kernels(kernel, lambda: ops.embed_fwd(cmd, arg, grp if use_grp else None, Ec, table, base, Pt,
                                                 Gt if use_grp else None, x, T, L, V, na, d, (0.0, 0, 0)))
    leaves = [t.clone().requires_grad_(True) for t in (Ec, Ea, W, b, Pt, Gt)]
    ec, ea, w, bb, pt, gt = leaves
    ci = cmd.long().reshape(-1)
    ref = ec[ci] + F.linear(ea[(arg + 1).long()].reshape(T, -1), w, bb) + pt.repeat(nseq, 1)
    if use_grp:
        ref = ref + gt[(cmd.long() == 0).cumsum(-1).reshape(-1)]
    assert _rel(x, ref.detach()) < 2e-5
    dx = _rand(T, d, seed=7)
    ref.backward(dx)
    grads = [torch.zeros_like(t) for t in (Ec, Ea, W, b, Pt, Gt)]
    scratch = torch.empty(na * V, d, device=DEV)
    ops.embed_bwd(cmd, arg, grp if use_grp else None, dx, Ea, W, grads[0], grads[4], grads[5] if use_grp else None,
                  grads[1], grads[2], grads[3], scratch, nseq, L, V, na, d, 10, (0.0, 0, 0))
    for name, got, leaf in zip("Ec Ea W b Pt Gt".split(), grads, leaves):
        if name == "Gt" and not use_grp:
            continue
        assert _rel(got, leaf.grad) < 5e-5, name


def test_seq_prep_matches_oracle_masks():
    ops = _ops()
    from oracle import svg_oracle as O
    cfg = O.make_cfg("hierarchical")
    cmd, _ = O.synth_batch(cfg, 16, seed=3)
    n, G, L = cmd.shape
    c = cmd.to(DEV).contiguous()
    nseq = n * G
    fe = torch.empty(nseq, dtype=torch.int32, device=DEV)
    vis = torch.empty(nseq, dtype=torch.uint8, device=DEV)
    kv = torch.empty(nseq * L, dtype=torch.uint8, device=DEV)
    grp = torch.empty(nseq * L, dtype=torch.uint8, device=DEV)
    counts = torch.zeros(2, device=DEV)
    ops.seq_prep(c, nseq, L, fe, vis, kv, grp, counts)
    ci = cmd.long()
    assert torch.equal(kv.cpu().bool().reshape(n, G, L), ~O.key_padding(ci))
    assert torch.equal(vis.cpu().bool().reshape(n, G), O.visibility(ci))
    assert torch.equal(grp.cpu().long().reshape(n, G, L), O.group_index(ci))
    wc = (O.extended_padding(ci) * O.visibility(ci).unsqueeze(-1).float())[..., 1:]
    wa = O.CMD_ARGS_MASK[ci[..., 1:]]
    assert counts[0].item() == wc.sum().item() and counts[1].item() == wa.sum().item()


def test_rows_embed_and_segsum():
    ops = _ops()
    nseq, L, d = 40, 31, 256
    R = nseq * L
    tab, add = _rand(L, d, seed=1), _rand(R, d, seed=2)
    x = torch.empty(R, d, device=DEV)
    ops.rows_embed_fwd(add, tab, x, R, L, d, (0.0, 0, 0))
    assert torch.allclose(x, add + tab.repeat(nseq, 1))
    dx = _rand(R, d, seed=3)
    dadd, dtab = torch.empty(R, d, device=DEV), torch.zeros(L, d, device=DEV)
    ops.rows_embed_bwd(dx, dadd, dtab, nseq, L, d, (0.0, 0, 0))
    assert torch.equal(dadd, dx) and _rel(dtab, dx.reshape(nseq, L, d).sum(0)) < 1e-5
    s = torch.empty(nseq, d, device=DEV)
    ops.seg_sum(dx, nseq, L, d, out_f32=s)
    assert _rel(s, dx.reshape(nseq, L, d).sum(1)) < 1e-5
    cs = torch.zeros(d, device=DEV)
    a = ops.act_from_float(dx, 2)
    ops.colsum(a, R, d, cs)
    assert _rel(cs, a.float().sum(0)) < 1e-5


# ------------------------------------------------------------------------------------------------ loss
CE_CASES = [pytest.param(257, "ce_args_kernel<9>", id="257"),
            pytest.param(512, "ce_args_kernel<16>", id="512")]   # relative argument targets: 2 * args_dim classes


@pytest.mark.parametrize("n_classes,kernel", CE_CASES)
def test_cross_entropy_kernels(n_classes, kernel):
    ops = _ops()
    from oracle import svg_oracle as O
    cfg = O.make_cfg("hierarchical")
    n = 8
    cmd, arg = O.synth_batch(cfg, n, seed=11)
    G, L = cmd.shape[1], cmd.shape[2]
    nseq, Ld = n * G, L - 1
    Md = nseq * Ld
    nw = 11 * n_classes
    ldw = nw // 64 * 64 + 64
    al = _rand(Md, nw, seed=1, scale=2.0)
    cl, vl = _rand(Md, 7, seed=2, scale=2.0), _rand(nseq, 2, seed=3)
    c, a = cmd.to(DEV).contiguous(), arg.to(DEV).contiguous()
    fe = torch.empty(nseq, dtype=torch.int32, device=DEV)
    vis = torch.empty(nseq, dtype=torch.uint8, device=DEV)
    counts, acc, out = torch.zeros(2, device=DEV), torch.zeros(8, device=DEV), torch.zeros(8, device=DEV)
    ops.seq_prep(c, nseq, L, fe, vis, None, None, counts)
    dla, dlc, dlv = ops.Act(Md, nw, 2, DEV, ld=ldw, zero=True), ops.Act(Md, 7, 2, DEV, ld=8), ops.Act(nseq, 2, 2, DEV, ld=8)
    expect_kernels(kernel, lambda: ops.ce_args(al, nw, c, a, counts, dla, acc, nseq, L, 11, n_classes))
    ops.ce_cmd(cl, c, fe, vis, counts, dlc, acc, nseq, L, 7)
    ops.ce_vis(vl, vis, dlv, acc, nseq, 1.0 / nseq)
    ops.loss_finalize(acc, counts, out, 1.0, 2.0, 1.0, 0.0, 0.1, 1.0 / nseq, 0.0, True, False)
    leaves = [t.clone().requires_grad_(True) for t in (al, cl, vl)]
    cfg.use_vae = False
    o = {"command_logits": leaves[1].reshape(n, G, Ld, 7), "args_logits": leaves[0].reshape(n, G, Ld, 11, n_classes),
         "visibility_logits": leaves[2].reshape(n, G, 1, 2), "tgt_commands": c, "tgt_args": a}
    O.CMD_ARGS_MASK = O.CMD_ARGS_MASK.to(DEV)
    try:
        ls = O.loss(o, cfg)
        for key, ten, leaf, dl in (("loss_args", al, leaves[0], dla), ("loss_cmd", cl, leaves[1], dlc),
                                   ("loss_visibility", vl, leaves[2], dlv)):
            g, = torch.autograd.grad(ls[key], leaf, retain_graph=True)
            assert _rel(dl.float(), g) < 1e-4, key
    finally:
        O.CMD_ARGS_MASK = O.CMD_ARGS_MASK.cpu()
    assert abs(out[0].item() - ls["loss"].item()) < 1e-5 * ls["loss"].item()
    assert abs(out[1].item() - ls["loss_cmd"].item()) < 1e-5 and abs(out[2].item() - ls["loss_args"].item()) < 1e-5
    assert abs(out[3].item() - ls["loss_visibility"].item()) < 1e-5
    assert dla.t[:, :, nw:].abs().max().item() == 0  # K padding of the head dgrad operand stays zero


def test_vae_and_kl():
    ops = _ops()
    n, dz = 64, 256
    mu, ls, eps, dz_ = _rand(n, dz, seed=1), _rand(n, dz, seed=2, scale=0.3), _rand(n, dz, seed=3), _rand(n, dz, seed=4)
    z = torch.empty(n, dz, device=DEV)
    ops.vae_fwd(mu, ls, eps, z, n * dz)
    m, l = mu.clone().requires_grad_(True), ls.clone().requires_grad_(True)
    zr = m + torch.exp(l / 2) * eps
    assert _rel(z, zr.detach()) < 1e-6
    kl = (-0.5 * torch.mean(1 + l - m.pow(2) - torch.exp(l))).clamp(min=0.1)
    ((zr * dz_).sum() + 3.0 * kl).backward()
    acc, out = torch.zeros(8, device=DEV), torch.zeros(8, device=DEV)
    ops.kl_sum(mu, ls, acc, n * dz)
    counts = torch.ones(2, device=DEV)
    ops.loss_finalize(acc, counts, out, 0.0, 0.0, 0.0, 1.0, 0.1, 0.0, 1.0 / (n * dz), False, True)
    assert abs(out[4].item() - kl.item()) < 1e-5
    dmu, dls = torch.empty(n, dz, device=DEV), torch.empty(n, dz, device=DEV)
    coef = torch.tensor([3.0], device=DEV)
    ops.vae_bwd(mu, ls, eps, dz_, coef, out, 1.0 / (n * dz), dmu, dls, n * dz)
    assert _rel(dmu, m.grad) < 1e-5 and _rel(dls, l.grad) < 1e-5


def test_cast_transpose_and_labels():
    ops = _ops()
    R, Cc = 258, 300
    x = _rand(R, Cc, seed=1)
    a, at = ops.Act(R, Cc, 2, DEV, ld=304), ops.Act(Cc, R, 2, DEV, ld=264)
    ops.cast_act(x, R, Cc, out=a, outT=at)
    assert _rel(a.float(), x) < 1e-5 and _rel(at.float(), x.t()) < 1e-5
    assert a.t[:, :, Cc:].abs().max().item() == 0 and at.t[:, :, R:].abs().max().item() == 0
    table = _rand(52, 64, seed=2)
    idx = torch.randint(0, 52, (40,), generator=torch.Generator().manual_seed(1)).to(DEV)
    g = ops.Act(40, 64, 2, DEV)
    ops.gather_rows(table, idx, 40, 64, g)
    assert _rel(g.float(), table[idx]) < 1e-5
    dt = torch.zeros(52, 64, device=DEV)
    gr = _rand(40, 64, seed=3)
    ops.scatter_rows(gr, idx, 40, 64, dt)
    assert _rel(dt, torch.zeros(52, 64, device=DEV).index_add_(0, idx, gr)) < 1e-5


def test_fused_adamw_matches_torch():
    """SURVEY.md 8f rank 2: multi-tensor AdamW + global-norm clipping vs torch.optim.AdamW + clip_grad_norm_."""
    from deepsvg_b200 import FusedAdamW
    shapes = [(257, 64), (256,), (768, 256), (7, 256), (2827, 256), (1,)]
    ref = [torch.nn.Parameter(_rand(*s, seed=i)) for i, s in enumerate(shapes)]
    mine = [torch.nn.Parameter(p.detach().clone()) for p in ref]
    o_ref = torch.optim.AdamW(ref, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    o_mine = FusedAdamW(mine, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
    for step in range(4):
        for i, (a, b) in enumerate(zip(ref, mine)):
            g = _rand(*a.shape, seed=100 * step + i, scale=0.3 if step % 2 else 3.0)
            a.grad, b.grad = g.clone(), g.clone()
        torch.nn.utils.clip_grad_norm_(ref, 1.0)
        o_ref.step()
        o_mine.step()
        for a, b in zip(ref, mine):
            assert _rel(b.detach(), a.detach()) < 2e-6


# ------------------------------------------------------------------------------------------------ causal attention
ATTN_CAUSAL_CASES = (
    [pytest.param(p, L, H, hd, k, id="%d-%d-%d-%d" % (p, L, H, hd)) for p, L, H, hd, k in [
        (2, 31, 4, 32, _attn("x3")), (1, 31, 4, 32, _attn("mma")), (1, 32, 8, 32, _attn("mma")),
        (1, 51, 8, 32, _attn("gmma", 32, 4)), (1, 66, 4, 64, _attn("gmma", 64, 5)), (2, 51, 4, 32, _attn("gx3", 32, 4)),
        # the general kernels at the other tile counts
        (1, 48, 4, 32, _attn("gmma", 32, 3)), (1, 65, 4, 32, _attn("gmma", 32, 5)), (1, 16, 4, 64, _attn("gmma", 64, 1)),
        (1, 17, 4, 64, _attn("gmma", 64, 2)), (1, 33, 4, 64, _attn("gmma", 64, 3)), (1, 64, 4, 64, _attn("gmma", 64, 4)),
        (2, 33, 4, 32, _attn("gx3", 32, 3)), (2, 80, 4, 32, _attn("gx3", 32, 5)), (2, 16, 4, 64, _attn("gx3", 64, 1)),
        (2, 32, 4, 64, _attn("gx3", 64, 2)), (2, 48, 4, 64, _attn("gx3", 64, 3)), (2, 49, 4, 64, _attn("gx3", 64, 4)),
        (2, 65, 4, 64, _attn("gx3", 64, 5)),
        # fp32 SIMT: head_dim 16, and every head_dim above 80 positions
        (1, 33, 8, 16, _attn("simt", 16)), (2, 33, 8, 16, _attn("simt", 16)), (2, ATTN_MAX_L[16], 8, 16, _attn("simt", 16)),
        (1, 81, 4, 32, _attn("simt", 32)), (2, 81, 4, 32, _attn("simt", 32)),
        (1, ATTN_MAX_L[64], 2, 64, _attn("simt", 64)), (2, 81, 2, 64, _attn("simt", 64))]]
)


@pytest.mark.parametrize("planes,L,H,hd,kernels", ATTN_CAUSAL_CASES)
def test_attention_causal_with_key_padding(planes, L, H, hd, kernels):
    """attn_mask = square_subsequent_mask plus key_padding_mask (the autoregressive decoder, model.py:264-269;
    functional.py:229-240) on every kernel family: the 32 x 32 mma / x3 kernels (head_dim 32, L <= 32), the general
    gmma / gx3 kernels (head_dim 32 / 64, L <= 80) and fp32 SIMT (head_dim 16, L > 80), one and two planes each."""
    ops = _ops()
    nseq, d = 29, H * hd
    M = nseq * L
    qa = ops.act_from_float(_rand(M, 3 * d, seed=1, scale=0.7), planes)
    qv = qa.float().double().requires_grad_(True)
    lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(3))
    vmask = (torch.arange(L)[None, :] < lens[:, None]).to(DEV)
    valid = vmask.to(torch.uint8).reshape(-1).contiguous()
    out = ops.Act(M, d, planes, DEV)
    expect_kernels(kernels[0], lambda: ops.attn_fwd(qa, valid, out, nseq, L, H, hd, (0.0, 0, 0), causal=True))
    q, k, v = (t.reshape(nseq, L, H, hd).transpose(1, 2) for t in qv.split(d, dim=-1))
    s = q @ k.transpose(-1, -2)
    s = s.masked_fill(torch.triu(torch.ones(L, L, dtype=torch.bool, device=DEV), 1), float("-inf"))
    s = s.masked_fill(~vmask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(M, d)
    # tensor-core kernels round P and dS to bf16 inside; SIMT keeps them in fp32, leaving the bf16 output rounding only
    tol = 1e-4 if planes == 2 else (5e-3 if kernels[0].startswith("attn_fwd_kernel") else 1.5e-2)
    assert _rel(out.float(), ref.detach()) < tol
    da = ops.act_from_float(_rand(M, d, seed=5), planes)
    ref.backward(da.float().double())
    dqkv = ops.Act(M, 3 * d, planes, DEV)
    expect_kernels(kernels[1], lambda: ops.attn_bwd(qa, valid, da, dqkv, nseq, L, H, hd, 0.5, (0.0, 0, 0), causal=True))
    g = qv.grad.clone()
    g[:, :d] *= 0.5
    for lo, hi, nm in ((0, d, "dq"), (d, 2 * d, "dk"), (2 * d, 3 * d, "dv")):
        e = (dqkv.float()[:, lo:hi] - g[:, lo:hi]).norm() / g[:, lo:hi].norm()
        assert e.item() < tol, (nm, e.item())
