"""The full-width 256-wide linear kernels (linear_kernel<256, 1, m>, m in 1-5 and 8): two consumer warpgroups with
m64n256 wgmma and the epilogue on the accumulator fragments.  Cases the per-role tables of test_kernels_gpu.py do not
reach: row counts at every warpgroup and tile boundary, ragged N and K, grids with fewer tiles than SMs and with several
tiles per CTA, dropout and row vectors on, the fused LayerNorm against linear followed by ln_fwd, and the dropout masks
against the ones cast_act draws."""
import pytest
import torch

from tests.test_kernels_gpu import DEV, _lin, _rand, _rel, expect_kernels

pytestmark = pytest.mark.gpu

P_DROP, SITE, SEED = 0.25, 9, 1234


def _ops():
    from deepsvg_b200 import ops
    return ops


def _keep(ops, M, N):
    """fp64 [M, N] dropout multipliers (0 or 1 / (1 - p)) as cast_act draws them for (SEED, SITE), index row N + col."""
    ones = torch.ones(M, N, device=DEV)
    out = ops.Act(M, N, 1, DEV)
    ops.cast_act(ones, M, N, out=out, drop=(P_DROP, SITE, SEED))
    keep = out.float() != 0
    thr16 = int(P_DROP * 65536.0 + 0.5)
    return keep.double() / (1.0 - thr16 / 65536.0)


# M mod 128 in {1, 63, 64, 65, 127} (above 16384 rows the 256-wide kernel runs); 16385 x 256 is 129 tiles, fewer than the
# SMs; 70000 x 768 is several tiles per CTA
SHAPES = [(16384 + r, 256, 256) for r in (1, 63, 64, 65, 127)] + [
    (16447, 384, 520), (16449, 520, 512), (20000, 512, 768), (70000 + 65, 768, 256)]
MODES = [1, 2, 3, 4, 5]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K", SHAPES, ids=["%d-%d-%d" % s for s in SHAPES])
def test_wide_modes(mode, M, N, K):
    ops = _ops()
    rpg = 25
    X, W = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5)
    b, res, rv = _rand(N, seed=3), _rand(M, N, seed=4), _rand((M + rpg - 1) // rpg, N, seed=5)
    msk = torch.relu(_rand(M, N, seed=6))
    xa, wa, ma = ops.act_from_float(X, 1), ops.act_from_float(W, 1), ops.act_from_float(msk, 1)
    acc = xa.float().double() @ wa.float().double().t()
    drop = (P_DROP, SITE, SEED)
    of, oa = torch.zeros(M, N, device=DEV), ops.Act(M, N, 1, DEV)
    if mode == 1:
        run = lambda: ops.linear(xa, wa, M, N, K, out_act=oa)
        ref = acc
    elif mode == 2:
        sc = 128
        run = lambda: ops.linear(xa, wa, M, N, K, bias=b, scale_cols=sc, scale=0.125, out_act=oa)
        ref = acc + b.double()
        ref[:, :sc] *= 0.125
    elif mode == 3:
        run = lambda: ops.linear(xa, wa, M, N, K, bias=b, relu=True, drop=drop, out_act=oa)
        ref = torch.relu(acc + b.double()) * _keep(ops, M, N)
    elif mode == 4:
        run = lambda: ops.linear(xa, wa, M, N, K, bias=b, drop=drop, rowvec=rv, rows_per_group=rpg, residual=res,
                                 out_f32=of)
        ref = (acc + b.double()) * _keep(ops, M, N) + rv.double().repeat_interleave(rpg, 0)[:M] + res.double()
    else:
        run = lambda: ops.linear(xa, wa, M, N, K, mask=ma, mask_scale=1.5, out_act=oa)
        ref = acc * (ma.float() != 0).double() * 1.5
    if (M, N, K) == SHAPES[0]:
        expect_kernels(_lin(256, 1, mode), run)
    else:
        run()
    torch.cuda.synchronize()
    if mode == 4:
        assert _rel(of, ref) < 2e-5
    else:
        assert _rel(oa.float(), ref) < 6e-3


@pytest.mark.parametrize("M,K", [(16385, 256), (16447, 512), (16448, 520), (16511, 256), (70000 + 65, 512)])
def test_wide_fused_layernorm(M, K):
    """Mode 8 against mode 4 followed by ln_fwd on the same inputs, and against an fp64 restatement."""
    ops = _ops()
    N, rpg = 256, 31
    X, W = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5)
    b, res, rv = _rand(N, seed=3), _rand(M, N, seed=4), _rand((M + rpg - 1) // rpg, N, seed=5)
    gamma, beta = 1.0 + 0.1 * _rand(N, seed=7), 0.1 * _rand(N, seed=8)
    xa, wa = ops.act_from_float(X, 1), ops.act_from_float(W, 1)
    drop = (P_DROP, SITE, SEED)
    kw = dict(bias=b, drop=drop, rowvec=rv, rows_per_group=rpg, residual=res)
    x1, y = torch.empty(M, N, device=DEV), ops.Act(M, N, 1, DEV)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    fused = lambda: ops.linear(xa, wa, M, N, K, out_f32=x1, ln=(gamma, beta, y, mean, rstd), **kw)
    x1s, ys = torch.empty(M, N, device=DEV), ops.Act(M, N, 1, DEV)
    means, rstds = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    split = lambda: ops.linear(xa, wa, M, N, K, out_f32=x1s, **kw)
    # which kernels these launch is asserted by test_kernels_gpu.py (LN_FUSED_CASES and the mode-4 lean cases)
    fused()
    split()
    ops.ln_fwd(x1s, gamma, beta, ys, means, rstds, M, N)
    torch.cuda.synchronize()
    assert torch.equal(x1, x1s)
    # the row means sit near zero: their summation-order differences are measured against the row's spread
    assert ((mean - means).abs() <= 1e-6 / rstds).all()
    assert ((rstd - rstds).abs() <= 1e-6 * rstds.abs()).all()
    # ln_fwd normalises as (x - mean) rstd with a two-pass variance, the fused kernel as x rstd - mean rstd with
    # E[x^2] - mean^2: within one bf16 ulp of the output (<= |y| 2^-7) plus fp32 rounding of the terms that cancel
    yf, ysf = y.float(), ys.float()
    terms = gamma.abs() * (x1s.abs() * rstds[:, None] + (means * rstds).abs()[:, None])
    assert ((yf - ysf).abs() <= ysf.abs() * 2.0 ** -7 + 1e-5 * terms).all()
    ref_x1 = ((xa.float().double() @ wa.float().double().t()) + b.double()) * _keep(ops, M, N) \
        + rv.double().repeat_interleave(rpg, 0)[:M] + res.double()
    assert _rel(x1, ref_x1) < 2e-5
