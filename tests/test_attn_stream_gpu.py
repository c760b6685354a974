"""The 32 x 32 tensor-core attention (attn_mma_fwd_kernel / attn_mma_bwd_kernel: single-plane bf16, head_dim 32, L <= 32)
streams whole sequences through a ring of shared-memory stages.  These cases pin what that staging must get right: every
L and head count against an fp64 restatement, sequence counts around the CTA x stage walk, zero padding of the rows >= L
(the neighbouring sequence's rows must never reach a sequence's outputs or gradients), and the dropout mask shared by
forward and backward."""
import pytest
import torch

from tests.test_kernels_gpu import DEV, expect_kernels

pytestmark = pytest.mark.gpu

HD = 32
KERNELS = ("attn_mma_fwd_kernel", "attn_mma_bwd_kernel")


def _ops():
    from deepsvg_b200 import ops
    return ops


def _inputs(nseq, L, H, seed=0, scale=0.7):
    g = torch.Generator().manual_seed(seed)
    d = H * HD
    qkv = (torch.randn(nseq * L, 3 * d, generator=g) * scale).to(DEV)
    do = torch.randn(nseq * L, d, generator=g).to(DEV)
    return qkv, do


def _run(qkv, do, nseq, L, H, valid=None, causal=False, drop=(0.0, 0, 0), check_kernels=False):
    ops = _ops()
    d, M = H * HD, nseq * L
    qa, da = ops.act_from_float(qkv, 1), ops.act_from_float(do, 1)
    out = ops.Act(M, d, 1, DEV, zero=True)
    dqkv = ops.Act(M, 3 * d, 1, DEV, zero=True)
    fwd = lambda: ops.attn_fwd(qa, valid, out, nseq, L, H, HD, drop, causal=causal)   # noqa: E731
    bwd = lambda: ops.attn_bwd(qa, valid, da, dqkv, nseq, L, H, HD, 0.5, drop, causal=causal)   # noqa: E731
    if check_kernels:
        expect_kernels(KERNELS[0], fwd)
        expect_kernels(KERNELS[1], bwd)
    else:
        fwd()
        bwd()
    torch.cuda.synchronize()
    return qa, da, out, dqkv


def _reference(qa, da, nseq, L, H, vmask=None, causal=False):
    """fp64 attention of the bf16 operands; returns (out [M, d], dqkv [M, 3d] with dq scaled by 0.5)."""
    d = H * HD
    qv = qa.float().double().requires_grad_(True)
    q, k, v = (t.reshape(nseq, L, H, HD).transpose(1, 2) for t in qv.split(d, dim=-1))
    s = q @ k.transpose(-1, -2)
    if vmask is not None:
        s = s.masked_fill(~vmask[:, None, None, :], float("-inf"))
    if causal:
        s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=DEV).triu(1), float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(nseq * L, d)
    ref.backward(da.float().double())
    g = qv.grad.clone()
    g[:, :d] *= 0.5
    return ref.detach(), g


def _check(out, dqkv, ref, g, d, rows=None):
    o, dq = out.float().double(), dqkv.float().double()
    if rows is not None:
        o, dq, ref, g = o[rows], dq[rows], ref[rows], g[rows]
    assert torch.isfinite(o).all() and torch.isfinite(dq).all()
    e = (o - ref).norm() / ref.norm()
    assert e.item() < 1.5e-2, ("o", e.item())
    for lo, hi, nm in ((0, d, "dq"), (d, 2 * d, "dk"), (2 * d, 3 * d, "dv")):
        err, norm = (dq[:, lo:hi] - g[:, lo:hi]).norm().item(), g[:, lo:hi].norm().item()
        if norm == 0.0:   # L = 1: softmax over one key is constant, so dq = dk = 0 exactly
            assert err == 0.0, (nm, err)
        else:
            assert err / norm < 1.5e-2, (nm, err / norm)


def _mask(nseq, L, seed=3):
    lens = torch.randint(1, L + 1, (nseq,), generator=torch.Generator().manual_seed(seed))
    vmask = (torch.arange(L)[None, :] < lens[:, None]).to(DEV)
    return vmask, vmask.to(torch.uint8).reshape(-1).contiguous()


@pytest.mark.parametrize("mode", ["plain", "masked", "causal"])
@pytest.mark.parametrize("H", [4, 8, 16])
@pytest.mark.parametrize("L", [1, 2, 8, 17, 31, 32])
def test_stream_matches_fp64(L, H, mode):
    """Every head count the tests use (one head per consumer warp at H <= 8, two per warp at H = 16) at every kind of L:
    one row, a partial 16-row tile, the group-level 8, one past a tile, one short of the full tile, the full tile."""
    nseq = 37
    qkv, do = _inputs(nseq, L, H)
    vmask, valid = _mask(nseq, L) if mode == "masked" else (None, None)
    qa, da, out, dqkv = _run(qkv, do, nseq, L, H, valid, causal=mode == "causal")
    ref, g = _reference(qa, da, nseq, L, H, vmask, causal=mode == "causal")
    _check(out, dqkv, ref, g, H * HD)


@pytest.mark.parametrize("H", [4, 8, 16])
def test_stream_kernels_selected(H):
    """One plane, head_dim 32, L <= 32 runs attn_mma_fwd_kernel / attn_mma_bwd_kernel and no other attention kernel, with
    one head per consumer warp (H <= 8) and with two (H = 16)."""
    qkv, do = _inputs(40, 17, H)
    _run(qkv, do, 40, 17, H, drop=(0.1, 5, 4321), check_kernels=True)


@pytest.mark.parametrize("L", [8, 31, 32])
@pytest.mark.parametrize("nseq", [1, 2, 529, 4096])
def test_stream_sequence_counts(nseq, L):
    """nseq = 1 and 2 launch fewer CTAs than SMs; 529 is one past a multiple of the CTA count times the ring depth of both
    kernels on 132 SMs (forward 2 x 132 CTAs, backward 132, two stages each), so some CTAs walk one more sequence than
    others and wrap the ring; 4096 is the path-level shape.  The last sequence always ends at the end of the tensor."""
    H = 8
    qkv, do = _inputs(nseq, L, H, seed=nseq)
    vmask, valid = _mask(nseq, L, seed=nseq)
    qa, da, out, dqkv = _run(qkv, do, nseq, L, H, valid)
    ref, g = _reference(qa, da, nseq, L, H, vmask)
    _check(out, dqkv, ref, g, H * HD)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("L", [1, 8, 17, 31])
def test_stream_padding_rows_never_leak(L, causal):
    """Every odd sequence is filled with +-1e4 (q, k, v and dO): were any row >= L of a 32-row tile taken from the
    next sequence instead of zeros, the even sequences' outputs and gradients would be off by orders of magnitude."""
    nseq, H = 300, 8
    qkv, do = _inputs(nseq, L, H, seed=7)
    big = torch.where(torch.rand(qkv.shape, generator=torch.Generator().manual_seed(8)) < 0.5, -1e4, 1e4).to(DEV)
    odd = (torch.arange(nseq * L, device=DEV) // L) % 2 == 1
    qkv[odd] = big[odd]
    do[odd] = big[odd, :do.shape[1]]
    vmask, valid = _mask(nseq, L)
    qa, da, out, dqkv = _run(qkv, do, nseq, L, H, valid, causal=causal)
    even = ~odd
    ref, g = _reference(qa, da, nseq, L, H, vmask, causal=causal)
    _check(out, dqkv, ref, g, H * HD, rows=even)


@pytest.mark.parametrize("L,H,nseq", [(32, 8, 4096), (8, 8, 512), (17, 4, 61), (31, 16, 45)])
def test_stream_dropout_mask_shared_and_reproducible(L, H, nseq):
    """With dropout, out is linear in v for the fixed probabilities and mask: out(v) . g == v . dv(g) holds only if the
    backward draws the forward's mask.  Two runs on the same inputs and seed are bit-identical."""
    d = H * HD
    qkv, do = _inputs(nseq, L, H, seed=11, scale=0.5)
    drop = (0.1, 5, 4321)
    qa, da, o1, dqkv1 = _run(qkv, do, nseq, L, H, drop=drop)
    _, _, o2, dqkv2 = _run(qkv, do, nseq, L, H, drop=drop)
    assert torch.equal(o1.t, o2.t) and torch.equal(dqkv1.t, dqkv2.t)
    _, _, o0, _ = _run(qkv, do, nseq, L, H)
    assert not torch.equal(o1.t, o0.t)
    lhs = (o1.float().double() * da.float().double()).sum().item()
    rhs = (qa.float()[:, 2 * d:].double() * dqkv1.float()[:, 2 * d:].double()).sum().item()
    assert abs(lhs - rhs) < 2e-2 * abs(lhs)
