"""The persistent single-plane weight-gradient kernel (outer_kernel<BQ, 1>) at the shapes of the train steps and at the edges
of its work decomposition, against a float64 restatement on the same bf16 operands (rel < 2e-5 for the gradient and its
bias column sums, as test_outer_matches_fp32).  Each case asserts a single launch; tests/test_gemm_wgrad_gpu.py asserts
which kernel the two entry points launch at path-level row counts.

A work item is (output tile, chunk of at most 48 row blocks of 64 rows); the launch picks the chunk count that balances
the items over the SMs, so most cases leave some CTAs with one item fewer than the others."""
import pytest
import torch

from tests.test_kernels_gpu import DEV, _rand, _rel

pytestmark = pytest.mark.gpu


def _ops():
    from deepsvg_b200 import ops
    return ops


def _act(ops, M, P, seed, ld=None):
    return ops.act_from_float(_rand(M, P, seed=seed), 1, ld=ld if ld is not None else (P + 7) // 8 * 8)


def _one_launch(fn):
    """fn() must issue exactly one launch of the library (tests/test_gemm_wgrad_gpu.py asserts which kernel)."""
    from deepsvg_b200 import _lib
    n0 = _lib.launch_count()
    fn()
    assert _lib.launch_count() - n0 == 1


def _ref(aa, ba):
    a = aa.float().double()
    return a.t() @ ba.float().double(), a.sum(0)


def _block(ops, M, d, ff):
    probs = []
    for i, (P, Q) in enumerate([(3 * d, d), (d, d), (ff, d), (d, ff)]):
        aa, ba = _act(ops, M, P, 10 + i), _act(ops, M, Q, 20 + i)
        probs.append((aa, ba, P, Q, torch.full((P, Q), 0.25, device=DEV), torch.full((P,), -0.5, device=DEV)))
    return probs


# (M, P, Q, lda): the args head (2827 outputs, rows padded to 2832), the command head (7 outputs), and single problems
# whose row count is not a multiple of 64, just below / at / above one 48-block chunk, or a few rows past a chunk boundary
@pytest.mark.parametrize("M,P,Q,lda", [(126976, 2827, 256, 2832), (126976, 7, 256, 8), (100003, 768, 256, 768),
                                       (3071, 768, 256, 768), (3072, 512, 256, 512), (3137, 512, 256, 512),
                                       (98305, 300, 200, 304), (16447, 1000, 250, 1000)])
def test_single_problem_with_device_alpha(M, P, Q, lda):
    ops = _ops()
    aa, ba = _act(ops, M, P, 1, ld=lda), _act(ops, M, Q, 2)
    Cout = torch.ones(P, Q, device=DEV)
    cs = torch.ones(P, device=DEV)
    sc = torch.tensor([2.0], device=DEV)
    _one_launch(lambda: ops.outer(aa, ba, M, P, Q, Cout, alpha=0.5, alpha_dev=sc, colsum=cs))
    rc, rs = _ref(aa, ba)
    assert _rel(Cout, (rc + 1.0).float()) < 2e-5
    assert _rel(cs, (rs + 1.0).float()) < 2e-5


def test_two_launches_accumulate_into_one_bucket():
    """Two gradient sources of one head (the args head has one per loss term) add into the same weight and bias slices
    of a flat fp32 bucket; the weight slice starts at an odd offset, so the reductions take the scalar path."""
    ops = _ops()
    M, P, Q = 126976, 2827, 256
    bucket = torch.zeros(1 + P * Q + P + 64, device=DEV)
    Cout = bucket[1:1 + P * Q].view(P, Q)
    cs = bucket[1 + P * Q:1 + P * Q + P]
    ba = _act(ops, M, Q, 3)
    want_c, want_s = torch.zeros(P, Q, dtype=torch.float64, device=DEV), torch.zeros(P, dtype=torch.float64, device=DEV)
    for seed, scale in ((4, 1.0), (5, 0.25)):
        aa = _act(ops, M, P, seed, ld=2832)
        sc = torch.tensor([scale], device=DEV)
        _one_launch(lambda: ops.outer(aa, ba, M, P, Q, Cout, alpha_dev=sc, colsum=cs))
        rc, rs = _ref(aa, ba)
        want_c += scale * rc
        want_s += scale * rs
    assert _rel(Cout, want_c.float()) < 2e-5
    assert _rel(cs, want_s.float()) < 2e-5
    assert bucket[0] == 0 and torch.count_nonzero(bucket[1 + P * Q + P:]) == 0


# (M, d_model, feed-forward): the path-level blocks of `hier` (encoder / decoder row counts) and of `scaled`
@pytest.mark.parametrize("M,d,ff", [(131072, 256, 512), (126976, 256, 512), (270336, 512, 512)])
def test_grouped_block_gradients(M, d, ff):
    """in_proj, out_proj, linear1 and linear2 gradients of one block in one launch, into non-zero buffers."""
    ops = _ops()
    probs = _block(ops, M, d, ff)
    _one_launch(lambda: ops.outer_group(probs, M))
    for aa, ba, P, Q, Cout, cs in probs:
        rc, rs = _ref(aa, ba)
        assert _rel(Cout, (rc + 0.25).float()) < 2e-5, (P, Q)
        assert _rel(cs, (rs - 0.5).float()) < 2e-5, (P, Q)
