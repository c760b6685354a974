"""Which kernel the weight-gradient entry points launch at path-level row counts: a block's grouped gradients and the args
head gradient both run the persistent single-plane kernel.  The numerics at the train steps' shapes and at the edges of
the work decomposition are in tests/test_wgrad_persistent_gpu.py."""
import pytest
import torch

from tests.test_kernels_gpu import DEV, _rel, expect_kernels
from tests.test_wgrad_persistent_gpu import _act, _block, _ops, _ref

pytestmark = pytest.mark.gpu

KERNEL = "outer_kernel<256, 1>"


@pytest.mark.parametrize("grouped", [True, False])
def test_kernel_selection(grouped):
    """A block's grouped gradients and a single-plane head gradient at path-level row counts run the persistent kernel."""
    ops = _ops()
    M = 16448
    if grouped:
        probs = _block(ops, M, 256, 512)
        expect_kernels(KERNEL, lambda: ops.outer_group(probs, M))
    else:
        aa, ba = _act(ops, M, 2827, 1, ld=2832), _act(ops, M, 256, 2)
        Cout, cs, sc = torch.zeros(2827, 256, device=DEV), torch.zeros(2827, device=DEV), torch.ones(1, device=DEV)
        expect_kernels(KERNEL, lambda: ops.outer(aa, ba, M, 2827, 256, Cout, alpha_dev=sc, colsum=cs))
        rc, rs = _ref(aa, ba)
        assert _rel(Cout, rc.float()) < 2e-5 and _rel(cs, rs.float()) < 2e-5
