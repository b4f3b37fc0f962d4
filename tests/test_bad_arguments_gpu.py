"""-m gpu: the inputs the C ABI rejects before launching, beyond those of test_kernels_gpu.test_bad_arguments_are_reported.  Each call
answers HAWQ_ERR_BAD_ARG and launches nothing: its pre-poisoned outputs and the status word stay as they were."""
import pytest
import torch

from hawq_b200 import ops
from hawq_b200._lib import EPI_RESIDUAL, ERR_BAD_ARG, HawqError, dyadic
from tests.kernel_harness import DEV, make_chan, rand_act, rng
from tests.util import POISON

pytestmark = pytest.mark.gpu

ROWS, C = 16, 64


def poisoned(numel, dtype):
    """a device buffer of `numel` elements whose every byte is POISON"""
    return torch.full((numel * torch.empty(0, dtype=dtype).element_size(),), POISON, dtype=torch.uint8, device=DEV).view(dtype)


def rejected(call, *outs):
    before, status = [o.clone() for o in outs], ops.get_status(0)
    with pytest.raises(HawqError) as err:
        call()
    torch.cuda.synchronize()
    assert err.value.code == ERR_BAD_ARG, err.value
    assert all(torch.equal(o, b) for o, b in zip(outs, before)), err.value
    assert ops.get_status(0) == status, err.value


@pytest.mark.parametrize("bad", [dict(res_kind=2), dict(res_bits=8), dict(y_bits=8), dict(low_bits=2), dict(low_me=(1 << 30, 0)),
                                 dict(y_bits=0, low_bits=0)], ids=["res_kind", "res_bits", "y_bits", "low_bits", "low_e_0", "no_output"])
def test_add_requant_checks_its_epilogue_as_conv2d_does(bad):
    """the RESIDUAL rules of hawq_conv2d: with low_e = 0 the kernel would shift by -1"""
    r = rng(408)
    acc, res = rand_act(r, ROWS * C, 32).to(DEV), rand_act(r, ROWS * C, 32).to(DEV)
    chan = make_chan(r, C, ratio_lo=0.01, ratio_hi=0.9).to(DEV)
    y, low = poisoned(ROWS * C, torch.int32), poisoned(ROWS * C, torch.int8)
    good = dict(relu=1, res_kind=0, res_bits=32, res_me=dyadic(0.6), y_bits=32, low_bits=8, low_me=dyadic(0.002), low_clamp=(-128, 127))
    ep = ops.epilogue(EPI_RESIDUAL, **{**good, **bad})
    rejected(lambda: ops.add_requant(acc, ROWS, C, chan, ep, res, None, y, low), y, low)


@pytest.mark.parametrize("n,hw,c", [(2, 0, C), (0, 49, C), (2, 49, 0)])
def test_avgpool_requant_rejects_empty_shapes(n, hw, c):
    """HW = 0 would divide by zero on the device"""
    stream, pooled = rand_act(rng(409), 2 * 49 * C, 32).to(DEV), poisoned(2 * C, torch.int8)
    rejected(lambda: ops.avgpool_requant(stream, n, hw, c, 32, dyadic(0.004), (-128, 127), pooled), pooled)


@pytest.mark.parametrize("n,hh,ww", [(0, 9, 9), (2, 0, 9), (2, 9, 0)])
def test_maxpool_requant_rejects_empty_shapes(n, hh, ww):
    """H = 0 would still make one output row, which the caller never allocated"""
    x16, y = torch.zeros(2 * 9 * 9 * C, dtype=torch.int16, device=DEV), poisoned(2 * 5 * 5 * C, torch.int32)
    rejected(lambda: ops.maxpool_requant(x16, n, hh, ww, C, 32, y, 0, (0, 1), (0, 0), None), y)


def test_quantize_input_and_requant_reject_an_empty_clamp_range():
    img, q = torch.zeros((2, 3, 4, 4), device=DEV), poisoned(2 * 3 * 4 * 4, torch.int8)
    rejected(lambda: ops.quantize_input(img, 0.02, (5, -5), q), q)
    r = rng(410)
    acc, chan, out = rand_act(r, ROWS * C, 32).to(DEV), make_chan(r, C, ratio_lo=0.01, ratio_hi=0.9).to(DEV), poisoned(ROWS * C, torch.int8)
    rejected(lambda: ops.requant(acc, ROWS, C, 32, chan, 1, 0, 8, (10, -10), out), out)
