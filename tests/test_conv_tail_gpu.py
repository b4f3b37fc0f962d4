"""-m gpu: the persistent tail kernel (conv_tail.cuh) that runs the 1x1 uint16-stream RESIDUAL launches (bottleneck tails) and every
resize unit.  Each CTA owns one channel block and walks row tiles gridDim / (Cout / 64) apart; the loads of its next tile are in
flight while it finishes the current one.  The geometries below give every CTA at least three row tiles with a ragged last one, or
more CTAs than tiles; the checks are those of test_kernels_gpu.py: bit-exact against the ABI model, in guarded allocations."""
import numpy as np
import pytest
import torch

from hawq_b200 import ops
from hawq_b200._lib import EPI_RESIDUAL, dyadic
from tests import abi_model as am
from tests.kernel_harness import (DEV, RATIO_ONE, check_conv1x1_requant_and_residual, check_conv_dual_stationary_weights,
                                  check_conv_epilogue_boundaries, check_conv_residual, images_for_three_tiles, row_tile_stride, run_both)

pytestmark = pytest.mark.gpu

# ResNet-50 stages: (H = W of the output, bottleneck width, Cout, identity stride of the resize unit)
STAGES = {1: (56, 64, 256, 1), 2: (28, 128, 512, 2), 3: (14, 256, 1024, 2), 4: (7, 512, 2048, 2)}


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("stage", sorted(STAGES))
def test_tail_resnet50_shapes(stage, a_bits):
    """the bottleneck tail of each stage (flags 1 and 2, 8-bit, 4-bit and no low-bit copy), and REQUANT on the same geometry"""
    hw, mid, cout, _ = STAGES[stage]
    check_conv1x1_requant_and_residual((images_for_three_tiles(hw * hw, cout), hw, hw, mid, cout), a_bits)


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("stage", sorted(STAGES))
def test_resize_unit_resnet50_shapes(stage, a_bits, flag):
    hw, mid, cout, s2 = STAGES[stage]
    check_conv_dual_stationary_weights((images_for_three_tiles(hw * hw, cout), hw, hw, mid, 64 if stage == 1 else cout // 2, cout, s2), a_bits, flag)


@pytest.mark.parametrize("a_bits", [8, 4])
def test_tail_more_ctas_than_tiles(a_bits):
    """M = 81: one ragged row tile per channel block, most CTAs of the grid get none"""
    check_conv1x1_requant_and_residual((1, 9, 9, 64, 256), a_bits)


@pytest.mark.parametrize("flags", [0, 1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
def test_tail_mixed_policies_many_tiles(a_bits, flags):
    """channel blocks of one launch on different requantisation policies (FP64, FP64 clamped and checked, Exact), with every CTA
    walking several row tiles"""
    check_conv_epilogue_boundaries((images_for_three_tiles(28 * 28, 512), 28, 28, 128, 512, 1, 1, 1, 0), a_bits, flags)


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("stage", [1, 3])
def test_tail_residual_epilogues_many_tiles(stage, a_bits, tc):
    """test_conv_residual's epilogues on a tail geometry with at least three row tiles per CTA: its uint16-stream cases run on the
    tail kernel, the int32 and res_kind 1 cases on conv_igemm"""
    hw, mid, cout, _ = STAGES[stage]
    check_conv_residual((images_for_three_tiles(hw * hw, cout), hw, hw, mid, cout, 1, 1, 1, 0), a_bits, tc)


@pytest.mark.parametrize("a_bits", [8, 4])
def test_flags_from_a_third_tile_only(a_bits):
    """Every CTA walks three row tiles; the last one is ragged.  As in test_rows_past_m_raise_no_flag, acc = -bias on every real
    row and the ratio is 2^17, so a zero-filled row past M would raise both flags if it were counted.  One real row in CTA 0's
    third tile differs: with one input value one step up, its stream value exceeds 65535 (HAWQ_FLAG_RESIDUAL_OVERFLOW, every
    output still exact); with the whole pixel zero, its term leaves int32 (HAWQ_FLAG_REQUANT_OVERFLOW under a promise).  Without
    that row no flag is raised."""
    cin, cout = 64, 64
    step = row_tile_stride(cout)
    m = (3 * step - 1) * 128 + 77
    numel = m * cout
    hot = 2 * step * 128 + 5                      # a row of CTA 0's third row tile
    if a_bits == 8:
        fill, up, dt, pix_bytes, wv, acc = -128, -127, torch.int8, cin, 127, cin * -128 * 127
    else:
        fill, up, dt, pix_bytes, wv, acc = 0xFF, 0xFE, torch.uint8, cin // 2, -127, cin * 15 * -127
    wt = torch.full((cout, 1, 1, cin), wv, dtype=torch.int8)
    chan = ops.make_chan([-acc] * cout, [2 ** 31] * cout, [14] * cout)
    d = ops.conv_desc(1, 1, m, cin, cout, 1, 1, 1, 0, a_bits)
    res = torch.from_numpy(np.random.RandomState(a_bits).randint(0, 65536, size=numel).astype(np.uint16).view(np.int16))
    for flags in (1, 2):
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=16, res_me=RATIO_ONE, y_bits=16, low_bits=8, low_me=dyadic(0.003),
                          low_clamp=(-128, 127), flags=flags)
        for hot_value, flag in [(None, 0), (up, 1)]:
            x = torch.full((m * pix_bytes,), fill, dtype=dt)
            if hot_value is not None:
                x[hot * pix_bytes] = hot_value
            cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, out=torch.zeros(numel, dtype=torch.int16),
                                             out_low=torch.zeros(numel, dtype=torch.int8)), ["out", "out_low"])
            assert am.status["flags"] == flag, (a_bits, flags, hot_value, am.status["flags"])
            for a, b in zip(cs, gs):
                assert torch.equal(a, b), (a_bits, flags, hot_value)
        x = torch.full((m * pix_bytes,), fill, dtype=dt)
        x[hot * pix_bytes:(hot + 1) * pix_bytes] = 0
        ops.reset_status(0)
        ops.conv2d(x.to(DEV), d, ep, wt.to(DEV), chan.to(DEV), res=res.to(DEV), out=torch.zeros(numel, dtype=torch.int16, device=DEV),
                   out_low=torch.zeros(numel, dtype=torch.int8, device=DEV))
        assert ops.get_status(0) & 4, (a_bits, flags)
        ops.reset_status(0)
