"""-m gpu: the convolution launches with more CTAs than fit on the GPU at once (two per SM), so that row tiles of the 1-D,
row-tile-major grid follow one another across waves: the ResNet-50 resize-unit tail (dual kernel, BN = 64) and a stage-2
bottleneck tail with a ragged last row tile (uint16 residual prefetched during the GEMM).  Same checks as the geometries of
test_kernels_gpu.py: bit-exact against the ABI model."""
import pytest

from tests.test_kernels_gpu import test_conv1x1_requant_and_residual as check_conv1x1
from tests.test_kernels_gpu import test_conv_dual_stationary_weights as check_conv_dual

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(12, 28, 28, 128, 512)])   # 74 row tiles (last one ragged) x 4 channel blocks = 296 CTAs
def test_conv1x1_many_waves(geom, a_bits):
    check_conv1x1(geom, a_bits)


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(8, 56, 56, 64, 64, 256, 1)])   # ResNet-50 stage 1: 196 row tiles x 4 channel blocks = 784 CTAs
def test_conv_dual_many_waves(geom, a_bits, flag):
    check_conv_dual(geom, a_bits, flag)
