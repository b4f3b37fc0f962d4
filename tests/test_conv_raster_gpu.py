"""-m gpu: the convolution launches with more CTAs than fit on the GPU at once (two per SM), so that row tiles of the 1-D,
row-tile-major grid follow one another across waves: the ResNet-50 resize-unit tail (dual kernel, BN = 64), a stage-2
bottleneck tail with a ragged last row tile (uint16 residual prefetched during the GEMM), and every epilogue family of
hawq_conv2d on a 3x3 and a strided geometry.  Same checks as the geometries of test_kernels_gpu.py: bit-exact against the ABI
model, in guarded allocations."""
import pytest

from tests.kernel_harness import (check_conv1x1_requant_and_residual, check_conv_dual_stationary_weights, check_conv_raw_and_dequant_geoms,
                                  check_conv_requant, check_conv_residual, sm_count)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(12, 28, 28, 128, 512)])   # 74 row tiles (last one ragged) x 4 channel blocks = 296 CTAs
def test_conv1x1_many_waves(geom, a_bits):
    check_conv1x1_requant_and_residual(geom, a_bits)


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(8, 56, 56, 64, 64, 256, 1)])   # ResNet-50 stage 1: 196 row tiles x 4 channel blocks = 784 CTAs
def test_conv_dual_many_waves(geom, a_bits, flag):
    check_conv_dual_stationary_weights(geom, a_bits, flag)


# per-image shape (H, W, Cin, kh, kw, stride, pad), each with 7 x 7 outputs per image; Cin stays small to bound the model's share
WAVE_SHAPES = {"3x3": (7, 7, 64, 3, 3, 1, 1), "1x1s2": (13, 13, 128, 1, 1, 2, 0)}


def many_wave_geom(shape, cout):
    """(N, H, W, Cin, Cout, kh, kw, stride, pad) with the smallest N whose grid has more CTAs than two per SM and a ragged last
    row tile.  Cout 192 runs BN = 64 (three channel blocks), Cout 256 BN = 128 (two)."""
    h, w, cin, kh, kw, s, p = WAVE_SHAPES[shape]
    per_image = 49
    nblk = cout // (128 if cout % 128 == 0 else 64)
    n = 1
    while -(-n * per_image // 128) * nblk <= 2 * sm_count() or n * per_image % 128 == 0:
        n += 1
    assert -(-n * per_image // 128) * nblk > 2 * sm_count() and n * per_image % 128
    return n, h, w, cin, cout, kh, kw, s, p


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("cout", [192, 256])
@pytest.mark.parametrize("shape", list(WAVE_SHAPES))
def test_conv_requant_many_waves(shape, cout, a_bits):
    """REQUANT to 8, 4, 16 and 32 bits (16 and 32 are stored directly from the accumulators)"""
    check_conv_requant(many_wave_geom(shape, cout), a_bits, 1)


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("cout", [192, 256])
@pytest.mark.parametrize("shape", list(WAVE_SHAPES))
def test_conv_residual_many_waves(shape, cout, a_bits):
    """RESIDUAL: int32 and uint16 operands (res_kind 0), per-channel int32 operands (res_kind 1), y_bits 32, 16 and 0"""
    check_conv_residual(many_wave_geom(shape, cout), a_bits, 1)


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("cout", [192, 256])
@pytest.mark.parametrize("shape", list(WAVE_SHAPES))
def test_conv_raw_and_dequant_many_waves(shape, cout, a_bits):
    """RAW_I32, and DEQUANT_F32 with an odd cout_store"""
    check_conv_raw_and_dequant_geoms(many_wave_geom(shape, cout), a_bits)
