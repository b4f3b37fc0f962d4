"""-m gpu: the stem, pooling, input-quantisation, dequantisation, nibble-packing and classifier kernels at their integer and launch
limits, against the numpy ABI model (tests/abi_model.py -> oracle/int_ref.py) on the same seeded buffers: every output bit-exact and
the status word equal to the model's.

Launch limits: the two stem kernels run min(tiles, 4 x SMs) persistent CTAs that loop over their tiles, and the element-wise kernels
loop grid-stride over at most 16 x SMs blocks of 256 threads (grid_for in api.cu).  The shapes that must make a CTA or a thread run
its loop body more than once are derived from the live SM count, and each test asserts that they do."""
import numpy as np
import pytest
import torch

from hawq_b200 import ops
from oracle.int_ref import dyadic          # the library's (m, e) pairs, and importable without it
from tests import abi_model as am
from tests.kernel_harness import DEV, I32_MAX, I32_MIN, RATIO_ONE, edge_biases, kernel_count, out_buf, rng, run_both, sm_count

pytestmark = pytest.mark.gpu


def stem_cta_cap():
    return 4 * sm_count()


def grid_stride_cap():
    """work items the element-wise kernels cover in one pass: 16 blocks of 256 threads per SM"""
    return 16 * sm_count() * 256


def at_least(per_unit, items):
    """the smallest count of units of per_unit work items that reaches items"""
    return -(-items // per_unit)


# ------------------------------------------------------------------------------------------------ stem
STEM_A = 147 * 128 * 128     # acc of an interior output of an all -128 image under a weight row of -128
STEM_BIASES = [I32_MIN, I32_MIN + 1, I32_MAX, -STEM_A, -STEM_A - 1, STEM_A, STEM_A + 1, None]    # None: random, |bias| <= 2^16
STEM_RATIOS = [RATIO_ONE, dyadic(0.5), dyadic(0.25), (0, 31), dyadic(5e-8), dyadic(1e-9), None]   # None: log-uniform in [1e-4, 1]
STEM_CASES = [
    # (m, e) of channel 63 (None: every ratio <= 1, the FP64 requantisation), clamp.  One ratio above 1 sends the whole CTA to the
    # exact 64-bit requantisation.  clamp_hi < 0: the documented max(0, clamp(q, lo, hi)) is 0 everywhere.
    (None, (-32768, 32767)), (None, (100, 200)), (None, (-300, -7)), (dyadic(3.0), (-32768, 32767)), ((2 ** 31, 11), (100, 200))]


def stem_images(r, n, h, w):
    """image i % 3 == 0: every value -128; 1: every value 127; 2: random"""
    v = r.randint(-128, 128, size=(n, h * w * 3))
    v[0::3] = -128
    v[1::3] = 127
    return torch.from_numpy(v.reshape(-1).astype(np.int8))


def stem_weights_chan(r, wide, rows):
    """Channel c: weight row -128 / 127 / -127 / random by c % 4, bias STEM_BIASES[(c // 4) % 8], ratio STEM_RATIOS[c % 7]; each
    (row, bias) pair occurs twice, with two different ratios.  The ratios 0.5 and 0.25 make round-half-even ties on random images.
    wide: (m, e) of channel 63.  rows: 7 (hawq_stem_conv_i8) or 8 (hawq_stem_pool_i8) kernel rows; the padding taps stay 0."""
    core = r.randint(-128, 128, size=(64, 7, 7, 3))
    bias, me = [], []
    for c in range(64):
        row = (-128, 127, -127, None)[c % 4]
        if row is not None:
            core[c] = row
        b = STEM_BIASES[(c // 4) % 8]
        bias.append(int(r.randint(-2 ** 16, 2 ** 16)) if b is None else b)
        mc = STEM_RATIOS[c % 7]
        me.append(dyadic(float(np.exp(r.uniform(np.log(1e-4), 0.0)))) if mc is None else mc)
    if wide is not None:
        me[63] = wide
    wt = torch.zeros((64, rows, 8, 4), dtype=torch.int8)
    wt[:, :7, :7, :3] = torch.from_numpy(core.astype(np.int8))
    return wt, ops.make_chan(bias, [m for m, _ in me], [e for _, e in me])


STEM_GEOMS = [
    # H, W, N, waves: N = None -> enough images for more than `waves` x (4 x SMs) tiles of 8 x 16 outputs
    (7, 7, 3, None),          # the smallest input: one tile, 4 x 4 outputs
    (9, 13, 2, None),         # odd sizes
    (33, 17, 2, None),        # Ho = 17, Wo = 9: a tile row with one valid output row
    (30, 46, None, 2),        # Ho = 15, Wo = 23: tiles ending inside and outside the image; CTAs run up to 3 tiles
    (224, 224, None, 1),      # ImageNet size, 98 tiles per image
]


@pytest.mark.parametrize("geom", STEM_GEOMS)
def test_stem_conv_edges(geom):
    """hawq_stem_conv_i8 with saturating biases, ratio edges, the exact branch, narrow and negative clamps and persistent CTAs that
    loop over several tiles."""
    h, w, n, waves = geom
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    per_image = -(-ho // 8) * -(-wo // 16)
    if n is None:
        n = at_least(per_image, waves * stem_cta_cap() + 1)
        assert n * per_image >= waves * stem_cta_cap() + 1
    r = rng(h * 1000 + w)
    x = stem_images(r, n, h, w)
    for wide, clamp in STEM_CASES:
        wt, chan = stem_weights_chan(r, wide, 7)
        (c16,), (g16,) = run_both("stem_conv", dict(x=x, w=wt, chan=chan, clamp=clamp, out=torch.zeros(n * ho * wo * 64, dtype=torch.int16),
                                                    n=n, hh=h, ww=w), ["out"])
        assert torch.equal(c16, g16), (geom, wide, clamp, int((c16 != g16).sum()))


STEM_POOL_GEOMS = [
    # H, W, N, waves: N = None -> enough images for more than `waves` x (4 x SMs) tiles of 3 x 7 pooled pixels.  W % 16 == 0, W <= 256
    (7, 16, 3, None),         # the smallest input: 2 x 4 pooled pixels
    (37, 48, 2, None),        # odd H: Po = 10, a band with one valid pooled row
    (30, 256, 1, None),       # the widest row the kernel takes
    (32, 48, None, 2),        # 6 tiles per image, bands ending inside the image; CTAs run up to 3 tiles
    (224, 224, None, 1),      # ImageNet size, 152 tiles per image
]
STEM_POOL_OUTS = [
    # y_bits, low_bits, low (m, e), low clamp: the low-bit ratio must be <= 1 in the fused kernel
    (16, 8, RATIO_ONE, (-128, 127)),
    (32, 4, dyadic(0.5), (0, 15)),
    (16, 0, (0, 1), (0, 0)),
    (32, 8, (0, 31), (-128, 127)),
    (16, 4, dyadic(0.003), (3, 9)),
    (32, 8, dyadic(2.0 ** -8), (-5, 100)),
]


@pytest.mark.parametrize("geom", STEM_POOL_GEOMS)
def test_stem_pool_fused_edges(geom):
    """hawq_stem_pool_i8 == hawq_stem_conv_i8 + hawq_maxpool_requant of the model, with the stem edges of test_stem_conv_edges, both
    residual-stream widths, low-bit ratios exactly 1, 0.5 (ties), m = 0 and small, narrow low clamps, and CTAs that loop over tiles."""
    h, w, n, waves = geom
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    po, qo = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    per_image = -(-po // 3) * -(-qo // 7)
    if n is None:
        n = at_least(per_image, waves * stem_cta_cap() + 1)
        assert n * per_image >= waves * stem_cta_cap() + 1
    r = rng(h * 1000 + w + 1)
    x = stem_images(r, n, h, w)
    numel = n * po * qo * 64
    for i, (y_bits, low_bits, low_me, low_clamp) in enumerate(STEM_POOL_OUTS):
        wide, clamp = STEM_CASES[i % len(STEM_CASES)]
        wt, chan = stem_weights_chan(r, wide, 8)
        args = dict(x=x, w256=wt, chan=chan, clamp=clamp, n=n, hh=h, ww=w, y_bits=y_bits, y=out_buf(numel, y_bits), low_bits=low_bits,
                    low_me=low_me, low_clamp=low_clamp, out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = ["y"] + (["out_low"] if low_bits else [])
        before = kernel_count(6)
        cs, gs = run_both("stem_pool", args, keys)
        assert kernel_count(6) == before + 1, "the fused stem did not take this launch"
        for a, b, k in zip(cs, gs, keys):
            assert torch.equal(a, b), (geom, wide, clamp, y_bits, low_bits, low_me, k, int((a != b).sum()))


# ------------------------------------------------------------------------------------------------ max-pool + requant
POOL_LOWS = [
    # low_bits, low (m, e), low clamp.  Ratios above 1 take the exact branch; from 2^16 up, 32767 * ratio leaves int32 and saturates.
    (8, RATIO_ONE, (-128, 127)),
    (8, dyadic(0.5), (-128, 127)),
    (4, dyadic(0.25), (0, 15)),
    (8, (0, 31), (-128, 127)),
    (8, dyadic(3.0), (-128, 127)),
    (8, (2 ** 31, 11), (-128, 127)),          # 2^20
    (4, dyadic(2.0 ** 17 + 5), (0, 15)),
    (8, dyadic(0.003), (20, 30)),
    (4, dyadic(1.5), (7, 8)),
    (0, (0, 1), (0, 0)),
]


def pool_input(r, n, h, w, c):
    """int16 [N, H, W, C] in [0, 32767]: by channel, small values (ties at 0.5 and 0.25, unsaturated low-bit copies), the whole
    range, or values near 32767; image 0 has a block of 32767 and image 1 (if any) a block of 0"""
    v = np.empty((n, h, w, c), dtype=np.int64)
    v[..., 0::3] = r.randint(0, 64, size=v[..., 0::3].shape)
    v[..., 1::3] = r.randint(0, 32768, size=v[..., 1::3].shape)
    v[..., 2::3] = r.randint(32000, 32768, size=v[..., 2::3].shape)
    v[0, : (h + 1) // 2, : (w + 1) // 2] = 32767
    if n > 1:
        v[1, h // 2:, w // 2:] = 0
    return torch.from_numpy(v.reshape(-1).astype(np.int16))


POOL_GEOMS = [(2, 1, 1), (3, 2, 3), (2, 3, 2), (2, 1, 7), (2, 9, 1), (2, 7, 10), (1, 12, 9)]     # N, H, W


@pytest.mark.parametrize("c", [8, 24, 64, 256])
def test_maxpool_requant_edges(c):
    """hawq_maxpool_requant at 1-, 2- and 3-pixel sides, odd and even sizes, inputs up to 32767, the exact branch of the low-bit
    requantisation (ratios above 1, up to 2^20, saturating), ratio exactly 1, m = 0, ties and narrow low clamps."""
    r = rng(300 + c)
    for n, h, w in POOL_GEOMS:
        x = pool_input(r, n, h, w, c)
        po, qo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        numel = n * po * qo * c
        for i, (low_bits, low_me, low_clamp) in enumerate(POOL_LOWS):
            y_bits = (16, 32, 0)[i % 3] if low_bits else 32
            args = dict(x=x, n=n, hh=h, ww=w, c=c, y_bits=y_bits, y=out_buf(numel, y_bits) if y_bits else None, low_bits=low_bits,
                        low_me=low_me, low_clamp=low_clamp, out_low=out_buf(numel, low_bits) if low_bits else None)
            keys = [k for k in ("y", "out_low") if args[k] is not None]
            cs, gs = run_both("maxpool_requant", args, keys)
            for a, b, k in zip(cs, gs, keys):
                assert torch.equal(a, b), (c, (n, h, w), y_bits, low_bits, low_me, k)


def test_maxpool_requant_several_passes():
    """More output groups of 8 channels than one grid-stride pass covers."""
    c, h, w = 64, 57, 57
    po = qo = (h - 1) // 2 + 1
    n = at_least(po * qo * c // 8, grid_stride_cap() + 1)
    assert n * po * qo * c // 8 > grid_stride_cap()
    r = rng(57)
    x = pool_input(r, n, h, w, c)
    numel = n * po * qo * c
    for y_bits, (low_bits, low_me, low_clamp) in [(16, POOL_LOWS[5]), (32, POOL_LOWS[2])]:
        args = dict(x=x, n=n, hh=h, ww=w, c=c, y_bits=y_bits, y=out_buf(numel, y_bits), low_bits=low_bits, low_me=low_me,
                    low_clamp=low_clamp, out_low=out_buf(numel, low_bits))
        cs, gs = run_both("maxpool_requant", args, ["y", "out_low"])
        for a, b, k in zip(cs, gs, ["y", "out_low"]):
            assert torch.equal(a, b), (y_bits, low_bits, k)


# ------------------------------------------------------------------------------------------------ average pool + requant
AVG_CASES = [   # (m, e), clamp
    (RATIO_ONE, (-128, 127)), (dyadic(0.5), (-128, 127)), (dyadic(0.25), (-5, 5)), ((0, 31), (-128, 127)), (dyadic(1e-9), (-128, 127)),
    (dyadic(0.004), (0, 127)), (dyadic(3.0), (-128, 127)), ((2 ** 31, 11), (-100, 100))]


def avg_input(r, n, hw, c, x_bits):
    """[N, HW, C].  x_bits 16, column j = n * C + c by j % 3: random, all 65535, small.  x_bits 32 by j % 7: random, all INT32_MAX,
    all INT32_MIN, then negative sums that are exact multiples of HW, -1 and -(HW - 1) modulo HW, and small values around 0."""
    cols = n * c
    if x_bits == 16:
        v = r.randint(0, 65536, size=(cols, hw))
        v[1::3] = 65535
        v[2::3] = r.randint(0, 4, size=v[2::3].shape)
    else:
        v = r.randint(I32_MIN, I32_MAX, size=(cols, hw), dtype=np.int64)
        v[1::7] = I32_MAX
        v[2::7] = I32_MIN
        for j, t in ((3, 0), (4, -1), (5, 1 - hw)):
            s = r.randint(-2 ** 24, 0, size=v[j::7].shape)
            s[:, 0] -= (s.sum(axis=1) - t) % hw                    # sum = t (mod HW), sum < 0
            v[j::7] = s
        v[6::7] = r.randint(-3, 2, size=v[6::7].shape)
    x = v.reshape(n, c, hw).transpose(0, 2, 1).reshape(-1)
    if x_bits == 16:
        return torch.from_numpy(x.astype(np.uint16).view(np.int16))
    return torch.from_numpy(x.astype(np.int32))


@pytest.mark.parametrize("x_bits", [16, 32])
@pytest.mark.parametrize("hw", [1, 4, 49, 64])
def test_avgpool_requant_edges(hw, x_bits):
    """hawq_avgpool_requant: sums near HW * 2^31, negative sums on and next to multiples of HW (an exact negative multiple loses one;
    at HW = 1 every negative value is one), and ratios exactly 1, 0.5 / 0.25 (ties), m = 0, tiny and above 1 (saturating)."""
    r = rng(hw * 10 + x_bits)
    for c in (8, 2048):
        n = 3
        x = avg_input(r, n, hw, c, x_bits)
        for me, clamp in AVG_CASES:
            (a,), (b,) = run_both("avgpool_requant", dict(x=x, n=n, hw=hw, c=c, x_bits=x_bits, me=me, clamp=clamp,
                                                          out=torch.zeros(n * c, dtype=torch.int8)), ["out"])
            assert torch.equal(a, b), (hw, x_bits, c, me, clamp)


@pytest.mark.parametrize("hw, x_bits", [(1, 32), (4, 16)])
def test_avgpool_requant_several_passes(hw, x_bits):
    """More (image, channel) outputs than one grid-stride pass covers."""
    c = 2048
    n = at_least(c, grid_stride_cap() + 1)
    assert n * c > grid_stride_cap()
    r = rng(4 * hw + x_bits)
    x = avg_input(r, n, hw, c, x_bits)
    for me, clamp in (AVG_CASES[1], AVG_CASES[6]):
        (a,), (b,) = run_both("avgpool_requant", dict(x=x, n=n, hw=hw, c=c, x_bits=x_bits, me=me, clamp=clamp,
                                                      out=torch.zeros(n * c, dtype=torch.int8)), ["out"])
        assert torch.equal(a, b), (hw, x_bits, me)


# ------------------------------------------------------------------------------------------------ input quantisation
FLT_MAX = float(np.finfo(np.float32).max)
F32_CASES = [(2.0 ** -4, (-128, 127)), (0.0173, (-127, 127)), (2.0 ** -10, (-20, 50)), (1e30, (-128, 127))]   # scale, clamp


@pytest.mark.parametrize("c", [1, 3, 4])
def test_quantize_input_f32_edges(c):
    """hawq_quantize_input_f32 with +-inf, +-FLT_MAX, -0.0 and exact round-half-even ties: at scale 2^-4, x = (k + 1/2) * scale is a
    tie for every k in [-130, 130] (beyond +-128 the tie is clamped).  NaN is outside the reference's semantics and not tested."""
    r = rng(40 + c)
    n, h, w = 2, 17, 13
    xf = r.randn(n * c * h * w).astype(np.float32) * 40
    ties = (np.arange(-130, 131) + 0.5).astype(np.float32) * np.float32(2.0 ** -4)
    specials = np.array([np.inf, -np.inf, FLT_MAX, -FLT_MAX, -0.0, 0.0, 1e-30, -1e-30], dtype=np.float32)
    xf[:ties.size] = ties
    xf[-specials.size:] = specials
    x = torch.from_numpy(xf.reshape(n, c, h, w))
    for scale, clamp in F32_CASES:
        with np.errstate(over="ignore"):
            (a,), (b,) = run_both("quantize_input", dict(x=x, scale=scale, clamp=clamp, out=torch.zeros(n * h * w * c, dtype=torch.int8)), ["out"])
        assert torch.equal(a, b), (c, scale, clamp)


def test_quantize_input_f32_several_passes():
    """More pixels than one grid-stride pass covers."""
    c, h, w = 3, 224, 224
    n = at_least(h * w, grid_stride_cap() + 1)
    assert n * h * w > grid_stride_cap()
    r = rng(224)
    x = torch.from_numpy(r.randn(n, c, h, w).astype(np.float32) * 2)
    for scale, clamp in F32_CASES[:2]:
        (a,), (b,) = run_both("quantize_input", dict(x=x, scale=scale, clamp=clamp, out=torch.zeros(n * h * w * c, dtype=torch.int8)), ["out"])
        assert torch.equal(a, b), (scale, clamp)


U8_NORMS = [   # mean, std, scale, clamp
    ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225), 0.0207, (-127, 127)),
    ((0.5, 0.25, 0.75), (0.5, 0.1, 2.0), 0.0131, (0, 127)),
    ((0.5, 0.5, 0.5), (1e-4, 1e-4, 1e-4), 0.05, (-128, 127)),      # tiny std: everything but u = 127.5 saturates at either end
    ((0.0, 1.0, 0.3), (1.0, 1.0, 0.05), 0.007, (0, 127)),
]


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 2), (1, 1, 3), (1, 2, 2), (2, 3, 5), (3, 7, 9), (1, 5, 7), (2, 16, 16)])
def test_quantize_input_u8_tails(shape):
    """hawq_quantize_input_u8 with N * H * W = 0, 1, 2, 3 (mod 4), i.e. 0, 3, 2 or 1 tail bytes after the last whole word, an image
    shorter than one word, and non-ImageNet normalisations."""
    n, h, w = shape
    r = rng(n * 100 + h * 10 + w)
    u8 = torch.from_numpy(r.randint(0, 256, size=(n, h, w, 3)).astype(np.uint8))
    if n * h * w >= 256:
        u8.view(-1)[:768] = torch.arange(256, dtype=torch.uint8).repeat_interleave(3)       # every value in every channel
    for mean, std, scale, clamp in U8_NORMS:
        (a,), (b,) = run_both("quantize_input_u8", dict(x=u8, mean=mean, std=std, scale=scale, clamp=clamp, out=out_buf(n * h * w * 3, 8)),
                              ["out"])
        assert torch.equal(a, b), (shape, mean, std, scale)


def test_quantize_input_u8_several_passes():
    """More 4-byte words than one grid-stride pass covers, followed by 3 tail bytes."""
    h, w = 223, 223
    n = at_least(h * w * 3 // 4, grid_stride_cap() + 1)
    n += (1 - n * h * w) % 4                                           # N * H * W = 1 (mod 4): 3 tail bytes
    assert n * h * w * 3 // 4 > grid_stride_cap() and n * h * w * 3 % 4 == 3
    r = rng(223)
    u8 = torch.from_numpy(r.randint(0, 256, size=(n, h, w, 3)).astype(np.uint8))
    for mean, std, scale, clamp in U8_NORMS[:2]:
        (a,), (b,) = run_both("quantize_input_u8", dict(x=u8, mean=mean, std=std, scale=scale, clamp=clamp, out=out_buf(n * h * w * 3, 8)),
                              ["out"])
        assert torch.equal(a, b), (mean, std, scale)


# ------------------------------------------------------------------------------------------------ dequant, nibble packing
def dequant_input(r, numel, bits, signed):
    """x_bits 32: the int32 limits, values around 2^24 (odd: the int -> float conversion rounds) and random int32; narrower widths
    span their whole range"""
    if bits == 4:
        return torch.from_numpy(am.pack_i4(r.randint(0, 16, size=numel)))
    if bits == 32:
        v = r.randint(I32_MIN, I32_MAX, size=numel, dtype=np.int64)
        near = np.array([2 ** 24 + 1, 2 ** 24 + 3, 2 ** 25 + 1, 2 ** 25 + 2, 2 ** 25 + 6, 2 ** 30 + 1, 2 ** 31 - 65, 2 ** 31 - 64], dtype=np.int64)
        edges = np.concatenate([[I32_MIN, I32_MIN + 1, I32_MAX, I32_MAX - 1], near, -near])
        v[:edges.size] = edges
        v[edges.size:2 * edges.size] = r.randint(2 ** 24, 2 ** 25, size=edges.size) | 1
        return torch.from_numpy(v.astype(np.int32))
    lo, hi = (-2 ** (bits - 1), 2 ** (bits - 1)) if signed else (0, 2 ** bits)
    v = r.randint(lo, hi, size=numel)
    v[:2] = lo, hi - 1
    dt = {(8, True): np.int8, (8, False): np.uint8, (16, True): np.int16, (16, False): np.uint16}[(bits, signed)]
    return torch.from_numpy(v.astype(dt).view(np.int8 if bits == 8 else np.int16))


def check_dequant(x, n, h, w, c, bits, signed, scale):
    with np.errstate(over="ignore"):
        (a,), (b,) = run_both("dequant", dict(x=x, n=n, hh=h, ww=w, c=c, x_bits=bits, x_signed=signed, scale=scale,
                                              out=torch.zeros(n, c, h, w)), ["out"])
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), ((n, h, w, c), bits, signed, scale)   # bit patterns: inf, -0.0


DEQUANT_CASES = [(c, bits, signed) for c in (3, 5) for bits, signed in [(8, True), (8, False), (16, True), (16, False), (32, True)]] + \
                [(8, 4, False), (24, 4, False)]


@pytest.mark.parametrize("c, bits, signed", DEQUANT_CASES)
def test_dequant_edges(c, bits, signed):
    """hawq_dequant_f32 at odd C and packed C = 8 / 24; int32 values at +-2^31 and around 2^24 + odd, where the conversion to float
    rounds (to nearest even); scale 1 shows that rounding directly and 3e38 overflows to inf."""
    r = rng(c * 64 + bits + signed)
    n, h, w = 2, 5, 7
    x = dequant_input(r, n * h * w * c, bits, signed)
    for scale in (0.0371, 1.0, 3e38):
        check_dequant(x, n, h, w, c, bits, signed, scale)


@pytest.mark.parametrize("c, bits", [(3, 32), (8, 4)])
def test_dequant_several_passes(c, bits):
    """More output elements than one grid-stride pass covers."""
    h, w = 224, 224
    n = at_least(c * h * w, grid_stride_cap() + 1)
    assert n * c * h * w > grid_stride_cap()
    x = dequant_input(rng(bits), n * h * w * c, bits, bits == 32)
    check_dequant(x, n, h, w, c, bits, bits == 32, 0.0371)


def test_pack_unpack_i4_several_passes():
    """hawq_pack_i4 / hawq_unpack_i4 of all 16 values over more groups of 8 than one grid-stride pass covers."""
    groups = grid_stride_cap() + 4099
    v = np.tile(np.arange(16, dtype=np.uint8), groups // 2)
    v[8 * 4099:] = rng(16).randint(0, 16, size=v.size - 8 * 4099)
    assert v.size // 8 > grid_stride_cap()
    src = torch.from_numpy(v)
    packed = torch.zeros(v.size // 2, dtype=torch.uint8, device=DEV)
    ops.pack_i4(src.to(DEV), packed)
    back = torch.zeros(v.size, dtype=torch.uint8, device=DEV)
    ops.unpack_i4(packed, back)
    torch.cuda.synchronize()
    assert torch.equal(packed.cpu(), torch.from_numpy(am.pack_i4(v)))
    assert torch.equal(back.cpu(), src)


# ------------------------------------------------------------------------------------------------ classifier
@pytest.mark.parametrize("nb", [1, 257])
@pytest.mark.parametrize("kk, co, cp", [(128, 8, 8), (128, 5, 8), (8192, 8, 8), (8192, 7, 8), (8320, 61, 64)])
def test_linear_k_limits(kk, co, cp, nb):
    """hawq_linear_i8 at K = 128, K = 8192 (the largest K of the dp4a kernel) and K = 8320 (the convolution instead), with rows of
    -128 / 127, constant weight rows and biases at the int32 limits and on both sides of the window where acc + bias cannot
    saturate; N = 257 leaves a ragged block of rows."""
    r = rng(kk + co + nb)
    x = r.randint(-128, 128, size=(nb, kk))
    x[0::3] = -128
    x[1::3] = 127
    wl = r.randint(-128, 128, size=(cp, kk))
    for c in range(cp):
        row = (-128, 127, -127, None)[c % 4]
        if row is not None:
            wl[c] = row
    wl[co:] = 0
    edges = edge_biases(kk, 8)
    chl = ops.make_chan([edges[(c + c // 8) % 8] for c in range(cp)], [2 ** 30] * cp, [40] * cp)
    fs = torch.from_numpy(r.uniform(1e-5, 1e-3, size=cp).astype(np.float32))
    before = kernel_count(0)
    (c,), (g,) = run_both("linear", dict(x=torch.from_numpy(x.reshape(-1).astype(np.int8)), w=torch.from_numpy(wl.astype(np.int8)), chan=chl,
                                         fscale=fs, out=torch.zeros((nb, co)), n=nb, k=kk, cout=co, cout_pad=cp), ["out"])
    assert kernel_count(0) == before + (kk > 8192), "the dp4a kernel takes K <= 8192, the convolution larger K"
    assert torch.equal(c.view(torch.int32), g.view(torch.int32)), (kk, co, cp, nb)
