"""-m gpu: every CUDA kernel behind the C ABI against the numpy ABI model (tests/abi_model.py -> oracle/int_ref.py)
on the same seeded buffers.  Integer work: bit-exact, no tolerance."""
import numpy as np
import pytest
import torch

from hawq_b200 import ops
from hawq_b200._lib import EPI_DEQUANT_F32, EPI_RAW_I32, EPI_REQUANT, EPI_RESIDUAL, HawqError, dyadic
from tests import abi_model as am
from tests.kernel_harness import (DEV, I32_MAX, I32_MIN, RATIO_ONE, TC_FLAG, boundary_weights_chan, check_conv1x1_requant_and_residual,
                                  check_conv_dual_stationary_weights, check_conv_epilogue_boundaries, check_conv_raw_and_dequant_geoms,
                                  check_conv_requant, check_conv_residual, check_stem_and_pool, edge_biases, extreme_act, make_chan,
                                  out_buf, out_hw, rand_act, res_chan_with_ties, rng, run_both)
from tests.util import POISON

pytestmark = pytest.mark.gpu


CONV_GEOMS = [
    # N, H, W, Cin, Cout, kh, kw, stride, pad
    (2, 8, 8, 64, 64, 1, 1, 1, 0),
    (3, 7, 7, 64, 128, 3, 3, 1, 1),       # M = 147: ragged last tile
    (2, 14, 14, 128, 64, 3, 3, 2, 1),
    (2, 9, 9, 256, 256, 1, 1, 2, 0),
    (1, 20, 12, 64, 192, 3, 3, 1, 1),     # Cout = 192 -> BN = 64 path with 3 column tiles
    (5, 6, 6, 128, 128, 3, 3, 1, 1),
    (3, 7, 7, 128, 128, 1, 1, 1, 0),      # 1x1 stride 1, M = 147: ragged (zero-filled) last tile
    (2, 5, 5, 192, 256, 1, 1, 1, 0),      # M = 50 < one tile, K = 3 k-tiles
    (2, 7, 7, 512, 128, 3, 3, 1, 1),      # K = 4608, 72 k-tiles: the deepest ResNet layer
    (2, 9, 9, 64, 64, 5, 5, 1, 2),
    (2, 15, 15, 64, 128, 7, 7, 2, 3),
    (2, 8, 8, 64, 128, 1, 3, 1, 0),
    (2, 8, 8, 64, 64, 3, 1, 1, 0),
    (2, 7, 7, 64, 64, 1, 1, 1, 1),        # 1x1 with padding: the border ring of outputs sees only zeros
    (2, 11, 11, 64, 128, 3, 3, 3, 2),
    (3, 2, 3, 64, 64, 5, 5, 1, 2),        # input smaller than the kernel
]


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", CONV_GEOMS)
def test_conv_requant(geom, a_bits, tc):
    check_conv_requant(geom, a_bits, tc)


@pytest.mark.parametrize("ratio_kind", ["pow2_ties", "above_one_mixed"])
def test_conv_requant_ties_and_generic_path(ratio_kind):
    """Identity 1x1 weights make acc = x, so v = x + bias sweeps chosen integers: power-of-two ratios give exact .5 ties
    (round-half-to-even, NOT TVM's half-up); ratios > 1 force the generic 64-bit requant instead of the FP64-FMA fast path."""
    r = rng(99)
    n, h, w, c = 2, 16, 16, 64
    x = rand_act(r, n * h * w * c, 8)
    wt = torch.zeros((c, 1, 1, c), dtype=torch.int8)
    for i in range(c):
        wt[i, 0, 0, i] = 1
    if ratio_kind == "pow2_ties":
        ratios = [2.0 ** -(i % 8 + 1) for i in range(c)]
        bias = [1000 * i + 8 * (i % 3) for i in range(c)]
    else:
        ratios = [float(np.exp(r.uniform(np.log(0.3), np.log(6.0)))) for _ in range(c)]
        bias = r.randint(-50000, 50000, size=c).tolist()
    me = [dyadic(v) for v in ratios]
    chan = ops.make_chan(bias, [m for m, _ in me], [e for _, e in me])
    d = ops.conv_desc(n, h, w, c, c, 1, 1, 1, 0, 8)
    for out_bits, clamp, relu in [(32, (-2 ** 31, 2 ** 31 - 1), 0), (16, (-32768, 32767), 0), (8, (-128, 127), 1)]:
        ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp)
        (c_out,), (g_out,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(n * h * w * c, out_bits)), ["out"])
        assert torch.equal(c_out, g_out), (ratio_kind, out_bits)
    # residual form with a scalar ratio > 1 on the identity operand and on the low-bit copy
    res = rand_act(r, n * h * w * c, 32)
    ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=32, res_me=dyadic(1.5 if ratio_kind != "pow2_ties" else 0.25), y_bits=32,
                      low_bits=8, low_me=dyadic(2.0 ** -7), low_clamp=(-128, 127))
    cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, out=out_buf(n * h * w * c, 32),
                                     out_low=out_buf(n * h * w * c, 8)), ["out", "out_low"])
    for a, b in zip(cs, gs):
        assert torch.equal(a, b), ratio_kind


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", CONV_GEOMS[:4] + CONV_GEOMS[6:])
def test_conv_residual(geom, a_bits, tc):
    check_conv_residual(geom, a_bits, tc)


@pytest.mark.parametrize("geom", [CONV_GEOMS[0], CONV_GEOMS[3], CONV_GEOMS[5]])
def test_conv_residual_wide_ratios_on_tensor_cores(geom):
    """HAWQ_EP_RATIOS_LE_2P20: ratios above 1 (typical for the 16-bit residual requant) are exact, and a term leaving int32 is flagged."""
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = rng(4242 + sum(geom))
    ho, wo = out_hw(h, w, kh, kw, s, p)
    numel = n * ho * wo * cout
    x = rand_act(r, n * h * w * cin, 8)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, kh, kw, cin)).astype(np.int8))
    chan = make_chan(r, cout, bias_mag=2000, ratio_lo=0.2, ratio_hi=40.0)
    d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, 8)
    for res_kind, res_bits, y_bits, low_bits in [(0, 16, 16, 8), (0, 32, 32, 4), (1, 32, 16, 8)]:
        res = rand_act(r, numel, res_bits if res_kind == 0 else 32)
        if res_bits == 16 and res_kind == 0:
            res = torch.from_numpy(r.randint(0, 900, size=numel).astype(np.uint16).view(np.int16))
        res_chan = make_chan(r, cout, ratio_lo=0.5, ratio_hi=3.0) if res_kind == 1 else None
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=res_kind, res_bits=res_bits, res_me=dyadic(1.37), y_bits=y_bits,
                          low_bits=low_bits, low_me=dyadic(0.0004), low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=2)
        cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, res_chan=res_chan, out=out_buf(numel, y_bits),
                                         out_low=out_buf(numel, low_bits)), ["out", "out_low"])
        for a, b in zip(cs, gs):
            assert torch.equal(a, b), (geom, res_kind, res_bits, y_bits, low_bits)
    # a term that leaves int32 on the fast path must raise HAWQ_FLAG_REQUANT_OVERFLOW (the generic kernel would saturate)
    res = torch.full((numel,), 2 ** 30, dtype=torch.int32)
    ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=32, res_me=dyadic(1000.0), y_bits=32, flags=2)
    ops.reset_status(0)
    ops.conv2d(x.to(DEV), d, ep, wt.to(DEV), chan.to(DEV), res=res.to(DEV), out=torch.zeros(numel, dtype=torch.int32, device=DEV))
    assert ops.get_status(0) & 4
    ops.reset_status(0)


WS_GEOMS = [
    # N, H, W, Cin, Cout, k, stride, pad : REQUANT with re-tiled weights (w_layout 1), more tiles than SMs
    (7, 56, 56, 64, 64, 3, 1, 1),      # 172 row tiles, one channel block
    (4, 49, 49, 128, 128, 3, 1, 1),    # K = 1152, 152 tiles
    (3, 57, 57, 256, 256, 1, 1, 0),    # 1x1 stride 1, 154 tiles, 2 channel blocks
    (2, 31, 31, 128, 128, 1, 2, 0),    # strided 1x1
    (2, 30, 30, 64, 192, 3, 2, 1),     # strided 3x3, 3 narrow channel blocks
    (1, 9, 9, 64, 64, 1, 1, 0),        # single k-tile, single ragged tile
]


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", WS_GEOMS)
def test_conv_requant_retiled_weights_many_tiles(geom, a_bits):
    n, h, w, cin, cout, k, s, p = geom
    r = rng(9001 + sum(v * (i + 2) for i, v in enumerate(geom)) + a_bits)
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128, 128, size=(cout, k, k, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    chan = make_chan(r, cout, ratio_lo=2e-5, ratio_hi=2e-3)
    wg = ops.upload_weights(wt, DEV)
    d = ops.conv_desc(n, h, w, cin, cout, k, k, s, p, a_bits, 1)
    for out_bits, clamp, relu in [(8, (-128, 127), 1), (4, (0, 15), 1), (8, (-127, 127), 0)]:
        ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=TC_FLAG)
        (c,), (g,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(n * ho * wo * cout, out_bits)), ["out"],
                              gpu_overrides=dict(w=wg))
        assert torch.equal(c, g), (geom, a_bits, out_bits, relu)


DUAL_GEOMS = [
    # N, Ho, Wo, Cin (last conv), Cin2 (identity conv), Cout, identity stride
    (2, 7, 7, 64, 64, 256, 1),         # ResNet-50 stage-1 shape: M = 98 (< one tile), 2 column tiles of 128
    (3, 5, 7, 128, 256, 512, 2),       # stride-2 identity, M = 105
    (2, 12, 12, 64, 128, 192, 2),      # Cout = 192 -> BN = 64, M = 288: 3 row tiles, ragged last
    (1, 9, 16, 192, 64, 128, 1),       # 3 + 1 k-tiles
]


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", DUAL_GEOMS)
def test_conv_dual_resize_unit(geom, a_bits, flag):
    """hawq_conv2d_dual (both convolutions in one kernel) == RAW_I32 identity conv + res_kind-1 RESIDUAL conv of the ABI model."""
    n, ho, wo, cin, cin2, cout, s2 = geom
    r = rng(777 + sum(v * (i + 3) for i, v in enumerate(geom)) * 4 + a_bits + flag)
    h2, w2 = (ho - 1) * s2 + 1 + (s2 - 1), (wo - 1) * s2 + 1     # one extra (unused) row for strided inputs
    assert (h2 - 1) // s2 + 1 == ho and (w2 - 1) // s2 + 1 == wo
    numel = n * ho * wo * cout
    x = rand_act(r, n * ho * wo * cin, a_bits)
    x2 = rand_act(r, n * h2 * w2 * cin2, a_bits)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    wt2 = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin2)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
        ops.permute_weights_for_i4(wt2)
    hi = 0.9 if flag == 1 else 30.0
    chan = make_chan(r, cout, bias_mag=3000, ratio_lo=1e-2, ratio_hi=hi)
    chan2 = make_chan(r, cout, bias_mag=3000, ratio_lo=1e-2, ratio_hi=hi)
    d = ops.conv_desc(n, ho, wo, cin, cout, 1, 1, 1, 0, a_bits, 1)
    d2 = ops.conv_desc(n, h2, w2, cin2, cout, 1, 1, s2, 0, a_bits, 1)
    wg, wg2 = ops.upload_weights(wt, DEV), ops.upload_weights(wt2, DEV)
    for low_bits in (8, 4, 0):
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, low_bits=low_bits, low_me=dyadic(0.003),
                          low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flag)
        args = dict(x=x, desc=d, ep=ep, w=wt, chan=chan, desc2=d2, x2=x2, w2=wt2, chan2=chan2, out=out_buf(numel, 16),
                    out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = ["out"] + (["out_low"] if low_bits else [])
        cs, gs = run_both("conv2d_dual", args, keys, gpu_overrides=dict(w=wg, w2=wg2))
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (geom, a_bits, flag, low_bits, k_)


def test_conv_dual_rejects_unsupported():
    d = ops.conv_desc(1, 4, 4, 64, 64, 1, 1, 1, 0, 8, 0)       # w_layout 0: no re-tiled copy
    ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, flags=1)
    z = torch.zeros(64 * 64 * 2, dtype=torch.int8, device=DEV)
    ch = torch.zeros(64, 4, dtype=torch.int32, device=DEV)
    y = torch.zeros(16 * 64, dtype=torch.int16, device=DEV)
    with pytest.raises(HawqError):
        ops.conv2d_dual(z, d, ep, z, ch, d, z, z, ch, out=y)


def test_residual_overflow_flag():
    r = rng(5)
    n, h, w, cin, cout = 1, 4, 4, 64, 64
    x = rand_act(r, n * h * w * cin, 8)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    chan = make_chan(r, cout, ratio_lo=0.5, ratio_hi=0.9)
    res = torch.full((n * h * w * cout,), 60000, dtype=torch.int32)
    d = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, 8)
    ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=32, res_me=dyadic(1.9), y_bits=16)
    ops.reset_status(0)
    y = torch.zeros(n * h * w * cout, dtype=torch.int16, device=DEV)
    ops.conv2d(x.to(DEV), d, ep, wt.to(DEV), chan.to(DEV), res=res.to(DEV), out=y)
    assert ops.get_status(0) & 1
    assert int((y.cpu().view(torch.int16).to(torch.int32) & 0xFFFF).max()) == 65535
    ops.reset_status(0)
    assert ops.get_status(0) == 0


def test_conv_raw_and_dequant():
    r = rng(9)
    n, h, w, cin, cout, k, s, p = 2, 6, 6, 128, 128, 1, 2, 0
    ho = wo = 3
    x = rand_act(r, n * h * w * cin, 8)
    wt = torch.from_numpy(r.randint(-128, 128, size=(cout, k, k, cin)).astype(np.int8))
    chan = make_chan(r, cout)
    d = ops.conv_desc(n, h, w, cin, cout, k, k, s, p, 8)
    for tc in (0, 1):
        (c,), (g,) = run_both("conv2d", dict(x=x, desc=d, ep=ops.epilogue(EPI_RAW_I32, flags=TC_FLAG * tc), w=wt, chan=chan,
                                             out=out_buf(n * ho * wo * cout, 32)), ["out"])
        assert torch.equal(c, g), tc
    # linear tail: 1000 classes padded to 1024
    nb, kk, co, cp = 5, 512, 1000, 1024
    xl = rand_act(r, nb * kk, 8)
    wl = torch.zeros((cp, kk), dtype=torch.int8)
    wl[:co] = torch.from_numpy(r.randint(-128, 128, size=(co, kk)).astype(np.int8))
    chl = make_chan(r, cp)
    fs = torch.from_numpy(r.uniform(1e-5, 1e-3, size=cp).astype(np.float32))
    (c,), (g,) = run_both("linear", dict(x=xl, w=wl, chan=chl, fscale=fs, out=torch.zeros((nb, co)), n=nb, k=kk, cout=co, cout_pad=cp), ["out"])
    assert torch.equal(c, g)


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [CONV_GEOMS[1], CONV_GEOMS[2], CONV_GEOMS[4]])
def test_conv_raw_and_dequant_geoms(geom, a_bits):
    check_conv_raw_and_dequant_geoms(geom, a_bits)


def poisoned(numel, dtype):
    """a buffer the call must ignore: every byte POISON"""
    return torch.full((numel * torch.empty(0, dtype=dtype).element_size(),), POISON, dtype=torch.uint8).view(dtype)


def test_unused_pointers_stay_untouched():
    """Every pointer a descriptor leaves unused is passed non-null and poisoned (run_both requires it to stay byte-identical):
    res / res_chan / out_low of REQUANT, RAW_I32 and DEQUANT_F32, fscale outside DEQUANT_F32, out with y_bits 0, out_low with
    low_bits 0, res_chan with res_kind 0, and the unused outputs of hawq_conv2d_dual, hawq_maxpool_requant and hawq_stem_pool_i8."""
    r = rng(404)
    n, h, w, cin, cout = 3, 7, 7, 64, 192                                  # M = 147: ragged last row tile, BN = 64
    m = n * h * w
    x = rand_act(r, m * cin, 8)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, 3, 3, cin)).astype(np.int8))
    chan = make_chan(r, cout, ratio_lo=1e-2, ratio_hi=0.9)
    d = ops.conv_desc(n, h, w, cin, cout, 3, 3, 1, 1, 8)
    res32 = rand_act(r, m * cout, 32)
    unused_res = dict(res=poisoned(m * cout, torch.int32), res_chan=poisoned(cout * 4, torch.int32).view(cout, 4))
    unused_fs = dict(fscale=poisoned(cout, torch.float32))
    unused_low = dict(out_low=poisoned(m * cout, torch.int8))
    low8 = dict(low_bits=8, low_me=dyadic(0.004), low_clamp=(-128, 127))
    cases = [   # epilogue, buffers, the outputs among them
        (ops.epilogue(EPI_REQUANT, relu=1, out_bits=8, clamp=(-128, 127), flags=TC_FLAG),
         dict(out=out_buf(m * cout, 8), **unused_res, **unused_fs, **unused_low), ["out"]),
        (ops.epilogue(EPI_REQUANT, out_bits=32, clamp=(-2 ** 31, 2 ** 31 - 1)),
         dict(out=out_buf(m * cout, 32), **unused_res, **unused_fs, **unused_low), ["out"]),
        (ops.epilogue(EPI_RAW_I32), dict(out=out_buf(m * cout, 32), **unused_res, **unused_fs, **unused_low), ["out"]),
        (ops.epilogue(EPI_DEQUANT_F32, cout_store=cout - 5),
         dict(out=torch.zeros(m * (cout - 5)), fscale=torch.from_numpy(r.uniform(1e-5, 1e-3, size=cout).astype(np.float32)), **unused_res,
              **unused_low), ["out"]),
        (ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=32, res_me=dyadic(0.37), y_bits=0, **low8, flags=TC_FLAG),
         dict(res=res32, res_chan=unused_res["res_chan"], out=poisoned(m * cout, torch.int32), out_low=out_buf(m * cout, 8), **unused_fs), ["out_low"]),
        (ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=32, res_me=dyadic(0.37), y_bits=32),
         dict(res=res32, res_chan=unused_res["res_chan"], out=out_buf(m * cout, 32), **unused_fs, **unused_low), ["out"]),
        (ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, flags=TC_FLAG),
         dict(res=res32, res_chan=make_chan(r, cout, ratio_lo=1e-2, ratio_hi=0.9), out=out_buf(m * cout, 16), **unused_fs, **unused_low), ["out"]),
    ]
    for ep, bufs, keys in cases:
        run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, **bufs), keys)

    # resize-unit kernel without a low-bit copy
    x2 = rand_act(r, m * cin, 8)
    w1 = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    w2 = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    d1 = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, 8, 1)
    ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, flags=TC_FLAG)
    run_both("conv2d_dual", dict(x=x, desc=d1, ep=ep, w=w1, chan=chan, desc2=d1, x2=x2, w2=w2, chan2=make_chan(r, cout, ratio_lo=1e-2, ratio_hi=0.9),
                                 out=out_buf(m * cout, 16), **unused_low), ["out"],
             gpu_overrides=dict(w=ops.upload_weights(w1, DEV), w2=ops.upload_weights(w2, DEV)))

    # max-pool + requant without the stream, and without the low-bit copy
    ph, pw, c = 9, 11, 64
    xp = torch.from_numpy(r.randint(0, 32768, size=2 * ph * pw * c).astype(np.int16))
    pm = 2 * ((ph - 1) // 2 + 1) * ((pw - 1) // 2 + 1) * c
    for y_bits, low_bits in [(0, 8), (16, 0), (32, 0)]:
        args = dict(x=xp, n=2, hh=ph, ww=pw, c=c, y_bits=y_bits, y=out_buf(pm, y_bits or 32), low_bits=low_bits, low_me=dyadic(0.003),
                    low_clamp=(-128, 127), out_low=out_buf(pm, 8))
        if not y_bits:
            args["y"] = poisoned(pm, torch.int32)
        if not low_bits:
            args["out_low"] = poisoned(pm, torch.int8)
        run_both("maxpool_requant", args, ["y" if y_bits else "out_low"])

    # fused stem without the low-bit copy (the stream is always written)
    sh, sw = 17, 32
    xs = torch.from_numpy(r.randint(-128, 128, size=2 * sh * sw * 3).astype(np.int8))
    ws = torch.zeros((64, 8, 8, 4), dtype=torch.int8)
    ws[:, :7, :7, :3] = torch.from_numpy(r.randint(-128, 128, size=(64, 7, 7, 3)).astype(np.int8))
    po, qo = ((sh - 1) // 2) // 2 + 1, ((sw - 1) // 2) // 2 + 1
    run_both("stem_pool", dict(x=xs, w256=ws, chan=make_chan(r, 64, ratio_lo=0.05, ratio_hi=0.8), clamp=(-32768, 32767), n=2, hh=sh, ww=sw, y_bits=16,
                               y=out_buf(2 * po * qo * 64, 16), low_bits=0, low_me=(0, 1), low_clamp=(0, 0), out_low=poisoned(2 * po * qo * 64, torch.int8)),
             ["y"])


@pytest.mark.parametrize("shape", [(130, 2048, 1000, 1024), (128, 512, 10, 64), (3, 192, 100, 128), (1, 64, 64, 64)])
def test_linear_shapes(shape):
    """QuantLinear tail over both implementations: dp4a kernel (K % 128 == 0) and the generic convolution path (other K)."""
    nb, kk, co, cp = shape
    r = rng(31 + nb + kk + co)
    xl = rand_act(r, nb * kk, 8)
    wl = torch.zeros((cp, kk), dtype=torch.int8)
    wl[:co] = torch.from_numpy(r.randint(-128, 128, size=(co, kk)).astype(np.int8))
    chl = make_chan(r, cp, bias_mag=2 ** 20)
    fs = torch.from_numpy(r.uniform(1e-5, 1e-3, size=cp).astype(np.float32))
    (c,), (g,) = run_both("linear", dict(x=xl, w=wl, chan=chl, fscale=fs, out=torch.zeros((nb, co)), n=nb, k=kk, cout=co, cout_pad=cp), ["out"])
    assert torch.equal(c, g), shape


@pytest.mark.parametrize("shape", [(2, 32, 32), (1, 224, 224), (3, 30, 46)])
def test_stem_and_pool(shape):
    check_stem_and_pool(shape)


def test_avgpool_quantize_requant_dequant_pack():
    r = rng(21)
    n, c = 3, 512
    for x_bits in (16, 32):
        x = rand_act(r, n * 49 * c, x_bits)
        if x_bits == 32:
            x[:49 * c] = torch.from_numpy(r.randint(-3, 1, size=49 * c).astype(np.int32))   # negative sums
        (a,), (b,) = run_both("avgpool_requant", dict(x=x, n=n, hw=49, c=c, x_bits=x_bits, me=dyadic(0.004 if x_bits == 16 else 0.9),
                                                      clamp=(-128, 127), out=torch.zeros(n * c, dtype=torch.int8)), ["out"])
        assert torch.equal(a, b)
    xf = torch.from_numpy(r.randn(2, 3, 17, 13).astype(np.float32) * 2)
    xf[0, 0, 0, :4] = torch.tensor([0.5, 1.5, 2.5, -0.5]) * 0.0173      # ties
    (a,), (b,) = run_both("quantize_input", dict(x=xf, scale=0.0173, clamp=(-128, 127), out=torch.zeros(2 * 17 * 13 * 3, dtype=torch.int8)), ["out"])
    assert torch.equal(a, b)
    rows, ch = 37, 64
    for x_bits, per_ch, out_bits in [(32, 1, 8), (16, 0, 4), (32, 1, 16), (16, 0, 8)]:
        x = rand_act(r, rows * ch, x_bits)
        chan = make_chan(r, ch if per_ch else 1, bias_mag=1 if not per_ch else 1000, ratio_lo=1e-3, ratio_hi=0.1)
        clamp = {4: (0, 15), 8: (-128, 127), 16: (-32768, 32767)}[out_bits]
        (a,), (b,) = run_both("requant", dict(x=x, rows=rows, c=ch, x_bits=x_bits, chan=chan, chan_stride=per_ch, relu=1, out_bits=out_bits,
                                              clamp=clamp, out=out_buf(rows * ch, out_bits)), ["out"])
        assert torch.equal(a, b)
    acc = rand_act(r, rows * ch, 32)
    chan = make_chan(r, ch, ratio_lo=0.01, ratio_hi=0.9)
    for res_kind, res_bits, y_bits, low_bits in [(0, 16, 16, 8), (1, 32, 32, 4), (0, 32, 32, 0)]:
        res = rand_act(r, rows * ch, res_bits if res_kind == 0 else 32)
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=res_kind, res_bits=res_bits, res_me=dyadic(0.6), y_bits=y_bits, low_bits=low_bits,
                          low_me=dyadic(0.002), low_clamp=(0, 15) if low_bits == 4 else (-128, 127))
        args = dict(acc=acc, rows=rows, c=ch, chan=chan, ep=ep, res=res, res_chan=make_chan(r, ch, ratio_lo=0.01, ratio_hi=0.9) if res_kind else None,
                    y=out_buf(rows * ch, y_bits), out_low=out_buf(rows * ch, low_bits) if low_bits else None)
        keys = [k for k in ("y", "out_low") if args[k] is not None]
        cs, gs = run_both("add_requant", args, keys)
        for a, b in zip(cs, gs):
            assert torch.equal(a, b)
    for bits, signed in [(4, False), (8, True), (16, False), (32, True)]:
        x = rand_act(r, 2 * 5 * 3 * 16, bits)
        (a,), (b,) = run_both("dequant", dict(x=x, n=2, hh=5, ww=3, c=16, x_bits=bits, x_signed=signed, scale=0.0371, out=torch.zeros(2, 16, 5, 3)), ["out"])
        assert torch.equal(a, b)
    v = torch.from_numpy(r.randint(0, 16, size=4096).astype(np.uint8))
    packed = torch.zeros(2048, dtype=torch.uint8, device=DEV)
    ops.pack_i4(v.to(DEV), packed)
    back = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    ops.unpack_i4(packed, back)
    torch.cuda.synchronize()
    assert torch.equal(packed.cpu(), torch.from_numpy(am.pack_i4(v.numpy()))) and torch.equal(back.cpu(), v)


@pytest.mark.parametrize("shape", [(2, 32, 32), (1, 7, 9), (3, 5, 5)])
def test_quantize_input_u8(shape):
    """uint8 pixels -> int8 network input: equal to the ABI model AND to the two-step torch pipeline + hawq_quantize_input_f32."""
    n, h, w = shape
    r = rng(77 + n * h * w)
    u8 = torch.from_numpy(r.randint(0, 256, size=(n, h, w, 3)).astype(np.uint8))
    if n == 2:
        u8.view(-1)[:768] = torch.arange(256, dtype=torch.uint8).repeat_interleave(3)       # every value in every channel
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    for scale, clamp in [(0.0207, (-128, 127)), (0.005, (-128, 127)), (0.05, (-127, 127))]:
        (c,), (g,) = run_both("quantize_input_u8", dict(x=u8, mean=mean, std=std, scale=scale, clamp=clamp, out=out_buf(n * h * w * 3, 8)), ["out"])
        assert torch.equal(c, g), (shape, scale)
        x = u8.permute(0, 3, 1, 2).to(torch.float32).div(255)
        x = x.sub(torch.tensor(mean).view(1, 3, 1, 1)).div(torch.tensor(std).view(1, 3, 1, 1))
        two_step = torch.zeros(n * h * w * 3, dtype=torch.int8, device=DEV)
        ops.quantize_input(x.contiguous().to(DEV), scale, clamp, two_step)
        assert torch.equal(two_step.cpu(), g), (shape, scale, "vs torch pipeline")


def test_bad_arguments_are_reported():
    x = torch.zeros(64 * 4, dtype=torch.int8, device=DEV)
    w = torch.zeros((64, 1, 1, 48), dtype=torch.int8, device=DEV)
    chan = ops.make_chan([0] * 64, [0] * 64, [1] * 64).to(DEV)
    with pytest.raises(HawqError, match="multiples of 64"):
        ops.conv2d(x, ops.conv_desc(1, 2, 2, 48, 64, 1, 1, 1, 0, 8), ops.epilogue(EPI_REQUANT, out_bits=8, clamp=(-128, 127)), w, chan, out=x)
    with pytest.raises(HawqError, match="requires relu"):
        ops.conv2d(x, ops.conv_desc(1, 2, 2, 64, 64, 1, 1, 1, 0, 8), ops.epilogue(EPI_RESIDUAL, relu=0, res_bits=32, res_me=(1 << 30, 31), y_bits=16),
                   w, chan, res=x, out=x)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.conv2d(x.cpu(), ops.conv_desc(1, 2, 2, 64, 64, 1, 1, 1, 0, 8), ops.epilogue(EPI_RAW_I32), w, chan, out=x)


# ------------------------------------------------------------------------------------------------ 3x3 stride 1, re-tiled weights
HALO_GEOMS = [
    # N, H, W, Cin, Cout  (3x3 stride 1 pad 1)
    (2, 56, 56, 64, 64),       # ResNet-50 stage 1: R = 2 rows per tile
    (2, 28, 28, 128, 128),     # stage 2: R = 4, two 64-channel chunks, BN = 128
    (3, 14, 14, 256, 256),     # stage 3: R = 8 -> tiles of 8 + 6 rows, BN = 64 (weights of a 128-block do not fit)
    (3, 7, 7, 64, 128),        # one image per tile (R = H)
    (1, 20, 12, 64, 192),      # Cout = 192: BN = 64, three channel blocks; H % R != 0
    (5, 6, 6, 128, 128),
    (1, 9, 30, 64, 64),        # R = 4, H = 9: last tile has one valid row
    (2, 5, 126, 64, 64),       # widest supported row: W + 2 = 128, R = 1
    (150, 4, 4, 64, 64),       # more tiles than SMs
]


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", HALO_GEOMS)
def test_conv_halo_requant(geom, a_bits):
    """3x3 stride-1 REQUANT layers with re-tiled weights take the wgmma convolution (conv_igemm.cuh): bit-exact vs the ABI model,
    and the launch counter proves that kernel ran."""
    from hawq_b200 import _lib
    n, h, w, cin, cout = geom
    r = rng(sum(v * (i + 7) for i, v in enumerate(geom)) * 8 + a_bits)
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128 if a_bits == 8 else -8, 128 if a_bits == 8 else 8, size=(cout, 3, 3, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    w_dev = ops.upload_weights(wt, DEV)
    for out_bits, clamp, relu in [(8, (-128, 127), 1), (4, (0, 15), 1), (8, (-128, 127), 0)]:
        chan = make_chan(r, cout, ratio_lo=1e-5)
        d = ops.conv_desc(n, h, w, cin, cout, 3, 3, 1, 1, a_bits)
        ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=TC_FLAG)
        before = _lib.load().hawq_debug_kernel_count(0)
        over = dict(w=w_dev, desc=ops.conv_desc(n, h, w, cin, cout, 3, 3, 1, 1, a_bits, 1))
        (c_out,), (g_out,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(n * h * w * cout, out_bits)), ["out"], over)
        assert _lib.load().hawq_debug_kernel_count(0) == before + 1, "the wgmma convolution did not take this launch"
        assert torch.equal(c_out, g_out), (geom, a_bits, out_bits)
        assert ops.get_status(0) == 0


# ------------------------------------------------------------------------------------------------ 1x1 stride 1
C1_GEOMS = [
    # N, H, W, Cin, Cout
    (3, 57, 57, 256, 64),      # ResNet-50 stage-1 conv1 shape, 77 ragged row tiles, BN = 64
    (2, 28, 28, 512, 128),     # KT = 8: two stages of 4 k-tiles per tile
    (2, 14, 14, 1024, 256),    # KT = 16, two channel blocks
    (3, 7, 7, 2048, 512),      # KT = 32: BN = 64 (a 128-row weight slab does not fit), 8 channel blocks
    (5, 20, 20, 64, 256),      # conv3 shape: single k-tile per tile
    (1, 9, 9, 192, 128),       # KT = 3: KC = 3
    (40, 30, 30, 128, 512),    # 282 row tiles x 4 channel blocks: several tiles per CTA
]


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", C1_GEOMS)
def test_conv1x1_requant_and_residual(geom, a_bits):
    check_conv1x1_requant_and_residual(geom, a_bits)


# ------------------------------------------------------------------------------------------------ resize-unit tails, ResNet-50 shapes
DUALK_GEOMS = [
    # N, Ho, Wo, Cin (last conv), Cin2 (identity conv), Cout, identity stride   (identity input = s * Ho x s * Wo)
    (2, 56, 56, 64, 64, 256, 1),        # ResNet-50 stage 1: 49 row tiles of 128
    (3, 28, 28, 128, 256, 512, 2),      # stage 2: strided identity input, ragged last row tile
    (2, 14, 14, 256, 512, 1024, 2),     # stage 3
    (5, 7, 7, 512, 1024, 2048, 2),      # stage 4: M = 245, half-empty last row tile
    (2, 12, 12, 64, 128, 192, 2),       # Cout = 192 -> BN = 64
    (9, 4, 4, 64, 64, 128, 2),          # eight images per row tile
]


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", DUALK_GEOMS)
def test_conv_dual_stationary_weights(geom, a_bits, flag):
    check_conv_dual_stationary_weights(geom, a_bits, flag)


@pytest.mark.parametrize("shape", [(2, 224, 224), (3, 64, 48), (1, 32, 192), (5, 20, 16), (2, 58, 32)])
def test_stem_pool_fused(shape):
    """hawq_stem_pool_i8 (fused stem: conv + max-pool + 16-bit requant + ReLU + low-bit copy) == hawq_stem_conv_i8 followed by
    hawq_maxpool_requant of the ABI model, for the uint16 and the int32 stream, 8 / 4-bit and no low copy, bands that end inside the image."""
    n, h, w = shape
    r = rng(n * h + 3 * w)
    x = torch.from_numpy(r.randint(-128, 128, size=n * h * w * 3).astype(np.int8))
    wt = torch.zeros((64, 8, 8, 4), dtype=torch.int8)
    wt[:, :7, :7, :3] = torch.from_numpy(r.randint(-128, 128, size=(64, 7, 7, 3)).astype(np.int8))
    chan = make_chan(r, 64, ratio_lo=0.05, ratio_hi=0.8)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    po, qo = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    for y_bits, low_bits, clamp in [(16, 8, (-32768, 32767)), (32, 4, (-32768, 32767)), (16, 0, (-3000, 20000)), (16, 4, (-32768, 32767))]:
        args = dict(x=x, w256=wt, chan=chan, clamp=clamp, n=n, hh=h, ww=w, y_bits=y_bits, y=out_buf(n * po * qo * 64, y_bits),
                    low_bits=low_bits, low_me=dyadic(0.003), low_clamp=(0, 15) if low_bits == 4 else (-128, 127),
                    out_low=out_buf(n * po * qo * 64, low_bits) if low_bits else None)
        keys = ["y"] + (["out_low"] if low_bits else [])
        cs, gs = run_both("stem_pool", args, keys)
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (shape, y_bits, low_bits, k_, int((a != b).sum()))
    assert ops.get_status(0) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(5, 20, 12), (2, 58, 36), (1, 16, 272)])
def test_stem_pool_declines_shapes_outside_the_kernel(shape):
    """Row pitches that are not a multiple of 16 bytes and rows wider than 256 pixels are outside the fused stem's envelope: hawq_stem_pool_i8
    answers HAWQ_ERR_UNSUPPORTED without launching anything (the host then runs hawq_stem_conv_i8 + hawq_maxpool_requant)."""
    from hawq_b200._lib import HawqError, ERR_UNSUPPORTED
    n, h, w = shape
    r = rng(7)
    x = torch.from_numpy(r.randint(-128, 128, size=n * h * w * 3).astype(np.int8)).cuda()
    wt = torch.zeros((64, 8, 8, 4), dtype=torch.int8).cuda()
    chan = make_chan(r, 64, ratio_lo=0.05, ratio_hi=0.8).cuda()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    po, qo = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    y = torch.zeros(n * po * qo * 64, dtype=torch.int16, device="cuda")
    with pytest.raises(HawqError) as err:
        ops.stem_pool(x, wt, chan, (-32768, 32767), n, h, w, 16, y, 0, (0, 1), (0, 0), None)
    assert err.value.code == ERR_UNSUPPORTED
    assert int(y.abs().max()) == 0


# ------------------------------------------------------------------------------------------------ int32 and ratio boundaries
BOUNDARY_GEOMS = [
    # N, H, W, Cin, Cout, kh, kw, stride, pad: ragged last row tile in each
    (3, 6, 6, 64, 320, 3, 3, 1, 1),       # BN = 64: five column blocks, M = 108
    (3, 5, 5, 512, 512, 3, 3, 1, 1),      # BN = 128, K = 4608 (72 k-tiles), M = 75
    (3, 9, 9, 128, 512, 1, 1, 1, 0),      # 1x1, M = 243: two row tiles
]


@pytest.mark.parametrize("flags", [0, 1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", BOUNDARY_GEOMS)
def test_conv_epilogue_boundaries(geom, a_bits, flags):
    check_conv_epilogue_boundaries(geom, a_bits, flags)


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("cout", [320, 512])
def test_conv_dual_boundaries(cout, a_bits, flag):
    """hawq_conv2d_dual with saturating biases on both convolutions, identity ratios 0.5 / 0.25 (ties on negative operands) and the
    ratio edges of boundary_weights_chan on the main convolution."""
    n, ho, wo, cin, cin2, s2 = 3, 7, 7, 128, 64, 2                  # M = 147: ragged last row tile
    r = rng(555 + cout + 7 * a_bits + flag)
    h2, w2 = ho * s2, wo * s2
    numel = n * ho * wo * cout
    bn = 128 if cout % 128 == 0 else 64
    x = extreme_act(r, n, ho * wo, cin, a_bits)
    x2 = extreme_act(r, n, h2 * w2, cin2, a_bits)
    wt, chan = boundary_weights_chan(r, cout, bn, 1, 1, cin, a_bits)
    wt2, _ = boundary_weights_chan(r, cout, bn, 1, 1, cin2, a_bits)
    edges = edge_biases(cin2, a_bits)
    ties = res_chan_with_ties(r, cout)
    chan2 = ties.clone()
    chan2[:, 0] = torch.tensor([edges[c % 8] if (c // bn) % 2 else int(r.randint(-3000, 3001)) for c in range(cout)], dtype=torch.int32)
    d = ops.conv_desc(n, ho, wo, cin, cout, 1, 1, 1, 0, a_bits, 1)
    d2 = ops.conv_desc(n, h2, w2, cin2, cout, 1, 1, s2, 0, a_bits, 1)
    wg, wg2 = ops.upload_weights(wt, DEV), ops.upload_weights(wt2, DEV)
    for low_bits in (8, 4, 0):
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, low_bits=low_bits, low_me=dyadic(0.003),
                          low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flag)
        args = dict(x=x, desc=d, ep=ep, w=wt, chan=chan, desc2=d2, x2=x2, w2=wt2, chan2=chan2, out=out_buf(numel, 16),
                    out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = ["out"] + (["out_low"] if low_bits else [])
        cs, gs = run_both("conv2d_dual", args, keys, gpu_overrides=dict(w=wg, w2=wg2))
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (cout, a_bits, flag, low_bits, k_, int((a != b).sum()))


@pytest.mark.parametrize("a_bits", [8, 4])
def test_rows_past_m_raise_no_flag(a_bits):
    """Rows of a ragged tile past M are zero-filled, so there acc = 0 and v = bias.  With acc = -bias on every real row and a
    ratio of 2^17, a zero-filled row would leave int32 (HAWQ_FLAG_REQUANT_OVERFLOW) and, for int8 inputs, exceed the uint16
    stream (HAWQ_FLAG_RESIDUAL_OVERFLOW) if it were counted; the real rows stay 0 + residual."""
    n, h, w, cin, cout = 1, 9, 9, 64, 128                              # M = 81 < one row tile
    numel = n * h * w * cout
    x = torch.full((n * h * w * cin // (2 if a_bits == 4 else 1),), 0xFF if a_bits == 4 else -128,
                   dtype=torch.uint8 if a_bits == 4 else torch.int8)
    wt = torch.full((cout, 1, 1, cin), 127, dtype=torch.int8)
    acc = cin * (15 if a_bits == 4 else -128) * 127
    chan = ops.make_chan([-acc] * cout, [2 ** 31] * cout, [14] * cout)
    d = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, a_bits)
    r = rng(a_bits)
    res16 = torch.from_numpy(r.randint(0, 65536, size=numel).astype(np.uint16).view(np.int16))
    res32 = rand_act(r, numel, 32)
    for flags in (0, 1, 2):
        for res, res_bits, y_bits, low_bits in [(res16, 16, 16, 8), (res32, 32, 32, 4)]:
            ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=res_bits, res_me=RATIO_ONE, y_bits=y_bits, low_bits=low_bits,
                              low_me=dyadic(0.003), low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flags)
            cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, out=out_buf(numel, y_bits),
                                             out_low=out_buf(numel, low_bits)), ["out", "out_low"])
            assert am.status["flags"] == 0
            for a, b in zip(cs, gs):
                assert torch.equal(a, b), (a_bits, flags, y_bits)
        if flags:   # the resize-unit kernel: identity operand 0 on every row
            x2 = torch.zeros_like(x)
            w2 = torch.zeros((cout, 1, 1, cin), dtype=torch.int8)
            chan2 = ops.make_chan([0] * cout, [2 ** 30] * cout, [31] * cout)
            dd = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, a_bits, 1)
            ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, low_bits=8, low_me=dyadic(0.003),
                              low_clamp=(-128, 127), flags=flags)
            args = dict(x=x, desc=dd, ep=ep, w=wt, chan=chan, desc2=dd, x2=x2, w2=w2, chan2=chan2, out=out_buf(numel, 16),
                        out_low=out_buf(numel, 8))
            cs, gs = run_both("conv2d_dual", args, ["out", "out_low"],
                              gpu_overrides=dict(w=ops.upload_weights(wt, DEV), w2=ops.upload_weights(w2, DEV)))
            assert am.status["flags"] == 0
            for a, b in zip(cs, gs):
                assert torch.equal(a, b), (a_bits, flags, "dual")


@pytest.mark.parametrize("flags", [0, 1])
def test_residual_stream_lands_on_65535_and_65536(flags):
    """y = r + bias exactly (zero weights, both ratios exactly 1): 65535 fits the uint16 stream, 65536 raises
    HAWQ_FLAG_RESIDUAL_OVERFLOW and is stored as 65535."""
    n, h, w, cin, cout = 2, 9, 9, 64, 128                              # M = 162: one full and one ragged row tile
    numel = n * h * w * cout
    r = rng(65535 + flags)
    x = rand_act(r, n * h * w * cin, 8)
    wt = torch.zeros((cout, 1, 1, cin), dtype=torch.int8)
    bias = r.randint(1, 30000, size=cout)
    chan = ops.make_chan(bias, [2 ** 31] * cout, [31] * cout)
    d = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, 8)
    for y, flag in [(65535, 0), (65536, 1)]:
        res = torch.from_numpy(np.tile(y - bias, n * h * w).astype(np.uint16).view(np.int16))
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=16, res_me=RATIO_ONE, y_bits=16, low_bits=8, low_me=dyadic(0.003),
                          low_clamp=(-128, 127), flags=flags)
        cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, out=out_buf(numel, 16), out_low=out_buf(numel, 8)),
                          ["out", "out_low"])
        assert am.status["flags"] == flag
        assert int((cs[0].to(torch.int32) & 0xFFFF).min()) == 65535
        for a, b in zip(cs, gs):
            assert torch.equal(a, b), (flags, y)


@pytest.mark.parametrize("shape", [(130, 512, 999, 1024), (67, 192, 127, 128)])
def test_linear_bias_edges(shape):
    """DEQUANT_F32 tail at saturating biases and odd cout_store: the dp4a kernel (K % 128 == 0) and the convolution (other K)."""
    nb, kk, co, cp = shape
    r = rng(17 + nb + kk)
    x = r.randint(-128, 128, size=(nb, kk))
    x[0::3] = -128
    x[1::3] = 127
    wl = r.randint(-128, 128, size=(cp, kk))
    for c in range(cp):
        row = (-128, 127, -127, None)[(c // 8) % 4]
        if row is not None:
            wl[c] = row
    wl[co:] = 0
    edges = edge_biases(kk, 8)
    chl = ops.make_chan([edges[c % 8] for c in range(cp)], [2 ** 30] * cp, [40] * cp)
    fs = torch.from_numpy(r.uniform(1e-5, 1e-3, size=cp).astype(np.float32))
    (c,), (g,) = run_both("linear", dict(x=torch.from_numpy(x.reshape(-1).astype(np.int8)), w=torch.from_numpy(wl.astype(np.int8)), chan=chl,
                                         fscale=fs, out=torch.zeros((nb, co)), n=nb, k=kk, cout=co, cout_pad=cp), ["out"])
    assert torch.equal(c, g), shape


def test_requant_and_add_requant_stage1_bias_edges():
    """requant / add_requant at ResNet-50 stage-1 size (batch 8, 56 x 56 x 256: the grid-stride loops run several times) with
    int32-limit accumulators and biases."""
    r = rng(56)
    rows, ch = 8 * 56 * 56, 256
    edges = [I32_MIN, I32_MIN + 1, I32_MAX, I32_MAX - 1, 2 ** 30, -2 ** 30, 0, 1]
    me = [RATIO_ONE if c % 5 == 0 else dyadic([0.5, 0.25, 1.0, 3.0][c % 4] if c % 5 == 1 else float(np.exp(r.uniform(np.log(1e-9), 0.0))))
          for c in range(ch)]
    chan = ops.make_chan([edges[c % 8] if c % 2 else int(r.randint(-2 ** 20, 2 ** 20)) for c in range(ch)], [m for m, _ in me],
                         [e for _, e in me])
    acc = torch.from_numpy(r.randint(I32_MIN, I32_MAX, size=rows * ch, dtype=np.int64).astype(np.int32))
    acc[:ch], acc[ch:2 * ch] = I32_MIN, I32_MAX
    for x_bits, relu, out_bits in [(32, 1, 8), (32, 0, 16), (16, 1, 4), (32, 0, 8)]:
        x = acc if x_bits == 32 else rand_act(r, rows * ch, 16)
        clamp = {4: (0, 15), 8: (-128, 127), 16: (-32768, 32767)}[out_bits]
        (a,), (b,) = run_both("requant", dict(x=x, rows=rows, c=ch, x_bits=x_bits, chan=chan, chan_stride=1, relu=relu, out_bits=out_bits,
                                              clamp=clamp, out=out_buf(rows * ch, out_bits)), ["out"])
        assert torch.equal(a, b), (x_bits, relu, out_bits)
    res_chan = res_chan_with_ties(r, ch)
    for res_kind, res_bits, y_bits, low_bits in [(0, 16, 16, 8), (1, 32, 32, 4), (0, 32, 16, 0), (1, 32, 16, 8)]:
        if res_bits == 16:
            res = torch.from_numpy(r.randint(0, 65536, size=rows * ch).astype(np.uint16).view(np.int16))
        else:
            res = torch.from_numpy(r.randint(I32_MIN, I32_MAX, size=rows * ch, dtype=np.int64).astype(np.int32))
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=res_kind, res_bits=res_bits, res_me=dyadic(0.6), y_bits=y_bits, low_bits=low_bits,
                          low_me=dyadic(0.002), low_clamp=(0, 15) if low_bits == 4 else (-128, 127))
        args = dict(acc=acc, rows=rows, c=ch, chan=chan, ep=ep, res=res, res_chan=res_chan if res_kind else None,
                    y=out_buf(rows * ch, y_bits), out_low=out_buf(rows * ch, low_bits) if low_bits else None)
        keys = [k for k in ("y", "out_low") if args[k] is not None]
        cs, gs = run_both("add_requant", args, keys)
        for a, b, k in zip(cs, gs, keys):
            assert torch.equal(a, b), (res_kind, res_bits, y_bits, low_bits, k)
