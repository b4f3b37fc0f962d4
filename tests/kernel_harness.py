"""The kernel-parity harness of the GPU tests: seeded inputs, channel tables and edge cases, run_both (the numpy ABI model and the
library on the same buffers, bit-exact), and the check_* parity checks that several test modules run at their own geometries.  Its
ratio constants come from oracle.int_ref.dyadic (the library's pairs), so that importing it needs neither the GPU nor the library."""
import numpy as np
import torch

from hawq_b200 import _lib, ops
from hawq_b200._lib import EPI_DEQUANT_F32, EPI_RAW_I32, EPI_REQUANT, EPI_RESIDUAL, hawq_conv_desc
from oracle.int_ref import dyadic
from tests import abi_model as am
from tests.util import guarded_call

DEV = "cuda:0"


def rng(seed):
    return np.random.RandomState(seed)


def make_chan(r, c, bias_mag=2 ** 16, ratio_lo=1e-4, ratio_hi=0.05):
    bias = r.randint(-bias_mag, bias_mag, size=c)
    me = [dyadic(float(np.exp(r.uniform(np.log(ratio_lo), np.log(ratio_hi))))) for _ in range(c)]
    return ops.make_chan(bias, [m for m, _ in me], [e for _, e in me])


def rand_act(r, n_vals, bits, signed=True):
    if bits == 4:
        v = r.randint(0, 16, size=n_vals)
        return torch.from_numpy(am.pack_i4(v))
    if bits == 8:
        return torch.from_numpy(r.randint(-128, 128, size=n_vals).astype(np.int8))
    if bits == 16:
        return torch.from_numpy(r.randint(0, 40000, size=n_vals).astype(np.uint16).view(np.int16))
    return torch.from_numpy(r.randint(-40000, 40000, size=n_vals).astype(np.int32))


def out_buf(numel, bits):
    dt = {4: torch.uint8, 8: torch.int8, 16: torch.int16, 32: torch.int32}[bits]
    return torch.zeros(numel // 2 if bits == 4 else numel, dtype=dt)


def widest_row_bytes(args):
    """bytes of the widest row a call touches, at 4 bytes per element: a convolution row is Cin or Cout channels"""
    dims = [v for d in args.values() if isinstance(d, hawq_conv_desc) for v in (d.Cin, d.Cout)]
    return 4 * max(dims + [args[k] for k in ("c", "k", "cout_pad") if k in args] + [64])


def run_both(fn_name, cpu_args, out_keys, gpu_overrides=None):
    """cpu_args: dict of kwargs with CPU tensors; out_keys: names of output tensors.  Returns (cpu_outs, gpu_outs).
    The model runs first.  The library then runs with every tensor in a guarded, poisoned allocation (tests/util.guarded_call):
    its outputs must equal the model's byte for byte, every output byte must be written, and no guard byte, input or unused
    buffer may change.  Both status words start at 0, and the library's must equal the model's after the call."""
    ops.reset_status(0)
    am.status["flags"] = 0
    getattr(am, fn_name)(**cpu_args)
    args = dict(cpu_args, **(gpu_overrides or {}))
    outs, problems = guarded_call(getattr(ops, fn_name), args, {k: cpu_args[k] for k in out_keys}, DEV, 128 * widest_row_bytes(args))
    assert ops.get_status(0) == am.status["flags"], (fn_name, ops.get_status(0), am.status["flags"])
    assert not problems, (fn_name, problems)
    return [cpu_args[k] for k in out_keys], [outs[k].cpu() for k in out_keys]


def out_hw(h, w, kh, kw, s, p):
    return (h + 2 * p - kh) // s + 1, (w + 2 * p - kw) // s + 1


TC_FLAG = 1   # HAWQ_EP_RATIOS_LE_ONE: the ratio promise the engine makes for every HAWQ ResNet layer


def sm_count():
    return _lib.load().hawq_sm_count(ops.handle(0))


def kernel_count(family):
    """launches taken so far by the kernel family `family` of hawq_debug_kernel_count"""
    return _lib.load().hawq_debug_kernel_count(family)


BN = 64   # the tail kernel's channel block


def row_tile_stride(cout):
    """row tiles between the consecutive tiles of one CTA: the grid is two CTAs per SM, a multiple of Cout / 64"""
    return max(1, 2 * sm_count() // (cout // BN))


def images_for_three_tiles(pixels_per_image, cout):
    """the smallest batch of pixels_per_image output pixels per image whose row tiles give every CTA of the tail kernel at least
    three, the last one ragged"""
    n = 1
    while -(-n * pixels_per_image // 128) < 3 * row_tile_stride(cout) or n * pixels_per_image % 128 == 0:
        n += 1
    return n


# ------------------------------------------------------------------------------------------------ int32 and ratio boundaries
# Each CTA of conv_igemm.cuh picks its requantisation: FP64 (the bias folded into the int -> double conversion, one FMA per term)
# when every ratio is <= 1, or for RESIDUAL under a ratio promise when every ratio is <= 2^20 (each term then range-checked); the
# exact 64-bit form otherwise.  An FP64 CTA with a bias that can take acc + bias out of int32 clamps that sum.  These tests put
# accumulators, biases and ratios on those limits, side by side with ordinary channels in neighbouring column blocks, and demand
# whole outputs and the status word equal to the ABI model.
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
RATIO_ONE = (2 ** 31, 31)           # exactly 1 in the FP64 form (dyadic(1.0) is (2^30, 30))
WIDE_RATIOS = [dyadic(1.0), dyadic(1 + 2 ** -20), (2 ** 31, 11), dyadic(3.0), dyadic(1000.0)]   # (1, 2^20], 2^20 exactly
GENERIC_RATIOS = [(2 ** 30 + 1, 10), (2 ** 31, 10), (0, 31), RATIO_ONE]                         # above 2^20, m = 0, 1


def bias_window(k, a_bits):
    """the biases for which acc + bias cannot leave int32: |acc| <= K * 128 * 128 (int8) or K * 15 * 128 (unsigned 4-bit)"""
    b = min(k * (15 if a_bits == 4 else 128) * 128, 2 ** 31)
    return b - 2 ** 31, 2 ** 31 - 1 - b


def edge_biases(k, a_bits):
    lo, hi = bias_window(k, a_bits)
    return [I32_MIN, I32_MIN + 1, I32_MAX, lo - 1, lo, hi, hi + 1, 0]


def extreme_act(r, n, pix, c, a_bits):
    """image i % 3 == 0: every value -128 (4-bit: 15); 1: 127 (4-bit: 0); 2: random.  With a constant weight row, the outputs of
    the first two images whose window lies inside the image reach acc = K * x * w exactly (K * 128 * 128 for x = w = -128)."""
    consts = (-128, 127) if a_bits == 8 else (15, 0)
    v = r.randint(-128, 128, size=(n, pix * c)) if a_bits == 8 else r.randint(0, 16, size=(n, pix * c))
    for i in range(n):
        if i % 3 < 2:
            v[i] = consts[i % 3]
    v = v.reshape(-1)
    return torch.from_numpy(am.pack_i4(v)) if a_bits == 4 else torch.from_numpy(v.astype(np.int8))


def boundary_weights_chan(r, cout, bn, kh, kw, cin, a_bits):
    """Column block b (BN channels) by b % 4:
      0: random weights, |bias| <= 2^16, ratios <= 1 (0.5 and 0.25 give round-half-even ties): FP64;
      1: bias edges (int32 limits, both sides of the bias window, 0) on constant weight rows -128 / 127 / -127 and random rows,
         ratios <= 1 (1 exactly, 5e-8, m = 0, log-uniform down to 1e-9);
      2: as 1, plus zero-weight channels with a small bias and a ratio in (1, 2^20] (FP64, clamped and checked, under a promise);
      3: as 0, plus zero-weight channels with a small bias and a ratio above 2^20, m = 0 or exactly 1 (the exact 64-bit form).
    Zero-weight channels keep |bias| <= 1000, so that no term leaves int32 at ratios up to 2^21."""
    k = kh * kw * cin
    edges = edge_biases(k, a_bits)
    w = r.randint(-128, 128, size=(cout, kh, kw, cin))
    bias, me = [], []
    for c in range(cout):
        kind, j = (c // bn) % 4, c % bn
        if kind in (0, 3):
            b = int(r.randint(-2 ** 16, 2 ** 16))
            ratio = [0.5, 0.25][j % 2] if j % 4 < 2 else float(np.exp(r.uniform(np.log(1e-5), 0.0)))
            mc = dyadic(ratio)
        else:
            b = edges[j % 8]
            row = (-128, 127, -127, None)[(j // 8) % 4]
            if row is not None:
                w[c] = row
            mc = [RATIO_ONE, dyadic(5e-8), (0, 31), None, None][j % 5] or dyadic(float(np.exp(r.uniform(np.log(1e-9), 0.0))))
        if (kind == 2 and j % 16 == 15) or (kind == 3 and j % 8 == 7):
            ratios = WIDE_RATIOS if kind == 2 else GENERIC_RATIOS
            w[c] = 0
            b = int(r.randint(-1000, 1001))
            mc = ratios[(j // 16 if kind == 2 else j // 8) % len(ratios)]
        bias.append(b)
        me.append(mc)
    wt = torch.from_numpy(w.astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    return wt, ops.make_chan(bias, [m for m, _ in me], [e for _, e in me])


def res_chan_with_ties(r, cout):
    """per-channel ratios of a res_kind 1 operand: 0.5 and 0.25 (ties on every odd operand, negative ones included), else <= 1"""
    me = [dyadic([0.5, 0.25][c % 2] if c % 4 < 2 else float(np.exp(r.uniform(np.log(1e-3), 0.0)))) for c in range(cout)]
    return ops.make_chan([0] * cout, [m for m, _ in me], [e for _, e in me])


REQUANT_CASES = [(out_bits, clamp, relu) for out_bits, clamp in [(4, (0, 15)), (8, (-128, 127)), (16, (-32768, 32767)), (32, (I32_MIN, I32_MAX))]
                 for relu in (0, 1)] + [(8, (-128, -5), 1),   # ReLU with clamp_hi < 0: every output is clamp_hi
                                        (8, (-128, 0), 1)]    # ReLU with clamp_hi = 0: every output byte is 0
RESIDUAL_CASES = [  # res_kind, res_bits, y_bits, low_bits, relu
    (0, 16, 16, 8, 1), (0, 32, 32, 4, 1), (0, 32, 32, 0, 0), (0, 16, 0, 4, 1), (1, 32, 16, 4, 1), (1, 32, 0, 8, 1), (1, 32, 32, 0, 0)]


# ------------------------------------------------------------------------------------------------ MobileNetV2 inputs and channels
# (a_bits, value range of the input, out_bits, clamp): int8, 4-bit values in byte containers, packed nibbles
IO = [(8, "s8", 8, (-128, 127)), (8, "u4", 8, (0, 15)), (4, "u4", 4, (0, 15)), (8, "s8", 4, (0, 15)), (4, "u4", 8, (-128, 127))]


def act_in(r, n_vals, kind, a_bits):
    if a_bits == 4:
        return rand_act(r, n_vals, 4)
    lo, hi = (-128, 128) if kind == "s8" else (0, 16)
    return torch.from_numpy(r.randint(lo, hi, size=n_vals).astype(np.int8))


def chan_for(r, c, ratio_hi, clamp, caps, bias_span=3000, saturate=False):
    """ratios in [1e-4, ratio_hi] (> 1 takes the exact requantisation); caps: 'some' bind on every third channel, 'none' = hi."""
    me = [dyadic(float(np.exp(r.uniform(np.log(1e-4), np.log(ratio_hi))))) for _ in range(c)]
    bias = r.randint(-bias_span, bias_span, size=c).astype(np.int64)
    if saturate:                                           # acc + bias leaves int32 on some channels
        bias[::5] = 2 ** 31 - 1 - r.randint(0, 1000, size=len(bias[::5]))
        bias[1::5] = -2 ** 31 + r.randint(0, 1000, size=len(bias[1::5]))
    lo, hi = clamp
    cap = np.full(c, hi, dtype=np.int64)
    if caps == "some":
        cap[::3] = r.randint(min(max(lo, 0), hi), hi + 1, size=len(cap[::3]))
    return ops.make_chan(bias, [m for m, _ in me], [e for _, e in me], cap)


def pow2_chan(r, c):
    """Power-of-two ratios 2^-k (m = 2^30, e = 30 + k): with relu 0 negative accumulators land on RHE ties."""
    k = r.randint(1, 12, size=c)
    return ops.make_chan(r.randint(-64, 64, size=c) * 2 ** 6, [2 ** 30] * c, list(30 + k), [2 ** 31 - 1] * c)


def dw_rect(r, n, hh, ww, c, stride, io, variant):
    """variant 0: random data, ReLU6 caps on some channels; 1: power-of-two ratios, relu 0; 2: x = w = -128 (int8 inputs; 15 in a
    4-bit input), power-of-two ratios, relu 0."""
    a_bits, kind, out_bits, clamp = io
    ho, wo = (hh - 1) // stride + 1, (ww - 1) // stride + 1
    if variant == 2:
        v = -128 if kind == "s8" else 15
        x = torch.full((n * hh * ww * c,), v, dtype=torch.int8) if a_bits == 8 else torch.from_numpy(am.pack_i4(np.full(n * hh * ww * c, 15)))
        w = torch.full((3, 3, c), -128, dtype=torch.int8)
    else:
        x = act_in(r, n * hh * ww * c, kind, a_bits)
        w = torch.from_numpy(r.randint(-128, 128, size=(3, 3, c)).astype(np.int8))
    relu = 2 if variant == 0 else 0
    chan = chan_for(r, c, 0.9, clamp, "some") if variant == 0 else pow2_chan(r, c)
    args = dict(x=x, n=n, hh=hh, ww=ww, c=c, stride=stride, a_bits=a_bits, w=w, chan=chan, relu=relu, out_bits=out_bits, clamp=clamp,
                out=out_buf(n * ho * wo * c, out_bits))
    (cm,), (g,) = run_both("dwconv3x3", args, ["out"])
    assert torch.equal(cm, g), (n, hh, ww, c, stride, io, variant)


# ------------------------------------------------------------------------------------------------ parity checks run at several geometries
def check_conv_requant(geom, a_bits, tc):
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = rng(sum(v * (i + 3) for i, v in enumerate(geom)) * 8 + a_bits)
    ho, wo = out_hw(h, w, kh, kw, s, p)
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128 if a_bits == 8 else -8, 128 if a_bits == 8 else 8, size=(cout, kh, kw, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    for out_bits, clamp, relu in [(8, (-128, 127), 1), (4, (0, 15), 1), (16, (-32768, 32767), 0), (32, (-2 ** 31, 2 ** 31 - 1), 0)]:
        chan = make_chan(r, cout, ratio_lo=1e-5 if out_bits <= 8 else 1e-3)
        d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits)
        ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=TC_FLAG * tc)
        over = None
        if tc and DEV != "cpu" and (n + h) % 2 == 0:   # half of the geometries: weights re-tiled for linear bulk loads (w_layout = 1)
            over = dict(w=ops.upload_weights(wt, DEV), desc=ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits, 1))
        (c_out,), (g_out,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(n * ho * wo * cout, out_bits)), ["out"], over)
        assert torch.equal(c_out, g_out), (geom, a_bits, out_bits, tc)


def check_conv_residual(geom, a_bits, tc):
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = rng(sum(v * (i + 5) for i, v in enumerate(geom)) * 8 + a_bits + 1)
    ho, wo = out_hw(h, w, kh, kw, s, p)
    numel = n * ho * wo * cout
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, kh, kw, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    chan = make_chan(r, cout, ratio_lo=1e-2, ratio_hi=0.9)
    d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits)
    low_me = dyadic(0.004)
    for res_kind, res_bits, y_bits, low_bits, relu in [(0, 32, 32, 8, 1), (0, 16, 16, 4, 1), (1, 32, 32, 4, 1),
                                                       (0, 32, 32, 0, 0), (1, 32, 0, 8, 1), (0, 16, 16, 8, 1)]:
        res = rand_act(r, numel, res_bits if res_kind == 0 else 32)
        res_chan = make_chan(r, cout, ratio_lo=1e-2, ratio_hi=0.9) if res_kind == 1 else None
        res_me = dyadic(0.37)
        ep = ops.epilogue(EPI_RESIDUAL, relu=relu, res_kind=res_kind, res_bits=res_bits, res_me=res_me, y_bits=y_bits,
                          low_bits=low_bits, low_me=low_me, low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=TC_FLAG * tc)
        args = dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=res, res_chan=res_chan,
                    out=out_buf(numel, y_bits) if y_bits else None, out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = [k_ for k_ in ("out", "out_low") if args[k_] is not None]
        c_outs, g_outs = run_both("conv2d", args, keys)
        for a, b, k_ in zip(c_outs, g_outs, keys):
            assert torch.equal(a, b), (geom, a_bits, res_kind, res_bits, y_bits, low_bits, k_, tc)


def check_conv_raw_and_dequant_geoms(geom, a_bits):
    """RAW_I32, and DEQUANT_F32 with an odd cout_store below Cout (rows of cout_store floats; the last column block is stored in
    part), over ragged 3x3, strided and BN = 64 geometries with 8- and 4-bit inputs."""
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = rng(1303 + sum(v * (i + 3) for i, v in enumerate(geom)) * 8 + a_bits)
    ho, wo = out_hw(h, w, kh, kw, s, p)
    m = n * ho * wo
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128, 128, size=(cout, kh, kw, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    chan = make_chan(r, cout, bias_mag=2 ** 20)
    d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits)
    (c,), (g,) = run_both("conv2d", dict(x=x, desc=d, ep=ops.epilogue(EPI_RAW_I32, flags=TC_FLAG), w=wt, chan=chan, out=out_buf(m * cout, 32)),
                          ["out"])
    assert torch.equal(c, g), (geom, a_bits)
    cs = cout - 63
    fs = torch.from_numpy(r.uniform(1e-5, 1e-3, size=cout).astype(np.float32))
    (c,), (g,) = run_both("conv2d", dict(x=x, desc=d, ep=ops.epilogue(EPI_DEQUANT_F32, cout_store=cs), w=wt, chan=chan, fscale=fs,
                                         out=torch.zeros(m * cs)), ["out"])
    assert torch.equal(c.view(torch.int32), g.view(torch.int32)), (geom, a_bits)


def check_stem_and_pool(shape):
    n, h, w = shape
    r = rng(n * h + w)
    x = torch.from_numpy(r.randint(-128, 128, size=n * h * w * 3).astype(np.int8))
    wt = torch.zeros((64, 7, 8, 4), dtype=torch.int8)
    wt[:, :, :7, :3] = torch.from_numpy(r.randint(-128, 128, size=(64, 7, 7, 3)).astype(np.int8))
    chan = make_chan(r, 64, ratio_lo=0.05, ratio_hi=0.8)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    (c16,), (g16,) = run_both("stem_conv", dict(x=x, w=wt, chan=chan, clamp=(-32768, 32767), out=torch.zeros(n * ho * wo * 64, dtype=torch.int16),
                                                n=n, hh=h, ww=w), ["out"])
    assert torch.equal(c16, g16)
    po, qo = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    for y_bits, low_bits in [(16, 8), (32, 4), (16, 0), (0, 8)]:
        args = dict(x=c16, n=n, hh=ho, ww=wo, c=64, y_bits=y_bits, y=out_buf(n * po * qo * 64, y_bits) if y_bits else None,
                    low_bits=low_bits, low_me=dyadic(0.003), low_clamp=(0, 15) if low_bits == 4 else (-128, 127),
                    out_low=out_buf(n * po * qo * 64, low_bits) if low_bits else None)
        keys = [k for k in ("y", "out_low") if args[k] is not None]
        cs, gs = run_both("maxpool_requant", args, keys)
        for a, b in zip(cs, gs):
            assert torch.equal(a, b), (shape, y_bits, low_bits)


def check_conv1x1_requant_and_residual(geom, a_bits):
    """1x1 stride-1 layers take the wgmma convolution (conv_igemm.cuh) for the REQUANT and the uint16-stream RESIDUAL epilogues
    (ratios <= 1 and the checked <= 2^20 variant): bit-exact vs the ABI model; the launch counter proves which kernel ran."""
    from hawq_b200 import _lib
    n, h, w, cin, cout = geom
    r = rng(sum(v * (i + 11) for i, v in enumerate(geom)) * 8 + a_bits)
    numel = n * h * w * cout
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128 if a_bits == 8 else -8, 128 if a_bits == 8 else 8, size=(cout, 1, 1, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    d = ops.conv_desc(n, h, w, cin, cout, 1, 1, 1, 0, a_bits)
    count = lambda: _lib.load().hawq_debug_kernel_count(0)
    for out_bits, clamp, relu in [(8, (-128, 127), 1), (4, (0, 15), 1), (8, (-128, 127), 0), (8, (-100, 90), 1)]:
        chan = make_chan(r, cout, ratio_lo=1e-5)
        ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=TC_FLAG)
        before = count()
        (c_out,), (g_out,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(numel, out_bits)), ["out"])
        assert count() == before + 1, "the wgmma convolution did not take this REQUANT launch"
        assert torch.equal(c_out, g_out), (geom, a_bits, out_bits, relu)
    wt2 = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt2)
    for flag, low_bits, ratio_hi, res_ratio in [(1, 8, 0.9, 0.37), (1, 4, 0.9, 0.9), (1, 0, 0.5, 0.11), (2, 8, 40.0, 1.37), (2, 4, 3.0, 2.5)]:
        chan = make_chan(r, cout, bias_mag=2000, ratio_lo=1e-2, ratio_hi=ratio_hi)
        res = torch.from_numpy(r.randint(0, 900 if flag == 2 else 40000, size=numel).astype(np.uint16).view(np.int16))
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=16, res_me=dyadic(res_ratio), y_bits=16, low_bits=low_bits,
                          low_me=dyadic(0.004 if flag == 1 else 0.0004), low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flag)
        args = dict(x=x, desc=d, ep=ep, w=wt2, chan=chan, res=res, out=out_buf(numel, 16), out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = [k_ for k_ in ("out", "out_low") if args[k_] is not None]
        before = count()
        cs, gs = run_both("conv2d", args, keys)
        assert count() == before + 1, "the wgmma convolution did not take this RESIDUAL launch"
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (geom, a_bits, flag, low_bits, k_)


def check_conv_dual_stationary_weights(geom, a_bits, flag):
    """Resize-unit tails take the one-kernel dual convolution (hawq_debug_kernel_count family 4, hawq_conv2d_dual): bit-exact vs
    RAW_I32 identity conv + res_kind-1 RESIDUAL conv of the ABI model."""
    from hawq_b200 import _lib
    n, ho, wo, cin, cin2, cout, s2 = geom
    r = rng(31337 + sum(v * (i + 3) for i, v in enumerate(geom)) * 4 + flag + a_bits)
    h2, w2 = ho * s2, wo * s2
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
        before = _lib.load().hawq_debug_kernel_count(4)
        cs, gs = run_both("conv2d_dual", args, keys, gpu_overrides=dict(w=wg, w2=wg2))
        assert _lib.load().hawq_debug_kernel_count(4) == before + 1, "conv_dual did not take this launch"
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (geom, a_bits, flag, low_bits, k_)


def check_conv_epilogue_boundaries(geom, a_bits, flags):
    """Every conv2d epilogue at saturating biases and ratio edges, under each ratio promise (flags 1 with ratios above 1 is a broken
    promise: the output must still be exact)."""
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = rng(2024 + sum(v * (i + 3) for i, v in enumerate(geom)) * 8 + a_bits + 97 * flags)
    ho, wo = out_hw(h, w, kh, kw, s, p)
    numel = n * ho * wo * cout
    x = extreme_act(r, n, h * w, cin, a_bits)
    wt, chan = boundary_weights_chan(r, cout, 128 if cout % 128 == 0 else 64, kh, kw, cin, a_bits)
    d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits)
    failed = []   # every epilogue is checked; the assertion at the end names all that differ

    def check(ep, what, **bufs):
        keys = [k_ for k_ in ("out", "out_low") if bufs.get(k_) is not None]
        try:
            cs, gs = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, **bufs), keys)
        except AssertionError as mismatch:   # status word, output bytes, guards or inputs
            failed.append((what, str(mismatch)))
            return
        for a, b, k_ in zip(cs, gs, keys):
            if not torch.equal(a, b):
                failed.append((what, k_, int((a != b).sum())))

    for out_bits, clamp, relu in REQUANT_CASES:
        check(ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=flags), ("requant", out_bits, clamp, relu),
              out=out_buf(numel, out_bits))
    res_chan = res_chan_with_ties(r, cout)
    for res_kind, res_bits, y_bits, low_bits, relu in RESIDUAL_CASES:
        for res_ratio in (0.37, 1.37):
            if res_bits == 16:
                res = torch.from_numpy(r.randint(0, 65536, size=numel).astype(np.uint16).view(np.int16))
            elif res_kind == 1 or res_ratio < 1:   # full int32 range: every term stays inside int32 at ratios <= 1
                res = torch.from_numpy(r.randint(I32_MIN, I32_MAX, size=numel, dtype=np.int64).astype(np.int32))
                res[:cout] = I32_MIN
                res[cout:2 * cout] = I32_MAX
            else:
                res = rand_act(r, numel, 32)
            ep = ops.epilogue(EPI_RESIDUAL, relu=relu, res_kind=res_kind, res_bits=res_bits, res_me=dyadic(res_ratio), y_bits=y_bits,
                              low_bits=low_bits, low_me=dyadic(0.004), low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flags)
            check(ep, ("residual", res_kind, res_bits, y_bits, low_bits, res_ratio), res=res, res_chan=res_chan if res_kind else None,
                  out=out_buf(numel, y_bits) if y_bits else None, out_low=out_buf(numel, low_bits) if low_bits else None)
    check(ops.epilogue(EPI_RAW_I32, flags=flags), "raw", out=out_buf(numel, 32))
    assert not failed, (geom, a_bits, flags, failed)


def check_stem3x3_non_square(hw):
    """Wo = 129 (W 257, 258): three 64-column tiles, the last one pixel wide.  x = w = -128 with power-of-two ratios, then random data
    with ReLU6 caps and a low-bit copy."""
    hh, ww = hw
    r = np.random.RandomState(hh + 3 * ww)
    n = 2
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    clamp = (-32768, 32767)
    for variant, (relu, y_bits, low) in enumerate([(0, 32, (8, (2 ** 30, 40))), (2, 16, (4, dyadic(0.002))), (1, 32, None)]):
        wt = np.zeros((64, 3, 3, 4), dtype=np.int8)
        if variant == 0:
            x = torch.full((n * hh * ww * 3,), -128, dtype=torch.int8)
            wt[:32, :, :, :3] = -128
            k = r.randint(4, 14, size=64)
            chan = ops.make_chan(r.randint(-2 ** 20, 2 ** 20, size=64), [2 ** 30] * 64, list(30 + k), [2 ** 31 - 1] * 64)
        else:
            x = torch.from_numpy(r.randint(-128, 128, size=n * hh * ww * 3).astype(np.int8))
            wt[:32, :, :, :3] = r.randint(-128, 128, size=(32, 3, 3, 3))
            chan = chan_for(r, 64, 0.9, clamp, "some", bias_span=30000)
        low_bits, lm = (low[0], low[1]) if low else (0, (0, 1))
        low_clamp = (-128, 127) if low_bits == 8 else (0, 15)
        args = dict(x=x, w=torch.from_numpy(wt), chan=chan, relu=relu, clamp=clamp, n=n, hh=hh, ww=ww, y_bits=y_bits,
                    y=out_buf(n * ho * wo * 64, y_bits), low_bits=low_bits, low_me=lm, low_clamp=low_clamp,
                    out_low=out_buf(n * ho * wo * 64, low_bits) if low_bits else None)
        cm, g = run_both("stem3x3", args, ["y", "out_low"] if low_bits else ["y"])
        for a, b in zip(cm, g):
            assert torch.equal(a, b), (hw, variant)
