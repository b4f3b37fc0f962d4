"""TEST INFRASTRUCTURE (oracle, never imported by the product): exact INTEGER restatement of the
reference's quantized forward (SURVEY.md Appendix A), the arbiter for the CUDA kernels.

Everything is int64 numpy.  Convolutions are evaluated as fp64 GEMMs on integer-valued data, which is
exact while |partial sums| < 2^53 (asserted).  ``requant`` is the dyadic requantisation
``RHE(acc * m / 2^e)`` (round-half-to-even) done with exact integer shifts; inside the reference's own
exactness envelope (|acc| < 2^22, SURVEY A.6) it equals the reference's fp64 formulation
(utils/quantization_utils/quant_utils.py:394-413) bit-for-bit, which ``requant_fp64`` restates literally.

Layout: activations NHWC, weights OHWI (the layouts the CUDA engine uses).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

I64 = np.int64


# ----------------------------------------------------------------------------- dyadic arithmetic
def dyadic(r):
    """batch_frexp (quant_utils.py:188-213) for one positive double: m = round_half_up(mant * 2^31), e = 31 - exp.
    m may equal 2^31 (the reference does not renormalise)."""
    mant, ex = math.frexp(float(r))
    x = mant * 2.0 ** 31          # exact (power-of-two scaling)
    m = int(math.floor(x + 0.5))  # exact: x < 2^31 has >= 22 fractional bits of headroom; HALF_UP for x > 0
    return m, 31 - ex


def requant_ratio(a_sf, w_sf, z_sf):
    """new_scale of quant_utils.py:394-397: f64(f32(f64(a)*f64(w))) / f64(f32(z)); a, w, z are fp32."""
    a = np.asarray(a_sf, dtype=np.float32).astype(np.float64)
    w = np.asarray(w_sf, dtype=np.float32).astype(np.float64)
    z = np.asarray(z_sf, dtype=np.float32).astype(np.float64)
    return (a * w).astype(np.float32).astype(np.float64) / z


def dyadic_vec(ratios):
    r = np.atleast_1d(np.asarray(ratios, dtype=np.float64)).reshape(-1)
    me = [dyadic(v) for v in r]
    return np.array([m for m, _ in me], dtype=I64), np.array([e for _, e in me], dtype=I64)


def rhe_shift(p, e):
    """Exact round-half-to-even of p / 2^e for int64 p, 1 <= e <= 62 (elementwise e allowed)."""
    p = np.asarray(p, dtype=I64)
    e = np.asarray(e, dtype=I64)
    assert np.all(e >= 1) and np.all(e <= 62)
    q = p >> e                       # floor
    rem = p - (q << e)               # 0 <= rem < 2^e
    half = I64(1) << (e - 1)
    up = (rem > half) | ((rem == half) & ((q & 1) == 1))
    return q + up.astype(I64)


def requant(acc, m, e):
    """RHE(acc * m / 2^e); acc int64 [..., C], m/e scalars or [C].  acc may also be 2^31: the bias integer the reference's 32-bit
    quantiser gives a channel whose weights are all 0 (its upper bound 2^31 - 1 rounds to 2^31 in fp32), which such a channel's
    accumulator equals (conv_bias).  Such a channel's ratio can be below 2^-62 (e > 62): |acc * m| <= 2^62 then rounds to 0."""
    acc = np.asarray(acc, dtype=I64)
    m = np.asarray(m, dtype=I64)
    e = np.asarray(e, dtype=I64)
    assert acc.min(initial=0) >= -2 ** 31 and acc.max(initial=0) <= 2 ** 31, "accumulator leaves int32"
    assert np.all(m <= 2 ** 31)
    return np.where(e > 62, I64(0), rhe_shift(acc * m, np.minimum(e, 62)))


def conv_bias(acc, w, b):
    """acc + b per output channel (acc [..., C] without bias, w [C, ...] the channel's integer weights).  A channel with a weight is an
    int32 accumulator; one whose weights are all 0 holds its bias alone, which may be 2^31 (requant)."""
    y = acc + b
    if y.min(initial=0) < -2 ** 31 or y.max(initial=0) >= 2 ** 31:
        live = np.asarray(w).reshape(len(b), -1).any(axis=1)
        assert y[..., live].min(initial=0) >= -2 ** 31 and y[..., live].max(initial=0) < 2 ** 31, "accumulator leaves int32"
    return y


def requant_fp64(acc, m, e):
    """Literal restatement of quant_utils.py:406-408: round(f64(acc) * f64(m) / 2^e) with fp64 product."""
    out = np.asarray(acc, dtype=np.float64) * np.asarray(m, dtype=np.float64)
    out = out / (2.0 ** np.asarray(e, dtype=np.float64))
    return np.rint(out).astype(I64)


def clamp_range(bits, mode):
    """fixedpoint_fn clamp (quant_utils.py:365-368,410-413): symmetric [-2^(b-1), 2^(b-1)-1], asymmetric [0, 2^b-1]."""
    if mode == 'symmetric':
        return -(2 ** (bits - 1)), 2 ** (bits - 1) - 1
    return 0, 2 ** bits - 1


# ----------------------------------------------------------------------------- integer ops
def conv2d_nhwc(x, w, stride, pad):
    """x [N,H,W,C] ints, w [O,kh,kw,I] ints -> int64 [N,Ho,Wo,O]; exact via fp64 (asserted)."""
    xt = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float64))).permute(0, 3, 1, 2)
    wt = torch.from_numpy(np.ascontiguousarray(np.asarray(w, dtype=np.float64))).permute(0, 3, 1, 2)
    bound = float(np.abs(np.asarray(x)).max(initial=0)) * float(np.abs(np.asarray(w)).sum(axis=(1, 2, 3)).max(initial=0))
    assert bound < 2 ** 53, "fp64 conv would not be exact"
    y = F.conv2d(xt, wt, None, stride, pad)
    return np.ascontiguousarray(y.permute(0, 2, 3, 1).numpy()).astype(I64)


def linear(x, w):
    """x [N,K], w [O,K] ints -> int64 [N,O]."""
    return (np.asarray(x, dtype=np.float64) @ np.asarray(w, dtype=np.float64).T).astype(I64)


def maxpool_3x3_s2_p1(x):
    """nn.MaxPool2d(3, 2, 1) on NHWC integers (q_resnet.py:93,119)."""
    n, h, w, c = x.shape
    ho, wo = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
    lo = np.iinfo(I64).min
    xp = np.full((n, h + 2, w + 2, c), lo, dtype=I64)
    xp[:, 1:h + 1, 1:w + 1, :] = x
    out = np.full((n, ho, wo, c), lo, dtype=I64)
    for i in range(3):
        for j in range(3):
            out = np.maximum(out, xp[:, i:i + 2 * ho:2, j:j + 2 * wo:2, :][:, :ho, :wo, :])
    return out


def avgpool_trunc(x, k=7):
    """QuantAveragePool2d (quant_modules.py:585-602): trunc(mean_{k x k}(x_int) + 0.01) as pure integers.
    For S = sum >= 0 this is floor(S / k^2); for S < 0 the +0.01 makes exact multiples lose one
    (S = -k^2*q -> -q + 1) and every other value truncates toward zero."""
    n, h, w, c = x.shape
    assert h == k and w == k
    s = np.asarray(x, dtype=I64).sum(axis=(1, 2))
    kk = k * k
    pos = s // kk
    a = -s
    neg = np.where(a % kk == 0, -(a // kk) + (a > 0), -(a // kk))  # trunc toward zero; exact multiples lose one
    return np.where(s >= 0, pos, neg).reshape(n, 1, 1, c)


def quantize_input(x_nchw_f32, scale, bits=8, mode='symmetric'):
    """QuantAct input branch (quant_modules.py:271-274): clamp(round((1/s) * x)), fp32 arithmetic, RNE."""
    s = np.float32(scale)
    inv = np.float32(1.0) / s
    q = np.rint(np.asarray(x_nchw_f32, dtype=np.float32) * inv)
    lo, hi = clamp_range(bits, mode)
    q = np.clip(q, lo, hi).astype(I64)
    return np.ascontiguousarray(q.transpose(0, 2, 3, 1))


# ----------------------------------------------------------------------------- whole network
class IntResNet:
    """Integer-only ResNet built from a ``harvest`` (oracle.fakequant.FakeQuantResNet.harvest() layout):
    integer weights/biases + fp32 scales + act bit widths.  Dataflow = SURVEY Appendix A.4/A.5."""

    def __init__(self, h):
        self.h = h
        self.convs = {}
        for k, c in h["convs"].items():
            w = c["weight_integer"].numpy().astype(I64).transpose(0, 2, 3, 1)  # OIHW -> OHWI
            self.convs[k] = dict(w=np.ascontiguousarray(w), b=c["bias_integer"].numpy().astype(I64),
                                 w_sf=c["w_sf"].numpy().astype(np.float32), stride=c["stride"], pad=c["pad"])
        self.acts = {k: dict(scale=np.float32(a["scale"].item()), bits=a["bits"], mode=a["mode"])
                     for k, a in h["acts"].items()}
        self.fc = dict(w=h["fc"]["weight_integer"].numpy().astype(I64), b=h["fc"]["bias_integer"].numpy().astype(I64),
                       w_sf=h["fc"]["w_sf"].numpy().astype(np.float32))
        self.trace = None

    def _conv(self, name, x):
        c = self.convs[name]
        return conv_bias(conv2d_nhwc(x, c["w"], c["stride"], c["pad"]), c["w"], c["b"])

    def _case0(self, name, acc, a_sf, w_sf, relu):
        """acc -> [ReLU] -> requant(per-channel) -> clamp.  ReLU commutes with the positive-scale requant."""
        a = self.acts[name]
        m, e = dyadic_vec(requant_ratio(a_sf, w_sf, a["scale"]))
        if relu:
            acc = np.maximum(acc, 0)
        lo, hi = clamp_range(a["bits"], a["mode"])
        q = np.clip(requant(acc, m, e), lo, hi)
        self._rec(name, q, pre_relu_note=relu)
        return q

    def _rec(self, name, q, pre_relu_note=False):
        if self.trace is not None:
            self.trace[name] = q

    def _unit(self, p, x16, s16):
        h = self.h
        a = self.acts
        # unit entry: 16-bit residual -> low-bit (case 0 with weight scale 1)
        xa = self._case0(p + ".quant_act", x16, s16, np.float32(1.0), relu=False)
        s_a = a[p + ".quant_act"]["scale"]
        if h["resize"][p]:
            idc = self.convs[p + ".quant_identity_convbn"]
            ident = self._conv(p + ".quant_identity_convbn", xa)
            r1 = requant_ratio(s_a, idc["w_sf"], a[p + ".quant_act_int32"]["scale"])
        else:
            ident = x16
            r1 = requant_ratio(s16, np.float32(1.0), a[p + ".quant_act_int32"]["scale"])
        acc = self._conv(p + ".quant_convbn1", xa)
        x = self._case0(p + ".quant_act1", acc, s_a, self.convs[p + ".quant_convbn1"]["w_sf"], relu=True)
        s_x = a[p + ".quant_act1"]["scale"]
        last = p + ".quant_convbn2"
        acc = self._conv(last, x)
        if h["bottleneck"]:
            x = self._case0(p + ".quant_act2", acc, s_x, self.convs[last]["w_sf"], relu=True)
            s_x = a[p + ".quant_act2"]["scale"]
            last = p + ".quant_convbn3"
            acc = self._conv(last, x)
        # case 1: two independently rounded dyadic terms, no clamp (quant_utils.py:416-456)
        m1, e1 = dyadic_vec(r1)
        m2, e2 = dyadic_vec(requant_ratio(s_x, self.convs[last]["w_sf"], a[p + ".quant_act_int32"]["scale"]))
        y = requant(ident, m1, e1) + requant(acc, m2, e2)
        self._rec(p + ".quant_act_int32", y)
        return np.maximum(y, 0), a[p + ".quant_act_int32"]["scale"]

    def forward(self, x_nchw_f32=None, q_in=None, trace=False):
        """Either a float NCHW batch (quantised like quant_input) or an already-quantised NHWC int8 batch."""
        h = self.h
        self.trace = {} if trace else None
        a_in = self.acts["quant_input"]
        if q_in is None:
            q_in = quantize_input(x_nchw_f32, a_in["scale"], a_in["bits"], a_in["mode"])
        q_in = np.asarray(q_in, dtype=I64)
        self._rec("quant_input", q_in)
        init = h["init_name"]
        acc = self._conv(init, q_in)
        acc = maxpool_3x3_s2_p1(acc)
        # stem: pool -> 16-bit requant (clamped) -> ReLU (q_resnet.py:119-122); the hook sees the pre-ReLU value
        x16 = self._case0("quant_act_int32", acc, a_in["scale"], self.convs[init]["w_sf"], relu=False)
        x16 = np.maximum(x16, 0)
        s16 = self.acts["quant_act_int32"]["scale"]
        for s, n in enumerate(h["units_per_stage"]):
            for u in range(n):
                x16, s16 = self._unit("stage%d.unit%d" % (s + 1, u + 1), x16, s16)
        pooled = avgpool_trunc(x16, 7)
        xo = self._case0("quant_act_output", pooled, s16, np.float32(1.0), relu=False)
        s_o = self.acts["quant_act_output"]["scale"]
        xo = xo.reshape(xo.shape[0], -1)
        acc = linear(xo, self.fc["w"]) + self.fc["b"]
        self.fc_acc = acc
        scale = (self.fc["w_sf"] * np.float32(s_o)).astype(np.float32)     # bias_scaling_factor, fp32 (quant_modules.py:117)
        return acc.astype(np.float32) * scale                             # quant_modules.py:129-130

    __call__ = forward


# ----------------------------------------------------------------------------- MobileNetV2 (SURVEY 8(f) row 3: integer semantics)
def dwconv2d_nhwc(x, w, stride, pad):
    """Depthwise convolution: x [N,H,W,C] ints, w [C,kh,kw,1] ints -> int64 [N,Ho,Wo,C]; exact via fp64 (asserted)."""
    c = x.shape[3]
    xt = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float64))).permute(0, 3, 1, 2)
    wt = torch.from_numpy(np.ascontiguousarray(np.asarray(w, dtype=np.float64))).permute(0, 3, 1, 2)
    assert float(np.abs(np.asarray(x)).max(initial=0)) * float(np.abs(np.asarray(w)).sum(axis=(1, 2, 3)).max(initial=0)) < 2 ** 53
    y = F.conv2d(xt, wt, None, stride, pad, 1, c)
    return np.ascontiguousarray(y.permute(0, 2, 3, 1).numpy()).astype(I64)


def relu6_cap(a_sf, w_sf):
    """Accumulator value that ReLU6 turns every larger accumulator into.  The reference clamps the fp32 activation acc * (w_sf * a_sf)
    at 6.0 (nn.ReLU6, q_mobilenetv2.py:68,72) and the QuantAct behind it recovers integers with round(z / a_sf / w_sf) in fp32
    (quant_utils.py:392): a clamped value becomes C_c = round_f32(6 / a_sf / w_sf_c), an unclamped one its accumulator.  (C_c + 1)
    * s > 6 and (C_c - 1) * s < 6 by more than fp32 rounding can bridge, so the composition is exactly min(acc, C_c) per channel -
    and because the dyadic requantisation is monotone, ReLU6 is a per-channel upper clamp RHE(C_c * m_c / 2^e_c) of its output."""
    six = np.float32(6.0)
    return np.rint(six / np.float32(a_sf) / np.asarray(w_sf, dtype=np.float32)).astype(I64)


class IntMobileNetV2:
    """Integer-only MobileNetV2 from ``FakeQuantMobileNetV2.harvest()``: what a frozen engine has to compute (depthwise
    convolutions, ReLU6 as the per-channel accumulator cap above, signed 16-bit residual stream without ReLU, unit input as the
    case-1 identity, 1x1 QuantConv2d classifier).  Pinned to the reference by tests/test_mobilenetv2_cpu.py."""

    def __init__(self, h):
        self.h = h
        self.convs = {}
        for k, c in h["convs"].items():
            w = c["weight_integer"].numpy().astype(I64).transpose(0, 2, 3, 1)
            self.convs[k] = dict(w=np.ascontiguousarray(w), b=c["bias_integer"].numpy().astype(I64), w_sf=c["w_sf"].numpy().astype(np.float32),
                                 stride=c["stride"], pad=c["pad"], groups=c["groups"])
        self.acts = {k: dict(scale=np.float32(a["scale"].item()), bits=a["bits"], mode=a["mode"]) for k, a in h["acts"].items()}
        o = h["output"]
        self.out = dict(w=o["weight_integer"].numpy().astype(I64).reshape(o["weight_integer"].shape[0], -1),
                        w_sf=o["w_sf"].numpy().astype(np.float32),
                        b=None if o["bias_integer"] is None else o["bias_integer"].numpy().astype(I64))
        self.trace = None

    def _conv(self, name, x):
        c = self.convs[name]
        f = dwconv2d_nhwc if c["groups"] > 1 else conv2d_nhwc
        return conv_bias(f(x, c["w"], c["stride"], c["pad"]), c["w"], c["b"])

    def _case0(self, name, acc, a_sf, w_sf, relu6=False):
        a = self.acts[name]
        m, e = dyadic_vec(requant_ratio(a_sf, w_sf, a["scale"]))
        if relu6:
            acc = np.minimum(np.maximum(acc, 0), relu6_cap(a_sf, w_sf))
        lo, hi = clamp_range(a["bits"], a["mode"])
        q = np.clip(requant(acc, m, e), lo, hi)
        if self.trace is not None:
            self.trace[name] = q
        return q

    def _unit(self, p, residual, x16, s16):
        a, one = self.acts, np.float32(1.0)
        x = self._case0(p + ".quant_act", x16, s16, one)
        s = a[p + ".quant_act"]["scale"]
        for k in (1, 2):
            conv = "%s.conv%d" % (p, k)
            x = self._case0("%s.quant_act%d" % (p, k), self._conv(conv, x), s, self.convs[conv]["w_sf"], relu6=True)
            s = a["%s.quant_act%d" % (p, k)]["scale"]
        acc = self._conv(p + ".conv3", x)
        out = a[p + ".quant_act_int32"]
        if not residual:
            return self._case0(p + ".quant_act_int32", acc, s, self.convs[p + ".conv3"]["w_sf"]), out["scale"]
        m1, e1 = dyadic_vec(requant_ratio(s16, one, out["scale"]))                  # identity = the unit's 16-bit input
        m2, e2 = dyadic_vec(requant_ratio(s, self.convs[p + ".conv3"]["w_sf"], out["scale"]))
        y = requant(x16, m1, e1) + requant(acc, m2, e2)                              # case 1: no clamp, no ReLU (signed stream)
        if self.trace is not None:
            self.trace[p + ".quant_act_int32"] = y
        return y, out["scale"]

    def forward(self, x_nchw_f32, trace=False):
        self.trace = {} if trace else None
        a_in, one = self.acts["quant_input"], np.float32(1.0)
        q = quantize_input(x_nchw_f32, a_in["scale"], a_in["bits"], a_in["mode"])
        if self.trace is not None:
            self.trace["quant_input"] = q
        x16 = self._case0("quant_act_int32", self._conv("init_block", q), a_in["scale"], self.convs["init_block"]["w_sf"], relu6=True)
        s16 = self.acts["quant_act_int32"]["scale"]
        for p, residual in self.h["units"]:
            x16, s16 = self._unit(p, residual, x16, s16)
        x = self._case0("quant_act_before_final_block", x16, s16, one)
        s = self.acts["quant_act_before_final_block"]["scale"]
        x16 = self._case0("quant_act_int32_final", self._conv("features.final_block", x), s, self.convs["features.final_block"]["w_sf"], relu6=True)
        s16 = self.acts["quant_act_int32_final"]["scale"]
        pooled = avgpool_trunc(x16, self.h["pool"])
        xo = self._case0("quant_act_output", pooled, s16, one)
        s_o = self.acts["quant_act_output"]["scale"]
        acc = linear(xo.reshape(xo.shape[0], -1), self.out["w"])
        if self.out["b"] is not None:
            acc = acc + self.out["b"]
        return acc.astype(np.float32) * (self.out["w_sf"] * np.float32(s_o)).astype(np.float32)     # quant_modules.py:718,726-736

    __call__ = forward


def multibranch_requant(x_int, branch_scales, branch_channels, new_scale, bits, mode):
    """QuantAct on a channel-concatenation of branches with different scales (quant_modules.py:275-286, the InceptionV3 edges):
    every branch is requantised on its own with case 0 and weight scale s_i / s_i = 1: q = clamp(RHE(x_i * m_i / 2^e_i)) with
    (m_i, e_i) = batch_frexp(s_i / new_scale).  x_int: NHWC integers of the concatenation.  In an integer engine this is one
    per-channel requantisation (hawq_requant with chan[c] = (0, m_branch(c), e_branch(c)))."""
    out = np.empty_like(np.asarray(x_int, dtype=I64))
    lo, hi = clamp_range(bits, mode)
    c0 = 0
    for s, c in zip(branch_scales, branch_channels):
        m, e = dyadic_vec(requant_ratio(np.float32(s), np.float32(1.0), np.float32(new_scale)))
        out[..., c0:c0 + c] = np.clip(requant(np.asarray(x_int, dtype=I64)[..., c0:c0 + c], m, e), lo, hi)
        c0 += c
    return out
