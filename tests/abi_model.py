"""TEST INFRASTRUCTURE: an executable numpy model of the C ABI (include/hawq_b200.h) built on oracle/int_ref.py: every launcher
of the ResNet and MobileNetV2 engines, the ReLU6 caps of a REQUANT epilogue with relu 2 included.

Two uses:
  * ``install_cpu_backend(monkeypatch)`` replaces ``hawq_b200.ops`` launchers with this model so the host logic
    (lazy fusion in qtensor.py, parameter preparation, descriptors) can be checked on CPU against the goldens;
  * on the GPU box every kernel-level test calls the real library and this model on the same buffers and demands
    bit equality.
Functions take the same arguments as hawq_b200.ops and write their outputs in place (CPU tensors).
"""
import numpy as np
import torch

from oracle import int_ref as ir
from hawq_b200 import ops as real_ops
from hawq_b200._lib import EPI_DEQUANT_F32, EPI_RAW_I32, EPI_REQUANT, EPI_RESIDUAL

I64 = np.int64


# ---------------------------------------------------------------------------------------- storage codecs
def unpack_i4(bytes_u8):
    """hawq nibble order: each 4-byte group holds 8 channels; byte j = c_j | c_{j+4} << 4."""
    b = np.asarray(bytes_u8, dtype=np.uint8).reshape(-1, 4).astype(I64)
    return np.concatenate([b & 0xF, b >> 4], axis=1).reshape(-1)


def pack_i4(vals):
    v = np.asarray(vals, dtype=I64).reshape(-1, 8)
    assert v.min(initial=0) >= 0 and v.max(initial=0) <= 15
    return (v[:, :4] | (v[:, 4:] << 4)).astype(np.uint8).reshape(-1)


def decode(t, bits, signed):
    a = t.detach().cpu().numpy()
    if bits == 4:
        return unpack_i4(a.view(np.uint8))
    if bits == 8:
        return a.view(np.int8 if signed else np.uint8).reshape(-1).astype(I64)
    if bits == 16:
        return a.view(np.int16 if signed else np.uint16).reshape(-1).astype(I64)
    return a.view(np.int32).reshape(-1).astype(I64)


def encode_into(t, vals, bits):
    vals = np.asarray(vals, dtype=I64).reshape(-1)
    if bits == 4:
        src = pack_i4(vals)
        t.view(torch.uint8).reshape(-1).copy_(torch.from_numpy(src))
    elif bits == 8:
        t.view(torch.int8).reshape(-1).copy_(torch.from_numpy((vals & 0xFF).astype(np.uint8).view(np.int8)))
    elif bits == 16:
        t.view(torch.int16).reshape(-1).copy_(torch.from_numpy((vals & 0xFFFF).astype(np.uint16).view(np.int16)))
    else:
        t.view(torch.int32).reshape(-1).copy_(torch.from_numpy(vals.astype(np.int32)))


def chan_fields(chan):
    a = chan.detach().cpu().numpy().reshape(-1, 4)
    return a[:, 0].astype(I64), a[:, 1].astype(np.int32).view(np.uint32).astype(I64), a[:, 2].astype(I64)


def unpermute_i4_weights(w):
    """inverse of hawq_permute_weights_for_i4 on the last axis (blocks of 32)."""
    w = np.asarray(w)
    out = np.empty_like(w)
    wb = w.reshape(-1, 32)
    ob = out.reshape(-1, 32)
    for t in range(4):
        for j in range(4):
            ob[:, 8 * t + j] = wb[:, 4 * t + j]
            ob[:, 8 * t + 4 + j] = wb[:, 16 + 4 * t + j]
    return out


def sat32(v):
    return np.clip(v, -2 ** 31, 2 ** 31 - 1)


def rq(v, m, e):
    return sat32(ir.requant(v, m, e))


def chan_caps(chan):
    """hawq_chan.reserved: the per-channel output caps of relu 2 (ReLU6)."""
    return chan.detach().cpu().numpy().reshape(-1, 4)[:, 3].astype(I64)


def requant_clamp(v, m, e, relu, clamp, chan):
    """REQUANT epilogue of acc + bias = v: clamp(RHE(v * m / 2^e)) with ReLU folded into the lower bound; relu 2 (ReLU6) also
    caps channel c at min(clamp_hi, chan[c].reserved), below which the lower bound wins."""
    lo, hi = clamp
    if relu:
        v = np.maximum(v, 0)
    q = np.clip(rq(v, m, e), lo, hi)
    if relu == 2:
        q = np.maximum(min(max(lo, 0), hi), np.minimum(q, np.minimum(hi, chan_caps(chan))))
    return q


status = {"flags": 0}


# ---------------------------------------------------------------------------------------- ABI model
def conv2d(x, desc, ep, w, chan, res=None, res_chan=None, fscale=None, out=None, out_low=None, logical=None):
    """hawq_conv2d.  `logical` only feeds the launch timer."""
    n, h, wd, cin, cout = desc.N, desc.H, desc.W, desc.Cin, desc.Cout
    xa = decode(x, desc.a_bits, desc.a_bits == 8).reshape(n, h, wd, cin)
    wa = w.detach().cpu().numpy().astype(I64).reshape(-1)[:cout * desc.kh * desc.kw * cin].reshape(cout, desc.kh, desc.kw, cin)
    if desc.a_bits == 4:
        wa = unpermute_i4_weights(wa)
    acc = ir.conv2d_nhwc(xa, wa, desc.stride, desc.pad)
    bias, m, e = chan_fields(chan)
    v = sat32(acc + bias)
    if ep.mode == EPI_REQUANT:
        encode_into(out, requant_clamp(v, m, e, ep.relu, (ep.clamp_lo, ep.clamp_hi), chan), ep.out_bits)
    elif ep.mode == EPI_RESIDUAL:
        if ep.res_kind == 1:
            r = decode(res, 32, True).reshape(v.shape)
            _, m1, e1 = chan_fields(res_chan)
        else:
            r = decode(res, ep.res_bits, ep.res_bits == 32).reshape(v.shape)
            m1, e1 = I64(ep.res_m), I64(ep.res_e)
        if ep.flags & 3:   # fast-path promise: a term leaving int32 raises HAWQ_FLAG_REQUANT_OVERFLOW (contents then unspecified)
            for q in (ir.requant(r, m1, e1), ir.requant(v, m, e)):
                if q.min(initial=0) < -2 ** 31 or q.max(initial=0) > 2 ** 31 - 1:
                    status["flags"] |= 4
        y = sat32(rq(r, m1, e1) + rq(v, m, e))
        if ep.relu:
            y = np.maximum(y, 0)
        if ep.y_bits == 32:
            encode_into(out, y, 32)
        elif ep.y_bits == 16:
            if y.max(initial=0) > 65535:
                status["flags"] |= 1
            encode_into(out, np.minimum(y, 65535), 16)
        if ep.low_bits:
            encode_into(out_low, np.clip(rq(y, I64(ep.low_m), I64(ep.low_e)), ep.low_lo, ep.low_hi), ep.low_bits)
    elif ep.mode == EPI_RAW_I32:
        encode_into(out, v, 32)
    else:
        fs = fscale.detach().cpu().numpy().astype(np.float32)
        o = (v.reshape(-1, cout).astype(np.float32) * fs)[:, :ep.cout_store]
        out.view(-1, ep.cout_store).copy_(torch.from_numpy(np.ascontiguousarray(o)))


def conv2d_dual(x, desc, ep, w, chan, desc2, x2, w2, chan2, out=None, out_low=None):
    """hawq_conv2d_dual == RAW_I32 identity convolution followed by the res_kind 1 RESIDUAL convolution."""
    m = desc.N * desc.H * desc.W
    raw = torch.empty(m * desc.Cout, dtype=torch.int32)
    conv2d(x2, desc2, real_ops.epilogue(EPI_RAW_I32), w2, chan2, out=raw)
    ep1 = real_ops.epilogue(EPI_RESIDUAL, relu=ep.relu, res_kind=1, res_bits=32, y_bits=ep.y_bits, low_bits=ep.low_bits,
                            low_me=(ep.low_m, ep.low_e), low_clamp=(ep.low_lo, ep.low_hi), flags=ep.flags)
    conv2d(x, desc, ep1, w, chan, res=raw, res_chan=chan2, out=out, out_low=out_low)


def dwconv3x3(x, n, hh, ww, c, stride, a_bits, w, chan, relu, out_bits, clamp, out, logical=None):
    """hawq_dwconv3x3: depthwise 3x3 pad 1 (weights [3][3][C]) + the REQUANT epilogue."""
    xa = decode(x, a_bits, a_bits == 8).reshape(n, hh, ww, c)
    wa = w.detach().cpu().numpy().astype(I64).reshape(3, 3, c).transpose(2, 0, 1)[..., None]
    bias, m, e = chan_fields(chan)
    v = sat32(ir.dwconv2d_nhwc(xa, wa, stride, 1) + bias)
    encode_into(out, requant_clamp(v, m, e, relu, clamp, chan), out_bits)


def linear(x, w, chan, fscale, out, n, k, cout, cout_pad):
    d = real_ops.conv_desc(n, 1, 1, k, cout_pad, 1, 1, 1, 0, 8)
    conv2d(x, d, real_ops.epilogue(EPI_DEQUANT_F32, cout_store=cout), w, chan, fscale=fscale, out=out)


def stem_conv(x, w, chan, clamp, out, n, hh, ww):
    xa = decode(x, 8, True).reshape(n, hh, ww, 3)
    wa = w.detach().cpu().numpy().astype(I64).reshape(64, 7, 8, 4)[:, :, :7, :3]
    bias, m, e = chan_fields(chan)
    v = sat32(ir.conv2d_nhwc(xa, wa, 2, 3) + bias)
    q = np.maximum(np.clip(rq(v, m, e), clamp[0], clamp[1]), 0)
    encode_into(out, q, 16)


def stem3x3(x, w, chan, relu, clamp, n, hh, ww, y_bits, y, low_bits, low_me, low_clamp, out_low, logical=None):
    """hawq_stem3x3_i8: 3x3 stride 2 pad 1 convolution of 3 channels (weights [64][3][3][4]) + the REQUANT epilogue -> stream,
    and the next QuantAct's copy clamp(RHE(y * low_m / 2^low_e))."""
    xa = decode(x, 8, True).reshape(n, hh, ww, 3)
    wa = w.detach().cpu().numpy().astype(I64).reshape(64, 3, 3, 4)[..., :3]
    bias, m, e = chan_fields(chan)
    q = requant_clamp(sat32(ir.conv2d_nhwc(xa, wa, 2, 1) + bias), m, e, relu, clamp, chan)
    encode_into(y, q, y_bits)
    if low_bits:
        encode_into(out_low, np.clip(rq(q, I64(low_me[0]), I64(low_me[1])), low_clamp[0], low_clamp[1]), low_bits)


def stem_pool(x, w256, chan, clamp, n, hh, ww, y_bits, y, low_bits, low_me, low_clamp, out_low):
    """hawq_stem_pool_i8 == hawq_stem_conv_i8 followed by hawq_maxpool_requant."""
    w = w256.detach().cpu().reshape(64, 8, 8, 4)[:, :7].contiguous()
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    t16 = torch.zeros(n * ho * wo * 64, dtype=torch.int16)
    stem_conv(x, w, chan, clamp, t16, n, hh, ww)
    maxpool_requant(t16, n, ho, wo, 64, y_bits, y, low_bits, low_me, low_clamp, out_low)


def maxpool_requant(x, n, hh, ww, c, y_bits, y, low_bits, low_me, low_clamp, out_low):
    xa = decode(x, 16, True).reshape(n, hh, ww, c)
    assert xa.min(initial=0) >= 0, "hawq_maxpool_requant needs x >= 0 (it pads with 0 and reads the maxima as unsigned)"
    p = ir.maxpool_3x3_s2_p1(xa)
    if y_bits:
        encode_into(y, p, y_bits)
    if low_bits:
        encode_into(out_low, np.clip(rq(p, I64(low_me[0]), I64(low_me[1])), low_clamp[0], low_clamp[1]), low_bits)


def avgpool_requant(x, n, hw, c, x_bits, me, clamp, out):
    xa = decode(x, x_bits, x_bits == 32).reshape(n, hw, c)
    k = int(round(hw ** 0.5))
    p = ir.avgpool_trunc(xa.reshape(n, k, k, c), k).reshape(n, c)
    encode_into(out, np.clip(rq(p, I64(me[0]), I64(me[1])), clamp[0], clamp[1]), 8)


def quantize_input(x, scale, clamp, out):
    q = ir.quantize_input(x.detach().cpu().numpy(), np.float32(scale), 8, 'symmetric')
    encode_into(out, np.clip(q, clamp[0], clamp[1]), 8)


def quantize_input_u8(x, mean, std, scale, clamp, out):
    """ToTensor (u / 255), Normalize ((v - mean) / std), QuantAct input branch: one fp32 operation per step, like torch."""
    u = x.detach().cpu().numpy().astype(np.float32)                              # NHWC
    v = (u / np.float32(255.0) - np.asarray(mean, dtype=np.float32)) / np.asarray(std, dtype=np.float32)
    q = ir.quantize_input(np.ascontiguousarray(v.transpose(0, 3, 1, 2)), np.float32(scale), 8, 'symmetric')
    encode_into(out, np.clip(q, clamp[0], clamp[1]), 8)


def requant(x, rows, c, x_bits, chan, chan_stride, relu, out_bits, clamp, out):
    xa = decode(x, x_bits, x_bits == 32).reshape(rows, c)
    bias, m, e = chan_fields(chan)
    if chan_stride == 0:
        bias, m, e = bias[:1], m[:1], e[:1]
    v = sat32(xa + bias)
    if relu:
        v = np.maximum(v, 0)
    encode_into(out, np.clip(rq(v, m, e), clamp[0], clamp[1]), out_bits)


def add_requant(acc, rows, c, chan, ep, res, res_chan, y, out_low):
    a = decode(acc, 32, True).reshape(rows, c)
    bias, m, e = chan_fields(chan)
    if ep.res_kind == 1:
        r = decode(res, 32, True).reshape(rows, c)
        _, m1, e1 = chan_fields(res_chan)
    else:
        r = decode(res, ep.res_bits, ep.res_bits == 32).reshape(rows, c)
        m1, e1 = I64(ep.res_m), I64(ep.res_e)
    s = sat32(rq(r, m1, e1) + rq(sat32(a + bias), m, e))
    if ep.relu:
        s = np.maximum(s, 0)
    if ep.y_bits == 16:
        if s.max(initial=0) > 65535:
            status["flags"] |= 1
        encode_into(y, np.minimum(s, 65535), 16)
    elif ep.y_bits == 32:
        encode_into(y, s, 32)
    if ep.low_bits:
        encode_into(out_low, np.clip(rq(s, I64(ep.low_m), I64(ep.low_e)), ep.low_lo, ep.low_hi), ep.low_bits)


def dequant(x, n, hh, ww, c, x_bits, x_signed, scale, out):
    q = decode(x, x_bits, x_signed).reshape(n, hh, ww, c).transpose(0, 3, 1, 2)
    out.copy_(torch.from_numpy(np.ascontiguousarray(q.astype(np.float32) * np.float32(scale))).view_as(out))


def pack_i4_op(src, dst):
    dst.view(torch.uint8).reshape(-1).copy_(torch.from_numpy(pack_i4(src.detach().cpu().numpy().astype(I64))))


def unpack_i4_op(src, dst):
    dst.view(torch.uint8).reshape(-1).copy_(torch.from_numpy(unpack_i4(src.detach().cpu().numpy()).astype(np.uint8)))


def install_cpu_backend(monkeypatch):
    """Route hawq_b200.ops launchers to this model (CPU tensors).  Test-only."""
    from hawq_b200 import ops
    status["flags"] = 0
    for name, fn in dict(conv2d=conv2d, conv2d_dual=conv2d_dual, dwconv3x3=dwconv3x3, linear=linear, stem_conv=stem_conv, stem3x3=stem3x3,
                         stem_pool=stem_pool, maxpool_requant=maxpool_requant, avgpool_requant=avgpool_requant, quantize_input=quantize_input, quantize_input_u8=quantize_input_u8, requant=requant,
                         add_requant=add_requant, dequant=dequant, pack_i4=pack_i4_op, unpack_i4=unpack_i4_op).items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(ops, "reset_status", lambda idx: status.__setitem__("flags", 0))
    monkeypatch.setattr(ops, "get_status", lambda idx: status["flags"])
    from hawq_b200 import qtensor
    monkeypatch.setattr(qtensor, "_require_cuda", lambda x, what: None)
