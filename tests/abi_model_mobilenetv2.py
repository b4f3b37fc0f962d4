"""TEST INFRASTRUCTURE: the MobileNetV2 part of the executable numpy model of the C ABI (tests/abi_model.py, which it extends):
hawq_dwconv3x3, hawq_stem3x3_i8 and the ReLU6 caps of a REQUANT epilogue with relu 2.  Same calling conventions as hawq_b200.ops;
outputs are written in place (CPU tensors)."""
import numpy as np

from oracle import int_ref as ir
from tests import abi_model as am
from hawq_b200._lib import EPI_REQUANT

I64 = np.int64


def chan_caps(chan):
    """hawq_chan.reserved: the per-channel output caps of relu 2 (ReLU6)."""
    return chan.detach().cpu().numpy().reshape(-1, 4)[:, 3].astype(I64)


def requant_clamp(v, m, e, relu, clamp, chan):
    """REQUANT epilogue of acc + bias = v: clamp(RHE(v * m / 2^e)) with ReLU folded into the lower bound; relu 2 (ReLU6) also
    caps channel c at min(clamp_hi, chan[c].reserved), below which the lower bound wins."""
    lo, hi = clamp
    if relu:
        v = np.maximum(v, 0)
    q = np.clip(am.rq(v, m, e), lo, hi)
    if relu == 2:
        q = np.maximum(min(max(lo, 0), hi), np.minimum(q, np.minimum(hi, chan_caps(chan))))
    return q


def conv2d(x, desc, ep, w, chan, res=None, res_chan=None, fscale=None, out=None, out_low=None, logical=None):
    """hawq_conv2d: abi_model.conv2d, whose REQUANT treats any relu as ReLU, then the ReLU6 caps of relu 2 (applying
    min(q, min(hi, cap)) after the ReLU clamp equals requant_clamp).  `logical` only feeds the launch timer."""
    am.conv2d(x, desc, ep, w, chan, res=res, res_chan=res_chan, fscale=fscale, out=out, out_low=out_low)
    if ep.mode == EPI_REQUANT and ep.relu == 2:
        q = am.decode(out, ep.out_bits, ep.out_bits != 8 or ep.clamp_hi <= 127).reshape(-1, desc.Cout)
        lo, hi = ep.clamp_lo, ep.clamp_hi
        am.encode_into(out, np.maximum(min(max(lo, 0), hi), np.minimum(q, np.minimum(hi, chan_caps(chan)))), ep.out_bits)


def dwconv3x3(x, n, hh, ww, c, stride, a_bits, w, chan, relu, out_bits, clamp, out, logical=None):
    """hawq_dwconv3x3: depthwise 3x3 pad 1 (weights [3][3][C]) + the REQUANT epilogue."""
    xa = am.decode(x, a_bits, a_bits == 8).reshape(n, hh, ww, c)
    wa = w.detach().cpu().numpy().astype(I64).reshape(3, 3, c).transpose(2, 0, 1)[..., None]
    bias, m, e = am.chan_fields(chan)
    v = am.sat32(ir.dwconv2d_nhwc(xa, wa, stride, 1) + bias)
    am.encode_into(out, requant_clamp(v, m, e, relu, clamp, chan), out_bits)


def stem3x3(x, w, chan, relu, clamp, n, hh, ww, y_bits, y, low_bits, low_me, low_clamp, out_low, logical=None):
    """hawq_stem3x3_i8: 3x3 stride 2 pad 1 convolution of 3 channels (weights [64][3][3][4]) + the REQUANT epilogue -> stream,
    and the next QuantAct's copy clamp(RHE(y * low_m / 2^low_e))."""
    xa = am.decode(x, 8, True).reshape(n, hh, ww, 3)
    wa = w.detach().cpu().numpy().astype(I64).reshape(64, 3, 3, 4)[..., :3]
    bias, m, e = am.chan_fields(chan)
    q = requant_clamp(am.sat32(ir.conv2d_nhwc(xa, wa, 2, 1) + bias), m, e, relu, clamp, chan)
    am.encode_into(y, q, y_bits)
    if low_bits:
        am.encode_into(out_low, np.clip(am.rq(q, I64(low_me[0]), I64(low_me[1])), low_clamp[0], low_clamp[1]), low_bits)


def install_cpu_backend(monkeypatch):
    """abi_model.install_cpu_backend plus the MobileNetV2 launchers.  Test-only."""
    from hawq_b200 import ops
    am.install_cpu_backend(monkeypatch)
    for name, fn in dict(conv2d=conv2d, dwconv3x3=dwconv3x3, stem3x3=stem3x3).items():
        monkeypatch.setattr(ops, name, fn)
