"""Integer payload tensors and the frozen forward of the quant modules.

``IntActivation`` is what frozen engine modules hand to each other instead of the reference's fp32
``integer * scale`` tensors: a ``torch.Tensor`` wrapper subclass (logical shape NCHW, dtype fp32 as far as graph
code can tell) whose *node* carries either concrete integers in HBM (NHWC int8 / packed uint4 / uint16 or int32
residual stream) or a *pending* producer (a convolution, a residual sum, the stem, an average pool) that has not
been launched yet.  Pending producers are how the reference's module-by-module graph
(conv -> ReLU -> QuantAct, conv -> add -> QuantAct -> ReLU -> next QuantAct, reference
``utils/models/q_resnet.py:231-260``) turns into one fused kernel per convolution: the producer is launched when the
consuming ``QuantAct`` is reached, with that activation's dyadic requantisation (and, for residual sums, the NEXT
unit's low-bit activation) folded into the kernel epilogue.

``nn.ReLU``, ``nn.ReLU6``, ``nn.MaxPool2d``, ``+``, ``.view`` on an ``IntActivation`` are intercepted through
``__torch_function__`` and recorded on the node; anything else is not an integer-path operation and raises.

Channel padding: a convolution output or stream whose channel count is not a multiple of 64 (MobileNetV2's 16 / 24 / 32 / 96 /
144 ... channels) is stored zero-padded to the next multiple of 64 (``stored_channels``), so every 1x1 layer runs on the
convolution kernel unchanged.  Padded weight rows and columns, biases and multipliers are 0, so every padded channel is exactly 0
in every tensor (RHE(0) = 0, and a case-1 sum of zeros is 0).  ``Node.shape`` keeps the logical shape, ``Node.cs`` the stored
channel count that every descriptor uses.
"""
import contextlib
import copy
import math
import os
import threading

import numpy as np

import torch

from . import ops, quant_math as qmath
from ._lib import EPI_RAW_I32, EPI_REQUANT, EPI_RESIDUAL, EP_RATIOS_LE_2P20, ERR_UNSUPPORTED, HawqError


class EngineConfig(threading.local):
    """Per-thread execution mode of the frozen forward (no process-global state: several engines / threads may run at once).

    residual_bits: storage of the post-ReLU residual stream: 32 (always exact) or 16 (uint16 + sticky overflow flag
        HAWQ_FLAG_RESIDUAL_OVERFLOW; ``CompiledModel`` re-runs in 32-bit mode when the flag is raised).
    fast_kernels: False withholds every HAWQ_EP_RATIOS_* promise (always-saturating generic kernels).
    checked: True when the caller reads the device status word after the forward (``CompiledModel`` does).  The plain eager
        frozen forward does not, so it never promises HAWQ_EP_RATIOS_LE_2P20: the checked FP64 epilogue only *flags* an int32
        overflow and relies on the host to re-run, whereas ratios <= 1 cannot overflow and the exact form saturates like the reference."""
    residual_bits = 32
    fast_kernels = True
    checked = False
    # HBM container of 4-bit activations: 8 = one value per byte (the int8 kernels consume them directly: Hopper has no int4 MMA,
    # so packed nibbles must be expanded on chip before every use), 4 = packed nibbles (half the bytes of those tensors, expanded in
    # registers by the convolution).  Same integers either way; the byte container is the default, the packed one is kept for
    # bandwidth-bound deployments and is what the kernel tests exercise with a_bits = 4.
    a4_container = 4 if os.environ.get("HAWQ_B200_A4_STORAGE", "byte") == "packed" else 8
    dual = os.environ.get("HAWQ_B200_DUAL", "1") != "0"   # resize units: identity conv + last conv in one kernel (uint16 stream only)


config = EngineConfig()


@contextlib.contextmanager
def engine_mode(residual_bits=32, fast_kernels=True, checked=False):
    """Scoped execution mode (restored on exit, also when the forward raises)."""
    saved = (config.residual_bits, config.fast_kernels, config.checked)
    config.residual_bits, config.fast_kernels, config.checked = residual_bits, fast_kernels, checked
    try:
        yield config
    finally:
        config.residual_bits, config.fast_kernels, config.checked = saved


def _ratio_flags(*pairs):
    """HAWQ_EP_RATIOS_* promise for this thread's execution mode (see EngineConfig)."""
    if not config.fast_kernels:
        return 0
    f = ops.ratio_flags(*pairs)
    if f == EP_RATIOS_LE_2P20 and not config.checked:
        return 0
    return f


class Node:
    """Payload of an IntActivation.  kind:
         'int'      concrete integers: data (NHWC), bits, signed
         'conv'     pending convolution: mod, src(Node 'int'), a_sf, relu, pool (its shape before a fused MaxPool2d(3,2,1))
         'sum'      pending conv + identity: a (Node conv), b (Node conv | int)
         'residual' pending case-1 requant of a 'sum' by QuantAct `act` (+relu)
         'stem'     pending stem conv + pool + 16-bit requant by QuantAct `act` (+relu)
         'avgpool'  pending integer average pool of src
    """
    __slots__ = ("kind", "shape", "cs", "data", "bits", "signed", "mod", "src", "a_sf", "relu", "relu6", "pool", "a", "b", "act", "args")

    def __init__(self, kind, shape, **kw):
        self.kind, self.shape = kind, tuple(shape)
        self.cs = self.shape[1]          # stored channels: an input handed in by the caller is not padded
        self.data = self.mod = self.src = self.a_sf = self.a = self.b = self.act = self.args = self.pool = None
        self.bits, self.signed, self.relu, self.relu6 = 0, True, False, False
        for k, v in kw.items():
            setattr(self, k, v)

    def become_int(self, data, bits, signed):
        self.kind, self.data, self.bits, self.signed = "int", data, bits, signed
        self.cs = stored_channels(self.shape[1])
        self.mod = self.src = self.a = self.b = self.act = self.args = None


def stored_channels(c):
    """Channels of a kernel-written tensor with c logical channels in HBM: zero-padded to a multiple of 64."""
    return -(-c // 64) * 64


def _stored_shape(shape):
    return (shape[0], stored_channels(shape[1])) + tuple(shape[2:])


def _new_int(device, shape, bits, signed):
    """Node 'int' with fresh storage for a kernel output of logical shape `shape` (channels padded, stored_channels)."""
    return Node("int", shape, data=_alloc(device, _stored_shape(shape), bits), bits=bits, signed=signed, cs=stored_channels(shape[1]))


class IntActivation(torch.Tensor):
    @staticmethod
    def __new__(cls, node, device, shape=None):
        t = torch.Tensor._make_wrapper_subclass(cls, tuple(shape if shape is not None else node.shape),
                                                dtype=torch.float32, device=device, requires_grad=False)
        t.node = node
        return t

    def __repr__(self):
        n = self.node
        return "IntActivation(kind=%s, shape=%s, bits=%s, device=%s)" % (n.kind, tuple(self.shape), n.bits, self.device)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, "__name__", str(func))
        if name in ("relu", "relu_"):
            return _relu(args[0])
        if name in ("hardtanh", "hardtanh_", "relu6", "relu6_"):
            return _relu6(name, *args, **kwargs)
        if name in ("max_pool2d", "_max_pool2d", "max_pool2d_with_indices"):
            return _max_pool(*args, **kwargs)
        if name in ("add", "__add__", "__radd__", "__iadd__", "add_"):
            return _add(args[0], args[1])
        if name in ("view", "reshape", "flatten"):
            return _reshape(name, *args, **kwargs)
        if name in ("size", "dim", "__get__", "shape", "__repr__", "__str__", "is_cuda", "device"):
            with torch._C.DisableTorchFunctionSubclass():
                return func(*args, **kwargs)
        raise NotImplementedError(
            "torch op %r on an IntActivation is not part of the HAWQ integer path (supported between frozen "
            "modules: ReLU, ReLU6, MaxPool2d(3,2,1) after the stem, +, view/flatten). Use .dequantize() for a float tensor." % name)

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        raise NotImplementedError("aten op %s reached an IntActivation: only the HAWQ integer-path ops are defined on it" % func)

    def dequantize(self, scale):
        """fp32 NCHW ``integer * scale`` tensor (what the reference would have produced at this edge)."""
        n = materialize(self.node, self.device)
        s = float(scale.reshape(-1)[0]) if torch.is_tensor(scale) else float(scale)
        shp = self.node.shape
        nb, c = shp[0], shp[1]
        hh, ww = (shp[2], shp[3]) if len(shp) == 4 else (1, 1)
        out = torch.empty((nb, n.cs, hh, ww), dtype=torch.float32, device=self.device)
        ops.dequant(n.data, nb, hh, ww, n.cs, n.bits, n.signed, s, out)
        return out[:, :c].contiguous().view(*self.shape)

    def int_tensor(self):
        """Concrete integers as an int32 tensor in logical (NCHW / NC) order, padded channels dropped — for tests and debugging."""
        n = materialize(self.node, self.device)
        shp = self.node.shape
        v = unpack_to_int32(n).view(shp[0], *([shp[2], shp[3]] if len(shp) == 4 else []), n.cs)[..., :shp[1]]
        return v.permute(*((0, 3, 1, 2) if len(shp) == 4 else (0, 1))).contiguous()


def unpack_to_int32(n):
    """Node 'int' -> flat int32 tensor in storage (NHWC) order."""
    d = n.data
    if n.bits == 32:
        return d.view(torch.int32).reshape(-1).clone()
    if n.bits == 16:
        v = d.view(torch.int16).reshape(-1).to(torch.int32)
        return v if n.signed else (v & 0xFFFF)
    if n.bits == 8:
        return d.view(torch.int8 if n.signed else torch.uint8).reshape(-1).to(torch.int32)
    b = d.view(torch.uint8).reshape(-1, 4).to(torch.int32)            # hawq nibble order
    return torch.cat([b & 0xF, b >> 4], dim=1).reshape(-1)


# ------------------------------------------------------------------------------------------------ helpers
def _cpu_f32(t):
    return t.detach().to("cpu", torch.float32).reshape(-1)


def _key(t):
    return None if t is None else _cpu_f32(t).numpy().tobytes()


def _buf_key(t):
    return None if t is None else (id(t), t._version, t.data_ptr())


def _alloc(device, shape, bits):
    numel = math.prod(shape)
    if bits == 32:
        return torch.empty(numel, dtype=torch.int32, device=device)
    if bits == 16:
        return torch.empty(numel, dtype=torch.int16, device=device)
    if bits == 8:
        return torch.empty(numel, dtype=torch.int8, device=device)
    return torch.empty(numel // 2, dtype=torch.uint8, device=device)


def _act_clamp(act):
    return qmath.clamp_range(act.activation_bit, act.quant_mode)


def _store_bits(act):
    """Bits per value of `act`'s output in HBM (see EngineConfig.a4_container)."""
    b = act.activation_bit
    return config.a4_container if b == 4 else b


def _store_signed(act):
    """Whether the stored integers may be read as signed bytes: symmetric activations, and 4-bit values in byte containers (0..15)."""
    return act.quant_mode == "symmetric" or (act.activation_bit == 4 and _store_bits(act) == 8)


def _frozen_scale(act):
    """Scale of a frozen QuantAct, CPU fp32 [1]; refreshes the act_scaling_factor buffer like the reference forward."""
    c = act.__dict__.setdefault("_hawq_cache", {})
    # keyed on buffer identity + in-place version (no device->host copy on a hit: the buffers may live on the GPU and
    # this runs inside CUDA-graph capture); `x_min += lo` bumps _version, `x_min = ...` rebinds the buffer
    key = ("scale", _buf_key(act.x_min), _buf_key(act.x_max), act.activation_bit, act.quant_mode, act.__dict__.get("_override_gen", 0))
    if c.get("scale_key") != key:
        sf = act.current_scale().detach().to("cpu", torch.float32).reshape(1)
        act.act_scaling_factor = sf.to(act.x_min.device)
        c["scale"], c["me"], c["gen"] = sf, {}, c.get("gen", 0) + 1
        c["scale_key"] = key            # last: another thread that sees the key finds the entries it keys
    return c["scale"]


def _act_tag(kind, act):
    """Cache tag of per-channel epilogue parameters that depend on QuantAct `act` (invalidated when its scale changes)."""
    return (kind, id(act), act._hawq_cache["gen"])


def _dyadic(act, a_sf, w_sf, tag):
    """Cached (m list, e list) of the ratio (a_sf * w_sf) / act_scale (quant_utils.py:394-400)."""
    c = act._hawq_cache
    key = (tag, _key(a_sf), _key(w_sf))
    if key not in c["me"]:
        ratio = qmath.requant_ratio(_cpu_f32(a_sf), _cpu_f32(w_sf), c["scale"])
        c["me"][key] = qmath.dyadic_pairs(ratio)
    return c["me"][key]


def _ones():
    return torch.ones(1)


# ------------------------------------------------------------------------------------------------ conv params
_OWN_BUFFERS = ("weight_integer", "bias_integer", "convbn_scaling_factor", "conv_scaling_factor", "fc_scaling_factor")


def _param_versions(mod):
    """In-place modification counters of every float parameter / statistic the integer plan of `mod` derives from:
    ``load_state_dict`` and optimizer steps write in place, so a changed tuple invalidates the cached plan (the reference
    recomputes its integers on every forward, quant_modules.py:440-484; SURVEY.md 8(b) lifecycle row)."""
    vs = []
    for name, t in list(mod.named_parameters()) + list(mod.named_buffers()):
        if name.rsplit(".", 1)[-1] in _OWN_BUFFERS or "num_batches_tracked" in name:
            continue
        vs.append((id(t), t._version))
    vs.append(mod.__dict__.get("_override_gen", 0))          # integers installed from a quantized checkpoint
    return tuple(vs)


def _plan(mod, a_sf, device, key, build):
    """Integer plan of frozen module `mod` for input scale a_sf on `device`; `key` holds the bit widths and options it also
    depends on.  `build()` makes the plan when any of these or a parameter version (_param_versions) changed.  A new plan
    starts a new cache dict instead of clearing the old one in place: a CompiledModel may still replay graphs that read
    the old plan's buffers."""
    c = mod.__dict__.setdefault("_hawq_cache", {})
    key = (_key(a_sf), str(device), key, _param_versions(mod))
    ent = c.get(key)
    if ent is None:
        if c:
            c = mod.__dict__["_hawq_cache"] = {}
        with torch.no_grad():
            ent = c[key] = build()
    return ent


def _conv_cache(mod, a_sf, a_bits, device):
    """Device-resident integer parameters of a frozen conv module for input scale a_sf / input width a_bits."""
    return _plan(mod, a_sf, device, (a_bits, mod.weight_bit, mod.per_channel, mod.bias_bit, mod.quantize_bias),
                 lambda: _conv_params(mod, a_sf, a_bits, device))


def _conv_params(mod, a_sf, a_bits, device):
    """kind: 'conv' (conv_igemm: OHWI, channels padded to stored_channels), 'stem' (ResNet 7x7/2 stem), 'stem3' (MobileNetV2 3x3/2
    stem, hawq_stem3x3_i8: [64][3][3][4]) or 'dw' (depthwise 3x3, hawq_dwconv3x3: [3][3][C stored]).  cin / cout are the stored
    channel counts, cout_l the logical one."""
    conv = mod.conv
    src_dev = conv.weight.device
    w_sf, w_int, b_int, _ = mod.integer_params(a_sf.to(src_dev))
    w_sf = w_sf.detach().to("cpu", torch.float32)
    cout, cin_g, kh, kw = w_int.shape
    groups = conv.groups
    cin = cin_g * groups
    dw = groups != 1 and groups == cin == cout and kh == 3 and cin_g == 1
    if (groups != 1 and not dw) or conv.dilation[0] != 1 or conv.dilation[1] != 1 or kh != kw or conv.stride[0] != conv.stride[1]:
        raise NotImplementedError("hawq_b200 convolutions: groups=1 or depthwise 3x3, dilation=1, square kernels/strides only")
    w = w_int.detach().to("cpu").permute(0, 2, 3, 1).contiguous().to(torch.int8)      # OHWI
    cin_s, cout_s = stored_channels(cin), stored_channels(cout)
    bias = np.zeros(cout_s, dtype=np.int64)
    if b_int is not None:
        bias[:cout] = b_int.detach().to("cpu").to(torch.int64).numpy()
    zero_acc = np.ones(cout_s, dtype=bool)                         # channels whose accumulator is identically 0 (ops.make_chan)
    zero_acc[:cout] = ~w.reshape(cout, -1).any(dim=1).numpy()
    kind = "conv"
    if cin == 3 and kh == 7 and conv.stride[0] == 2 and conv.padding[0] == 3 and cout == 64:
        kind = "stem"
        wp = torch.zeros((cout, 8, 8, 4), dtype=torch.int8)       # kernel rows 7 -> 8, taps 7 -> 8, channels 3 -> 4 (zeros)
        wp[:, :7, :7, :3] = w
        w = wp[:, :7].contiguous()                                # stem kernel layout: K = 224
        cin_s = 3
    elif cin == 3 and kh == 3 and conv.stride[0] == 2 and conv.padding[0] == 1 and cout <= 64:
        kind = "stem3"
        wp = torch.zeros((64, 3, 3, 4), dtype=torch.int8)         # output channels -> 64, input channels 3 -> 4 (zeros)
        wp[:cout, :, :, :3] = w
        w, cin_s = wp, 3
    elif dw:
        if conv.padding[0] != 1 or conv.stride[0] not in (1, 2):
            raise NotImplementedError("hawq_b200 depthwise convolutions: 3x3, pad 1, stride 1 or 2")
        kind = "dw"
        wp = torch.zeros((3, 3, cout_s), dtype=torch.int8)        # channel-minor: one 16-byte load holds 16 channels of a tap
        wp[:, :, :cout] = w[:, :, :, 0].permute(1, 2, 0)
        w = wp
    else:
        wp = torch.zeros((cout_s, kh, kw, cin_s), dtype=torch.int8)
        wp[:cout, :, :, :cin] = w
        w = wp
        if a_bits == 4:
            ops.permute_weights_for_i4(w)
    tiled = kind == "conv" and torch.device(device).type == "cuda"
    return dict(w=ops.upload_weights(w, device) if tiled else w.to(device), w_layout=1 if tiled else 0, w_sf=w_sf, bias=bias,
                cout=cout_s if kind != "stem3" else 64, cin=cin_s, cout_l=cout, k=kh, stride=conv.stride[0], pad=conv.padding[0],
                stem=kind == "stem", kind=kind, chan={}, zero_acc=zero_acc)


def _pad_me(m, e, c):
    """(m, e) lists of the logical channels (or one scalar pair) -> c stored channels; padded channels get m = 0."""
    if len(m) == 1 or len(m) == c:
        return list(m), list(e)
    return list(m) + [0] * (c - len(m)), list(e) + [1] * (c - len(e))


def _chan_tensor(ent, tag, m, e, device, caps=None, raw=False):
    """Cached hawq_chan table of plan `ent`; `caps`: a function giving the ReLU6 caps (computed on a cache miss only); `raw`: a
    RAW_I32 table (ops.make_chan)."""
    t = ent["chan"].get(tag)
    if t is None:
        m, e = _pad_me(m, e, len(ent["bias"]))
        t = ent["chan"][tag] = ops.make_chan(ent["bias"], m, e, caps() if caps else None, ent["zero_acc"], raw).to(device)
    return t


def _relu6_caps(n, ent, m, e, hi):
    """Per-channel output caps of ReLU6 (hawq_chan.reserved with relu 2): ReLU6 caps the accumulator at
    C_c = round_f32(6 / a_sf / w_sf_c) (the reference clamps the fp32 value acc * a_sf * w_sf_c at 6 and its QuantAct recovers
    round(z / a_sf / w_sf_c)); the requantisation is monotone, so the output cap is RHE(C_c * m_c / 2^e_c).  A cap C_c >= 2^31
    can never bind: hi.  Padded channels: hi."""
    cl = ent["cout_l"]
    acc_cap = np.broadcast_to(np.rint(np.float32(6.0) / _cpu_f32(n.a_sf).numpy()[0] / _cpu_f32(ent["w_sf"]).numpy()), (cl,))
    mm, ee = (m, e) if len(m) == cl else (list(m) * cl, list(e) * cl)
    caps = [min(hi, ops.rhe_requant_host(int(c), mm[i], ee[i])) if c < 2 ** 31 else hi for i, c in enumerate(acc_cap)]
    return caps + [hi] * (len(ent["bias"]) - cl)


# ------------------------------------------------------------------------------------------------ lazy ops
def _relu6(name, x, *args, **kw):
    """nn.ReLU6 (F.hardtanh(x, 0, 6)) or F.relu6 on a pending convolution: recorded as `relu6`, applied by the consuming QuantAct
    as a per-channel clamp (_relu6_caps)."""
    if name.startswith("hardtanh"):
        pos = dict(zip(("min_val", "max_val"), args))
        lo, hi = kw.get("min_val", pos.get("min_val", -1.0)), kw.get("max_val", pos.get("max_val", 1.0))
        if float(lo) != 0.0 or float(hi) != 6.0:
            raise NotImplementedError("hardtanh(%s, %s) on an IntActivation: only ReLU6 = hardtanh(0, 6) is part of the integer path" % (lo, hi))
    n = x.node
    if n.kind != "conv" or n.pool is not None:
        raise NotImplementedError("ReLU6 on an IntActivation must follow a convolution directly (got a %s)" % n.kind)
    m = copy.copy(n)
    m.relu = m.relu6 = True
    return IntActivation(m, x.device, x.shape)


def _relu(x):
    n = x.node
    if n.kind in ("conv", "residual", "stem"):
        if n.kind == "conv" and n.pool is not None:
            raise NotImplementedError("ReLU after a pooled convolution must follow its QuantAct")
        m = copy.copy(n)
        m.relu = True
        return IntActivation(m, x.device, x.shape)
    if n.kind == "int":
        if not n.signed:
            return x
        dt = {8: torch.int8, 16: torch.int16, 32: torch.int32}[n.bits]
        m = Node("int", n.shape, data=torch.clamp_min(n.data.view(dt), 0), bits=n.bits, signed=n.signed)
        return IntActivation(m, x.device, x.shape)
    raise NotImplementedError("ReLU on a pending %s" % n.kind)


def _max_pool(x, kernel_size, stride=None, padding=0, dilation=1, ceil_mode=False, return_indices=False):
    n = x.node
    one = lambda v: v[0] if isinstance(v, (tuple, list)) else v
    k, s, p = one(kernel_size), one(stride if stride is not None else kernel_size), one(padding)
    if n.kind != "conv" or (k, s, p) != (3, 2, 1) or one(dilation) != 1 or ceil_mode or return_indices or n.relu:
        raise NotImplementedError("integer max-pool is fused only as MaxPool2d(3,2,1) directly after a convolution")
    nb, c, hh, ww = n.shape
    shape = (nb, c, (hh + 2 - 3) // 2 + 1, (ww + 2 - 3) // 2 + 1)
    m = Node("conv", shape, mod=n.mod, src=n.src, a_sf=n.a_sf, pool=n.shape)
    return IntActivation(m, x.device)


def _add(a, b):
    if not (isinstance(a, IntActivation) and isinstance(b, IntActivation)):
        raise NotImplementedError("IntActivation + non-IntActivation")
    na, nb = a.node, b.node
    if na.kind != "conv" or na.relu or na.pool is not None:
        if nb.kind == "conv" and not nb.relu and nb.pool is None:
            na, nb = nb, na
        else:
            raise NotImplementedError("integer residual add expects conv_output + identity")
    if tuple(na.shape) != tuple(nb.shape):
        raise RuntimeError("shape mismatch in residual add: %s vs %s" % (na.shape, nb.shape))
    return IntActivation(Node("sum", na.shape, a=na, b=nb), a.device)


def _reshape(name, x, *shape, **kw):
    with torch._C.DisableTorchFunctionSubclass():
        meta = torch.empty(x.shape, device="meta")
        new = getattr(meta, name)(*shape, **kw).shape
    n = x.node
    if n.kind != "int" or len(n.shape) == 4 and (n.shape[2] != 1 or n.shape[3] != 1):
        if tuple(new) == tuple(x.shape):
            return x
        raise NotImplementedError("view() of an IntActivation is only supported on [N,C,1,1] -> [N,C]")
    return IntActivation(n, x.device, tuple(new))


# ------------------------------------------------------------------------------------------------ launches
def _desc(n, ent):
    nb, _, hh, ww = n.src.shape
    return ops.conv_desc(nb, hh, ww, ent["cin"], ent["cout"], ent["k"], ent["k"], ent["stride"], ent["pad"], n.src.bits, ent["w_layout"])


def _launch_conv(n, ent, ep, chan, **kw):
    if n.src.cs != ent["cin"]:
        raise RuntimeError("convolution input has %d stored channels, its weights %d" % (n.src.cs, ent["cin"]))
    if (n.src.shape[1], n.shape[1]) != (ent["cin"], ent["cout"]):      # padded channels: the timer also counts the logical bytes
        kw["logical"] = (n.src.shape[1], n.shape[1])
    ops.conv2d(n.src.data, _desc(n, ent), ep, ent["w"], chan, **kw)


def _check_src(n):
    s = n.src
    if s.kind != "int" or s.bits not in (4, 8):
        raise NotImplementedError("convolution input must be a concrete 4/8-bit IntActivation")
    if s.bits == 8 and not s.signed:
        raise NotImplementedError("8-bit unsigned (asymmetric) activations are not supported by the int8 kernels")


def _conv_case0(n, act, device):
    """conv [+ReLU] -> QuantAct case 0, one kernel."""
    _check_src(n)
    ent = _conv_cache(n.mod, n.a_sf, n.src.bits, device)
    if ent["kind"] in ("stem", "stem3"):
        raise NotImplementedError("the stem convolution is only supported as conv -> MaxPool2d(3,2,1) -> 16-bit QuantAct (ResNet) "
                                  "or conv -> ReLU6 -> 16-bit QuantAct (MobileNetV2)")
    m, e = _dyadic(act, n.a_sf, ent["w_sf"], "case0")
    lo, hi = _act_clamp(act)
    caps = (lambda: _relu6_caps(n, ent, m, e, hi)) if n.relu6 else None
    chan = _chan_tensor(ent, _act_tag("c0r6" if n.relu6 else "c0", act), m, e, device, caps)
    bits = _store_bits(act)
    if bits == 16 and not n.relu:
        bits = 32        # a signed 16-bit stream (MobileNetV2's quant_act_int32): 16-bit operands are read as uint16, so int32
    out = _new_int(device, n.shape, bits, _store_signed(act))
    relu = 2 if n.relu6 else n.relu
    if ent["kind"] == "dw":
        if n.src.cs != ent["cout"]:
            raise RuntimeError("depthwise input has %d stored channels, its weights %d" % (n.src.cs, ent["cout"]))
        nb, _, hh, ww = n.src.shape
        ops.dwconv3x3(n.src.data, nb, hh, ww, ent["cout"], ent["stride"], n.src.bits, ent["w"], chan, relu, bits, (lo, hi), out.data,
                      logical=(n.shape[1],))
        return out
    ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=bits, clamp=(lo, hi), flags=_ratio_flags((m, e)))
    _launch_conv(n, ent, ep, chan, out=out.data)
    return out


def _conv_raw(n, ent, device):
    """identity-branch conv: int32 accumulator + bias."""
    chan = _chan_tensor(ent, "raw", [0] * ent["cout"], [1] * ent["cout"], device, raw=True)
    out = _alloc(device, _stored_shape(n.shape), 32)
    _launch_conv(n, ent, ops.epilogue(EPI_RAW_I32, flags=_ratio_flags()), chan, out=out)
    return out


def _low_out(low_act, act, shape, device):
    """Output of the next QuantAct `low_act`, written by the producer of a residual stream at QuantAct `act`'s scale as its
    low-bit copy: (low_bits, low_me, low_clamp, Node 'int'), or no copy (0 bits, no Node) when low_act is None."""
    if low_act is None:
        return 0, (0, 1), (0, 0), None
    _frozen_scale(low_act)                 # refreshes low_act's scale, which _dyadic reads
    lm, le = _dyadic(low_act, _frozen_scale(act), _ones(), "case0")
    bits = _store_bits(low_act)
    node = _new_int(device, shape, bits, _store_signed(low_act))
    return bits, (lm[0], le[0]), _act_clamp(low_act), node


def _launch_residual(r, low_act, device):
    """'residual' node -> concrete residual stream (and optionally the next QuantAct's low-bit output)."""
    act, s = r.act, r.a
    conv, ident = s.a, s.b
    _check_src(conv)
    ent = _conv_cache(conv.mod, conv.a_sf, conv.src.bits, device)
    a_sf, w_sf, id_sf, id_w_sf = r.args
    m2, e2 = _dyadic(act, a_sf, w_sf, "case1-main")
    chan = _chan_tensor(ent, _act_tag("c1", act), m2, e2, device)
    id_conv = ident.kind == "conv"
    if id_conv:
        _check_src(ident)
        ient = _conv_cache(ident.mod, ident.a_sf, ident.src.bits, device)
        m1, e1 = _dyadic(act, id_sf, id_w_sf, "case1-idconv")
        res, res_chan = None, _chan_tensor(ient, _act_tag("c1res", act), m1, e1, device)
        res_kind, res_bits, res_me, id_pair = 1, 32, (0, 1), (m1, e1)
    else:
        ident = materialize(ident, device)
        if ident.bits not in (16, 32):
            raise NotImplementedError("identity operand must be the 16/32-bit residual stream")
        m1, e1 = _dyadic(act, id_sf, id_w_sf, "case1-id")
        res, res_chan = ident.data, None
        res_kind, res_bits, res_me = 0, ident.bits, (m1[0], e1[0])
        id_pair = res_me
    y_bits = config.residual_bits if r.relu else 32      # without ReLU (MobileNetV2) the stream is signed: int32
    y = _alloc(device, _stored_shape(r.shape), y_bits)
    low_bits, low_me, low_clamp, low = _low_out(low_act, act, r.shape, device)
    ep = ops.epilogue(EPI_RESIDUAL, relu=r.relu, res_kind=res_kind, res_bits=res_bits, res_me=res_me, y_bits=y_bits,
                      low_bits=low_bits, low_me=low_me, low_clamp=low_clamp, flags=_ratio_flags((m2, e2), id_pair, low_me))
    outs = dict(out=y, out_low=low.data if low is not None else None)
    # resize units: both 1x1 convolutions in one kernel when the fast uint16 stream is in use; without a ratio promise
    # (saturating generic kernels) they take two launches
    dual = (id_conv and config.dual and y_bits == 16 and ep.flags != 0 and conv.src.bits == ident.src.bits
            and ent["k"] == 1 and ent["stride"] == 1 and ent["pad"] == 0 and ient["k"] == 1 and ient["pad"] == 0)
    if dual:
        try:
            ops.conv2d_dual(conv.src.data, _desc(conv, ent), ep, ent["w"], chan, _desc(ident, ient), ident.src.data, ient["w"],
                            res_chan, **outs)
        except HawqError as err:
            if err.code != ERR_UNSUPPORTED:
                raise
            dual = False                           # the library declined this combination: two launches, same results
    if not dual:
        if id_conv:
            res = _conv_raw(ident, ient, device)
        _launch_conv(conv, ent, ep, chan, res=res, res_chan=res_chan, **outs)
    r.become_int(y, y_bits, signed=(y_bits == 32))
    return low


def _launch_stem(st, low_act, device):
    """'stem' node: 7x7 conv (+bias, 16-bit requant, ReLU) -> int16, then max-pool -> residual stream (+ low-bit copy); or the
    MobileNetV2 stem, 3x3/2 conv (+bias, ReLU6, 16-bit requant) -> stream (+ low-bit copy) in one kernel."""
    conv, act = st.a, st.act
    src = conv.src
    if src.kind != "int" or src.bits != 8 or not src.signed:
        raise NotImplementedError("stem input must be signed int8")
    ent = _conv_cache(conv.mod, conv.a_sf, 8, device)
    if ent["kind"] == "stem3":
        m, e = _dyadic(act, conv.a_sf, ent["w_sf"], "case0")
        lo, hi = _act_clamp(act)
        caps = (lambda: _relu6_caps(conv, ent, m, e, hi)) if conv.relu6 else None
        chan = _chan_tensor(ent, _act_tag("c0r6" if conv.relu6 else "c0", act), m, e, device, caps)
        y_bits = config.residual_bits if conv.relu else 32
        y = _alloc(device, _stored_shape(st.shape), y_bits)
        low_bits, low_me, low_clamp, low = _low_out(low_act, act, st.shape, device)
        nb, _, hh, ww = src.shape
        ops.stem3x3(src.data, ent["w"], chan, 2 if conv.relu6 else conv.relu, (lo, hi), nb, hh, ww, y_bits, y, low_bits, low_me,
                    low_clamp, low.data if low is not None else None, logical=(st.shape[1],))
        st.become_int(y, y_bits, signed=(y_bits == 32))
        return low
    if not st.relu:
        raise NotImplementedError("the fused stem expects the reference order conv -> pool -> QuantAct(16) -> ReLU")
    m, e = _dyadic(act, conv.a_sf, ent["w_sf"], "case0")
    chan = _chan_tensor(ent, _act_tag("c0", act), m, e, device)
    nb, _, hh, ww = src.shape
    ho, wo = conv.pool[2:]
    y_bits = config.residual_bits
    y = _alloc(device, st.shape, y_bits)
    low_bits, low_me, low_clamp, low = _low_out(low_act, act, st.shape, device)
    # two kernels (convolution -> int16, then max-pool + requant): measured faster on H100 than the one-kernel hawq_stem_pool_i8, whose
    # persistent tiles recompute the overlapping pool windows' convolution outputs (DESIGN.md §6)
    t16 = torch.empty(nb * ho * wo * 64, dtype=torch.int16, device=device)
    ops.stem_conv(src.data, ent["w"], chan, _act_clamp(act), t16, nb, hh, ww)
    ops.maxpool_requant(t16, nb, ho, wo, 64, y_bits, y, low_bits, low_me, low_clamp, low.data if low is not None else None)
    st.become_int(y, y_bits, signed=(y_bits == 32))
    return low


def materialize(n, device):
    """Force a node to concrete integers (launching its producer without further fusion)."""
    if n.kind == "int":
        return n
    if n.kind == "residual":
        _launch_residual(n, None, device)
        return n
    if n.kind == "stem":
        _launch_stem(n, None, device)
        return n
    raise NotImplementedError("a pending %s has no integer value before its QuantAct" % n.kind)


# ------------------------------------------------------------------------------------------------ module forwards
def _require_cuda(x, what):
    if not x.is_cuda:        # NotImplementedError (a RuntimeError): this path has no CPU implementation
        raise NotImplementedError("%s is frozen: its forward runs on the hawq_b200 CUDA kernels and needs a CUDA input "
                           "(got %s). Un-freeze the model for CPU calibration; there is no CPU fallback." % (what, x.device))


def act_forward(act, x, a_sf, w_sf, identity, id_sf, id_w_sf):
    """Frozen QuantAct.forward (reference quant_modules.py:205-303) on the integer path."""
    scale = _frozen_scale(act)
    dev = x.device
    if not isinstance(x, IntActivation):
        _require_cuda(x, "QuantAct")
        if a_sf is not None:
            raise NotImplementedError("a frozen QuantAct in the middle of a graph expects the IntActivation produced by "
                                      "the previous frozen module, not a float tensor")
        if x.dim() != 4:
            raise NotImplementedError("input quantisation expects NCHW")
        nb, c, hh, ww = x.shape
        lo, hi = _act_clamp(act)
        if act.activation_bit != 8 or act.quant_mode != "symmetric":
            raise NotImplementedError("network input quantisation is 8-bit symmetric in HAWQ ResNets")
        out = torch.empty(nb * hh * ww * c, dtype=torch.int8, device=dev)
        ops.quantize_input(x.contiguous().float(), float(scale), (lo, hi), out)
        return (IntActivation(Node("int", (nb, c, hh, ww), data=out, bits=8, signed=True), dev), scale)
    n = x.node
    if identity is not None:                                   # case 1: becomes a pending residual
        if n.kind != "sum":
            raise NotImplementedError("QuantAct with identity expects x = conv_output + identity")
        if w_sf is None:
            raise RuntimeError("case 1 needs the weight scaling factor of the last convolution")
        if id_w_sf is None:
            id_w_sf = _ones()
        r = Node("residual", n.shape, a=n, act=act, args=(a_sf, w_sf, id_sf, id_w_sf))
        return (IntActivation(r, dev), scale)
    if a_sf is None:                                           # already-quantised input handed in by the caller
        if n.kind != "int":
            raise NotImplementedError("QuantAct without a previous scale expects concrete integers")
        return (x, scale)
    if n.kind == "conv":
        stem3 = _conv_cache(n.mod, n.a_sf, n.src.bits if n.src.bits in (4, 8) else 8, dev)["kind"] == "stem3"
        if n.pool is not None or stem3:                        # stem: conv -> pool -> QuantAct(16) [-> ReLU], conv -> ReLU6 -> QuantAct(16)
            st = Node("stem", n.shape, a=n, act=act)
            if act.activation_bit != 16:
                raise NotImplementedError("the stem convolution must be followed by the 16-bit quant_act_int32")
            return (IntActivation(st, dev), scale)
        return (IntActivation(_conv_case0(n, act, dev), dev), scale)
    if n.kind in ("residual", "stem"):                         # fuse this activation into the producer's epilogue
        low = (_launch_residual if n.kind == "residual" else _launch_stem)(n, act, dev)
        return (IntActivation(low, dev), scale)
    if n.kind == "avgpool":
        src = materialize(n.src, dev)
        m, e = _dyadic(act, a_sf, _ones(), "case0")
        lo, hi = _act_clamp(act)
        nb, c, hh, ww = src.shape
        if act.activation_bit != 8 or act.quant_mode != "symmetric":
            raise NotImplementedError("the pooled tail is 8-bit symmetric in HAWQ ResNets")
        out = _new_int(dev, (nb, c, 1, 1), 8, True)
        ops.avgpool_requant(src.data, nb, hh * ww, src.cs, src.bits, (m[0], e[0]), (lo, hi), out.data)
        return (IntActivation(out, dev), scale)
    if n.kind == "int":                                        # stand-alone requant of the residual stream
        if n.bits not in (16, 32):
            raise NotImplementedError("stand-alone requantisation expects the 16/32-bit residual stream")
        ws = w_sf if w_sf is not None else _ones()
        m, e = _dyadic(act, a_sf, ws, "case0")
        per_ch = len(m) > 1
        ck = ("chan", _key(a_sf), _key(ws), n.cs, str(dev))    # cached with the (m, e) pairs: no host copy inside graph capture
        chan = act._hawq_cache["me"].get(ck)
        if chan is None:
            m, e = _pad_me(m, e, n.cs)
            chan = act._hawq_cache["me"][ck] = ops.make_chan([0] * len(m), m, e).to(dev)
        rows = int(np.prod(n.shape)) // n.shape[1]
        lo, hi = _act_clamp(act)
        out = _new_int(dev, n.shape, _store_bits(act), _store_signed(act))
        ops.requant(n.data, rows, n.cs, n.bits, chan, 1 if per_ch else 0, False, _store_bits(act), (lo, hi), out.data)
        return (IntActivation(out, dev), scale)
    raise NotImplementedError("QuantAct on a pending %s" % n.kind)


def conv_forward(mod, x, a_sf):
    """Frozen QuantBnConv2d / QuantConv2d forward: records a pending convolution (launched by its consumer)."""
    if not isinstance(x, IntActivation):
        _require_cuda(x, type(mod).__name__)
        raise NotImplementedError("a frozen %s expects the IntActivation produced by a frozen QuantAct" % type(mod).__name__)
    if a_sf is None:
        raise ValueError("pre_act_scaling_factor is required")
    src = materialize(x.node, x.device)
    from .modules import QuantConv2d
    if type(mod) is QuantConv2d and tuple(mod.conv.kernel_size) == (1, 1) and tuple(src.shape[2:]) == (1, 1):
        # a 1x1 QuantConv2d on [N,C,1,1] with no QuantAct behind it (MobileNetV2's `output`): the classifier, fp32
        # float(acc + bias) * (w_sf_c * a_sf) as the reference's (out * bias_sf, w_sf) (quant_modules.py:718,726-736)
        ent = _linear_plan(mod, a_sf, x.device)
        logits = _linear_logits(src, ent)
        return (logits.view(src.shape[0], -1, 1, 1), ent["w_sf"])
    ent = _conv_cache(mod, a_sf, 8 if src.bits not in (4, 8) else src.bits, x.device)
    nb, _, hh, ww = src.shape
    ho = (hh + 2 * ent["pad"] - ent["k"]) // ent["stride"] + 1
    wo = (ww + 2 * ent["pad"] - ent["k"]) // ent["stride"] + 1
    n = Node("conv", (nb, ent["cout_l"], ho, wo), mod=mod, src=src, a_sf=a_sf)
    return (IntActivation(n, x.device), ent["w_sf"])


def linear_forward(mod, x, a_sf):
    """Frozen QuantLinear.forward (quant_modules.py:79-130) -> fp32 logits (a real torch tensor)."""
    if not isinstance(x, IntActivation):
        _require_cuda(x, "QuantLinear")
        raise NotImplementedError("a frozen QuantLinear expects the IntActivation produced by a frozen QuantAct")
    return _linear_logits(materialize(x.node, x.device), _linear_plan(mod, a_sf, x.device))


def _linear_plan(mod, a_sf, dev):
    return _plan(mod, a_sf, dev, (mod.weight_bit, mod.per_channel), lambda: _linear_params(mod, a_sf, dev))


def _linear_logits(n, ent):
    """fp32 [N, Cout] logits of the classifier plan `ent` on concrete int8 features n (hawq_linear_i8)."""
    if n.bits != 8 or not n.signed:
        raise NotImplementedError("classifier input must be signed int8")
    if n.cs != ent["k"]:
        raise RuntimeError("classifier input has %d stored features, its weights %d" % (n.cs, ent["k"]))
    nb = n.shape[0]
    out = torch.empty((nb, ent["cout"]), dtype=torch.float32, device=n.data.device)
    ops.linear(n.data, ent["w"], ent["chan"], ent["fscale"], out, nb, ent["k"], ent["cout"], ent["cpad"])
    return out


def _linear_params(mod, a_sf, dev):
    """QuantLinear, or a 1x1 QuantConv2d used as the classifier (weights [Cout, K, 1, 1])."""
    w_sf, w_int, b_int, bias_sf = mod.integer_params(a_sf.to(mod.weight.device))
    cout = w_int.shape[0]
    k = w_int[0].numel()
    if k % 64 != 0:
        raise NotImplementedError("QuantLinear in_features must be a multiple of 64")
    cpad = (cout + 63) // 64 * 64
    w = torch.zeros((cpad, k), dtype=torch.int8)
    w[:cout] = w_int.detach().to("cpu").reshape(cout, k).to(torch.int8)
    bias = np.zeros(cpad, dtype=np.int64)
    if b_int is not None:
        bias[:cout] = b_int.detach().to("cpu").to(torch.int64).numpy()
    fs = torch.zeros(cpad, dtype=torch.float32)
    fs[:cout] = bias_sf.detach().to("cpu", torch.float32).reshape(-1)   # fc_scaling_factor * act scale, fp32
    # a dead row (all weights 0) may hold the bias 2^31 (ops.make_chan); its logit float(2^31) * fs is stored as float(2^30) * 2 fs,
    # the same fp32 value
    dead = (bias >= 2 ** 31) & ~w.any(dim=1).numpy() & (bias % 2 == 0)
    bias[dead] //= 2
    fs[torch.from_numpy(dead)] *= 2
    return dict(w=w.to(dev), chan=ops.make_chan(bias, [0] * cpad, [1] * cpad, raw=True).to(dev), fscale=fs.to(dev), cout=cout, cpad=cpad, k=k,
                w_sf=w_sf.detach().to("cpu", torch.float32))


def avgpool_forward(mod, x, sf):
    n = x.node
    shape = n.shape
    if len(shape) != 4 or mod.kernel_size != shape[2] or shape[2] != shape[3] or mod.padding != 0:
        raise NotImplementedError("integer average pooling is global (kernel == feature map)")
    p = Node("avgpool", (shape[0], shape[1], 1, 1), src=n)
    return (IntActivation(p, x.device), sf.view(-1) if sf is not None else sf)
