"""Thin Python layer over the C ABI: torch tensors in, raw device pointers + the current CUDA stream out.

torch is used only as the owner of device memory and streams.  Every function launches asynchronously on
``torch.cuda.current_stream()`` and never synchronises, so sequences of calls can be captured in a CUDA graph.
There is no fallback: tensors must live on a CUDA device and the in-tree library must load.

Status words: every launch raises its sticky flags in the status word of a handle (hawq_create).  By default that is one handle
per device, shared by the process.  ``using_handle`` scopes another handle to the calling thread, so that an engine
(``CompiledModel``) owns its own word and engines that run at the same time on other streams or threads never see each
other's flags.
"""
import contextlib
import ctypes as C
import threading

import numpy as np
import torch

from . import _lib
from ._lib import EPI_RAW_I32, EPI_REQUANT, EPI_RESIDUAL, hawq_conv_desc, hawq_epilogue_desc

_handles = {}                  # device index -> the default handle
_handles_lock = threading.Lock()
_spare = {}                    # device index -> handles released by their owners, reused by acquire_handle
_local = threading.local()     # per thread: the handle in scope (using_handle) and the launch counter


def _create(device_index):
    out = C.c_void_p()
    _lib.check(_lib.load().hawq_create(int(device_index), C.byref(out)))
    return out


def handle(device_index):
    """The handle ops on device `device_index` use on this thread: the one in scope (using_handle), else the device's default."""
    cur = getattr(_local, "handle", None)
    if cur is not None and cur[0] == device_index:
        return cur[1]
    h = _handles.get(device_index)
    if h is None:
        with _handles_lock:
            h = _handles.get(device_index)
            if h is None:
                h = _handles[device_index] = _create(device_index)
    return h


def acquire_handle(device_index):
    """A handle of its own (its own status word) on device `device_index`, for as long as the caller holds it.  Give it back
    with release_handle; it is then reused rather than destroyed, because hawq_destroy synchronises the device."""
    with _handles_lock:
        spare = _spare.get(device_index)
        if spare:
            return spare.pop()
    return _create(device_index)


def release_handle(device_index, h):
    """Returns a handle from acquire_handle.  Its next owner (a CompiledModel) synchronises the device while it builds, before any
    forward whose status word it reads, and resets the word at the start of each, so work still queued by the last owner cannot
    reach it."""
    with _handles_lock:
        _spare.setdefault(device_index, []).append(h)


@contextlib.contextmanager
def using_handle(device_index, h):
    """Every op this thread runs on device `device_index` inside the block uses handle `h` (nested scopes restore the outer one)."""
    saved = getattr(_local, "handle", None)
    _local.handle = (device_index, h)
    try:
        yield h
    finally:
        _local.handle = saved


def thread_launch_count():
    """Kernels launched through this module by the calling thread (CompiledModel reports them as gpu_launches)."""
    return getattr(_local, "launches", 0)


def _ctx(t):
    if not t.is_cuda:
        raise RuntimeError("hawq_b200 integer ops need CUDA tensors (got %s); there is no CPU path" % t.device)
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    return handle(idx), C.c_void_p(torch.cuda.current_stream(idx).cuda_stream)


class _Ptr(C.c_void_p):
    """The device pointer of a tensor while this thread records launches (``recording``), with its storage's (base, bytes)."""


def _p(t):
    if t is None:
        return None
    if getattr(_local, "recorder", None) is None:
        return C.c_void_p(t.data_ptr())
    p = _Ptr(t.data_ptr())
    s = t.untyped_storage()
    p.storage = (s.data_ptr(), s.nbytes())
    return p


timer = None   # set to a list to record (kernel, info, start_event, end_event) per launch (bench.py roofline leg)


@contextlib.contextmanager
def recording():
    """Every launch this thread makes inside the block is appended to the yielded list as (entry point, arguments) (engine_file.py
    turns them into a plan file).  An argument is ("i32" | "u32" | "i64" | "f32", value), ("null",), ("ptr", address, storage base,
    storage bytes) (base and bytes None when the pointer did not come from a tensor), or ("blob", bytes) for a struct or array passed by
    pointer, by value.  The handle and the stream are implicit."""
    saved = getattr(_local, "recorder", None)
    _local.recorder = rec = []
    try:
        yield rec
    finally:
        _local.recorder = saved


_ARG_KINDS = {_lib._i32: "i32", _lib._u32: "u32", _lib._i64: "i64", _lib._f32: "f32"}


def _recorded(fn, args):
    out = []
    for a, ctype in zip(args, _lib.SIGNATURES[fn][1][1:-1]):
        if ctype is C.c_void_p:
            v = a.value if isinstance(a, C.c_void_p) else a
            out.append(("null",) if v is None else ("ptr", v) + getattr(a, "storage", (None, None)))
        elif ctype in _ARG_KINDS:
            out.append((_ARG_KINDS[ctype], a.value if isinstance(a, C._SimpleCData) else a))
        else:
            out.append(("blob", bytes(getattr(a, "_obj", a))))
    return fn, out


def _launch(t, fn, *args, label=None, work=None):
    """Calls ABI entry point `fn`(handle, *args, stream) on the device and current stream of tensor `t` and counts the launch.
    While `timer` is set, a launch with a `label` is bracketed by CUDA events and recorded with `work()`, its (MACs, bytes)."""
    h, s = _ctx(t)
    ev0 = None
    if label is not None and timer is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev0.record()
    _lib.check(getattr(_lib.load(), fn)(h, *args, s))
    _local.launches = thread_launch_count() + 1
    rec = getattr(_local, "recorder", None)
    if rec is not None:
        rec.append(_recorded(fn, args))
    if ev0 is not None:
        info = work()
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        timer.append((label, info, ev0, ev1))


def conv_work(desc, ep):
    """(MACs, algorithmic HBM bytes) of one fused convolution launch: activations in at their stored width (only the
    sampled pixels for strided 1x1), weights + per-channel parameters once, every output at its stored width, plus the
    residual operand for case-1 epilogues."""
    ho = (desc.H + 2 * desc.pad - desc.kh) // desc.stride + 1
    wo = (desc.W + 2 * desc.pad - desc.kw) // desc.stride + 1
    m = desc.N * ho * wo
    macs = m * desc.Cout * desc.kh * desc.kw * desc.Cin
    in_pix = m if desc.kh == 1 else desc.N * desc.H * desc.W
    b = in_pix * desc.Cin * desc.a_bits // 8 + desc.Cout * desc.kh * desc.kw * desc.Cin + 16 * desc.Cout
    outs = m * desc.Cout
    if ep.mode == EPI_REQUANT:
        b += outs * ep.out_bits // 8
    elif ep.mode == EPI_RESIDUAL:
        b += outs * (4 if ep.res_kind == 1 else ep.res_bits // 8) + outs * ep.y_bits // 8 + outs * ep.low_bits // 8
        if ep.res_kind == 1:
            b += 16 * desc.Cout
    elif ep.mode == EPI_RAW_I32:
        b += outs * 4
    else:
        b += m * ep.cout_store * 4 + 4 * desc.Cout
    return macs, b


def make_chan(bias, m, e, cap=None, zero_acc=None, raw=False):
    """hawq_chan[C] as an int32 [C,4] CPU tensor (m stored by bit pattern; `cap`: the ReLU6 output caps of relu 2, in reserved;
    `raw`: the table of a RAW_I32 or classifier launch, whose acc + bias is stored as is and m, e are unused).

    A bias outside int32 is never wrapped.  The reference's 32-bit bias quantiser clamps to [-2^31, 2^31 - 1] in fp32, where
    2^31 - 1 rounds to 2^31: a "dead" channel (all weights 0, its weight scale clamped to 1e-8 / n) with a positive folded bias gets
    exactly 2^31.  Its accumulator is identically 0 (`zero_acc[c]`), so a requantising table gives it RHE(2^31 * m / 2^e) from the
    bias alone, which is stored exactly: with m = 0 (a ratio below 2^-62, flushed by dyadic()) that is 0 for any bias, and bias 0 is
    stored; otherwise (bias / 2, m, e - 1), only while e - 1 >= 31, so that every ratio promise made from the original (m, e) pairs
    (ratio_flags) still holds.  Any other bias outside int32 raises OverflowError."""
    c = len(bias)
    b = np.array([int(v) for v in bias], dtype=object)
    m = np.broadcast_to(np.asarray(m, dtype=np.uint64), (c,)).astype(np.uint64)
    e = np.broadcast_to(np.asarray(e, dtype=np.int64), (c,)).astype(np.int64)
    for i in np.nonzero([not -2 ** 31 <= v < 2 ** 31 for v in b])[0]:
        exact = zero_acc is not None and zero_acc[i] and not raw
        if exact and m[i] == 0:
            b[i] = 0
        elif exact and e[i] >= 32 and b[i] % 2 == 0 and -2 ** 31 <= b[i] // 2 < 2 ** 31:
            b[i] //= 2
            e[i] -= 1
        else:
            raise OverflowError("bias integer %d of channel %d leaves int32 (m = %d, e = %d, accumulator %s)"
                                % (b[i], i, m[i], e[i], "identically 0" if zero_acc is not None and zero_acc[i] else "not known to be 0"))
    a = np.zeros((c, 4), dtype=np.int32)
    a[:, 0] = b.astype(np.int64)
    a[:, 1] = m.astype(np.uint32).view(np.int32)
    a[:, 2] = e.astype(np.int32)
    if cap is not None:
        a[:, 3] = np.asarray(cap, dtype=np.int64).astype(np.int32)
    return torch.from_numpy(a)


def rhe_requant_host(v, m, e):
    """RHE(v * m / 2^e) of one int32 value, exact (the library's host helper, the routine the kernels inline)."""
    return int(_lib.load().hawq_rhe_requant_host(int(v), int(m), int(e)))


def conv_desc(N, H, W, Cin, Cout, kh, kw, stride, pad, a_bits, w_layout=0):
    return hawq_conv_desc(N, H, W, Cin, Cout, kh, kw, stride, pad, a_bits, w_layout)


def upload_weights(w_ohwi_cpu, device):
    """int8 OHWI host weights -> device buffer [OHWI | re-tiled copy] (hawq_conv_desc.w_layout = 1)."""
    cout = w_ohwi_cpu.shape[0]
    k = w_ohwi_cpu.numel() // cout
    buf = torch.empty(2 * cout * k, dtype=torch.int8, device=device)
    buf[:cout * k].copy_(w_ohwi_cpu.reshape(-1))
    idx = buf.device.index if buf.device.index is not None else torch.cuda.current_device()
    _lib.check(_lib.load().hawq_retile_weights(handle(idx), C.c_void_p(buf.data_ptr()), cout, k, C.c_void_p(buf.data_ptr() + cout * k),
                                               C.c_void_p(torch.cuda.current_stream(idx).cuda_stream)))
    return buf


def epilogue(mode, relu=0, out_bits=0, clamp=(0, 0), res_kind=0, res_bits=0, res_me=(0, 1), y_bits=0, low_bits=0,
             low_me=(0, 1), low_clamp=(0, 0), cout_store=0, flags=0):
    return hawq_epilogue_desc(mode, int(relu), out_bits, clamp[0], clamp[1], res_kind, res_bits, res_me[0], res_me[1],
                              y_bits, low_bits, low_me[0], low_me[1], low_clamp[0], low_clamp[1], cout_store, flags)


def ratio_flags(*pairs):
    """HAWQ_EP_RATIOS_* promise for a set of (m, e) pairs (or (m list, e list)): LE_ONE when every ratio m * 2^-e <= 1
    (e >= 31 or m == 0), LE_2P20 when every ratio <= 2^20 (e >= 11), else 0.  (Whether the promise is made at all is the
    caller's execution mode: qtensor.EngineConfig.)"""
    min_e = 99
    for m, e in pairs:
        ms = m if isinstance(m, (list, tuple)) else [m]
        es = e if isinstance(e, (list, tuple)) else [e]
        for mi, ei in zip(ms, es):
            if mi != 0:
                min_e = min(min_e, ei)
    if min_e >= 31:
        return _lib.EP_RATIOS_LE_ONE
    if min_e >= 11:
        return _lib.EP_RATIOS_LE_2P20
    return 0


def _with_logical(work, logical_work, logical):
    """work() -> (MACs, bytes) at the stored (padded) channel counts; with `logical` (the model's channel counts) a third entry,
    the bytes at the logical counts, so that the cost of padding is visible."""
    if logical is None:
        return work
    return lambda: tuple(work()) + (logical_work(*logical)[1],)


def conv2d(x, desc, ep, w, chan, res=None, res_chan=None, fscale=None, out=None, out_low=None, logical=None):
    """`logical`: (Cin, Cout) of the model when the descriptor's are padded (timer work only)."""
    def logical_work(cin, cout):
        d = hawq_conv_desc(*[getattr(desc, f) for f, _ in hawq_conv_desc._fields_])
        d.Cin, d.Cout = cin, cout
        return conv_work(d, ep)
    _launch(x, "hawq_conv2d", C.byref(desc), C.byref(ep), _p(x), _p(w), _p(chan), _p(res), _p(res_chan), _p(fscale), _p(out),
            _p(out_low), label="conv_igemm", work=_with_logical(lambda: conv_work(desc, ep), logical_work, logical))


def dwconv3x3(x, n, hh, ww, c, stride, a_bits, w, chan, relu, out_bits, clamp, out, logical=None):
    """Depthwise 3x3 pad 1 + case-0 requant (hawq_dwconv3x3); `logical`: (C,) of the model when c is padded (timer work only)."""
    ho, wo = (hh - 1) // stride + 1, (ww - 1) // stride + 1

    def work(cc):
        return n * ho * wo * cc * 9, n * hh * ww * cc * a_bits // 8 + 9 * cc + 16 * cc + n * ho * wo * cc * out_bits // 8
    _launch(x, "hawq_dwconv3x3", n, hh, ww, c, stride, a_bits, _p(x), _p(w), _p(chan), int(relu), out_bits, clamp[0], clamp[1], _p(out),
            label="dwconv3x3", work=_with_logical(lambda: work(c), work, logical))


def stem3x3(x, w, chan, relu, clamp, n, hh, ww, y_bits, y, low_bits, low_me, low_clamp, out_low, logical=None):
    """MobileNetV2 stem: 3x3/2 convolution of 3 channels -> 64 stored channels + requant (hawq_stem3x3_i8), optional low-bit copy;
    `logical`: (Cout,) of the model (timer work only)."""
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1

    def work(cc):
        return n * ho * wo * cc * 27, n * hh * ww * 3 + cc * 36 + 16 * cc + n * ho * wo * cc * (y_bits + low_bits) // 8
    _launch(x, "hawq_stem3x3_i8", n, hh, ww, _p(x), _p(w), _p(chan), int(relu), clamp[0], clamp[1], y_bits, _p(y), low_bits, low_me[0],
            low_me[1], low_clamp[0], low_clamp[1], _p(out_low), label="stem3x3", work=_with_logical(lambda: work(64), work, logical))


def conv2d_dual(x, desc, ep, w, chan, desc2, x2, w2, chan2, out=None, out_low=None):
    """resize unit: identity 1x1 conv (desc2/x2/w2/chan2) + last 1x1 conv (desc/x/w/chan) + case-1 sum in one kernel."""
    def work():
        m = desc.N * desc.H * desc.W
        macs = m * desc.Cout * (desc.Cin + desc2.Cin)
        b = (m * (desc.Cin + desc2.Cin) * desc.a_bits // 8 + desc.Cout * (desc.Cin + desc2.Cin) + 32 * desc.Cout
             + m * desc.Cout * (ep.y_bits + ep.low_bits) // 8)
        return macs, b
    _launch(x, "hawq_conv2d_dual", C.byref(desc), C.byref(ep), _p(x), _p(w), _p(chan), C.byref(desc2), _p(x2), _p(w2), _p(chan2),
            _p(out), _p(out_low), label="conv_dual", work=work)


def linear(x, w, chan, fscale, out, n, k, cout, cout_pad):
    _launch(x, "hawq_linear_i8", n, k, cout, cout_pad, _p(x), _p(w), _p(chan), _p(fscale), _p(out), label="hawq_linear",
            work=lambda: (n * k * cout, n * k + cout_pad * k + 20 * cout_pad + n * cout * 4))


def stem_conv(x, w, chan, clamp, out, n, hh, ww):
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    _launch(x, "hawq_stem_conv_i8", n, hh, ww, _p(x), _p(w), _p(chan), clamp[0], clamp[1], _p(out), label="stem_conv",
            work=lambda: (n * ho * wo * 64 * 147, n * hh * ww * 3 + 64 * 224 + 1024 + n * ho * wo * 64 * 2))


def stem_pool(x, w256, chan, clamp, n, hh, ww, y_bits, y, low_bits, low_me, low_clamp, out_low):
    """Fused stem (conv 7x7/2 + max-pool 3x3/2 + 16-bit requant + ReLU + low-bit copy) in one kernel; raises HawqError(ERR_UNSUPPORTED)
    for shapes / ratios outside it (callers then use stem_conv + maxpool_requant, same integers)."""
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    po, qo = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    _launch(x, "hawq_stem_pool_i8", n, hh, ww, _p(x), _p(w256), _p(chan), clamp[0], clamp[1], y_bits, _p(y), low_bits, low_me[0],
            low_me[1], low_clamp[0], low_clamp[1], _p(out_low), label="stem_pool",
            work=lambda: (n * ho * wo * 64 * 147, n * hh * ww * 3 + 64 * 256 + 1024 + n * po * qo * 64 * (y_bits + low_bits) // 8))


def maxpool_requant(x, n, hh, ww, c, y_bits, y, low_bits, low_me, low_clamp, out_low):
    po, qo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    _launch(x, "hawq_maxpool_requant", n, hh, ww, c, _p(x), y_bits, _p(y), low_bits, low_me[0], low_me[1], low_clamp[0],
            low_clamp[1], _p(out_low), label="maxpool_requant",
            work=lambda: (0, n * hh * ww * c * 2 + n * po * qo * c * (y_bits + low_bits) // 8))


def avgpool_requant(x, n, hw, c, x_bits, me, clamp, out):
    _launch(x, "hawq_avgpool_requant", n, hw, c, x_bits, _p(x), me[0], me[1], clamp[0], clamp[1], _p(out), label="avgpool_requant",
            work=lambda: (0, n * hw * c * x_bits // 8 + n * c))


def quantize_input(x, scale, clamp, out):
    n, c, hh, ww = x.shape
    _launch(x, "hawq_quantize_input_f32", n, c, hh, ww, _p(x), float(scale), clamp[0], clamp[1], _p(out), label="quantize_input",
            work=lambda: (0, n * c * hh * ww * 5))


def quantize_input_u8(x, mean, std, scale, clamp, out):
    """uint8 NHWC images -> int8 NHWC network input (ToTensor + Normalize + QuantAct input branch in one kernel)."""
    n, hh, ww, c = x.shape
    if c != 3:
        raise ValueError("quantize_input_u8 expects NHWC images with 3 channels")
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    _launch(x, "hawq_quantize_input_u8", n, hh, ww, _p(x), m3, s3, float(scale), clamp[0], clamp[1], _p(out),
            label="quantize_input_u8", work=lambda: (0, n * hh * ww * 6))


def resize_crop_quantize_u8(pixels, table, size, crop, mean, std, scale, clamp, out):
    """Ragged uint8 HWC images -> int8 NHWC [B, Ch, Cw, 3] network input: Resize(size) + CenterCrop(crop) (torchvision on PIL, bit for
    bit) + ToTensor + Normalize + QuantAct input branch in one kernel.  pixels: the uint8 arena; table: int64 [B, 2] hawq_image_desc
    rows (eval_transform.PackedImages.table) on the device.  Timer work: the source bytes the crops read plus the output bytes."""
    ch, cw = crop
    b = table.shape[0]
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])

    def work():
        from .eval_transform import source_box
        t = table.cpu()
        read = 0
        for off, h, w in zip(t[:, 0].tolist(), t.view(torch.int32)[:, 2].tolist(), t.view(torch.int32)[:, 3].tolist()):
            if h > 0:
                (_, rows), (_, cols) = source_box(h, w, size, crop)
                read += rows * cols * 3
        return 0, read + b * ch * cw * 3
    _launch(pixels, "hawq_resize_crop_quantize_u8", b, _p(pixels), pixels.numel(), _p(table), size, ch, cw, m3, s3, float(scale), clamp[0],
            clamp[1], _p(out), label="resize_crop_quantize_u8", work=work)


def requant(x, rows, c, x_bits, chan, chan_stride, relu, out_bits, clamp, out):
    _launch(x, "hawq_requant", rows, c, x_bits, _p(x), _p(chan), chan_stride, int(relu), out_bits, clamp[0], clamp[1], _p(out))


def add_requant(acc, rows, c, chan, ep, res, res_chan, y, out_low):
    _launch(acc, "hawq_add_requant", rows, c, _p(acc), _p(chan), C.byref(ep), _p(res), _p(res_chan), _p(y), _p(out_low))


def dequant(x, n, hh, ww, c, x_bits, x_signed, scale, out):
    _launch(x, "hawq_dequant_f32", n, hh, ww, c, x_bits, int(x_signed), _p(x), float(scale), _p(out))


def pack_i4(src, dst):
    _launch(src, "hawq_pack_i4", src.numel(), _p(src), _p(dst))


def unpack_i4(src, dst):
    _launch(src, "hawq_unpack_i4", dst.numel(), _p(src), _p(dst))


def reset_status(device_index):
    h = handle(device_index)
    _lib.check(_lib.load().hawq_reset_status(h, C.c_void_p(torch.cuda.current_stream(device_index).cuda_stream)))


def copy_status(device_index, dst):
    h = handle(device_index)
    _lib.check(_lib.load().hawq_copy_status(h, _p(dst), C.c_void_p(torch.cuda.current_stream(device_index).cuda_stream)))


def get_status(device_index):
    h = handle(device_index)
    v = C.c_int32()
    _lib.check(_lib.load().hawq_get_status(h, C.c_void_p(torch.cuda.current_stream(device_index).cuda_stream), C.byref(v)))
    return int(v.value)


def permute_weights_for_i4(w_ohwi_int8):
    """In-place K permutation (host, contiguous int8 [Cout, kh, kw, Cin])."""
    assert w_ohwi_int8.dtype == torch.int8 and w_ohwi_int8.is_contiguous() and not w_ohwi_int8.is_cuda
    cin = w_ohwi_int8.shape[-1]
    _lib.check(_lib.load().hawq_permute_weights_for_i4(C.c_void_p(w_ohwi_int8.data_ptr()),
                                                       w_ohwi_int8.numel() // cin, cin))
    return w_ohwi_int8
