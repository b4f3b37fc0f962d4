"""Engine files: a compiled forward saved to one file and run without the model, its checkpoint or Python.

``CompiledModel.save(path)`` records one eager forward per sequence at the level of the C ABI (``ops.recording``): every launch as
(entry point, arguments).  Each pointer argument is resolved to one of four regions: the input binding (``static_in``), the output
binding (the logits), the constants (storages of the modules' plan caches: weights, per-channel tables, classifier scales, stored
in the file) and the arena (every other buffer the forward touches).  The library's runtime (``hawq_engine_load``,
include/hawq_b200.h) captures each sequence into a CUDA graph that calls the same entry points with the same arguments, so a loaded
engine runs the same kernels on the same integers as the CompiledModel it was saved from.  The format is documented in the header.

``load_engine(path)`` wraps that runtime; it needs neither the model code nor torch beyond the tensors it returns.
"""
import ctypes as C
import struct
import zlib

import torch

from . import _lib

ALIGN = 512                                     # torch's allocation alignment, which the 16-byte vector and cp.async paths rely on
SEQ_FAST, SEQ_INT32, SEQ_SAFE = 0, 1, 2         # enum hawq_engine_seq
REGIONS = {"input": 0, "output": 1, "const": 2, "arena": 3}          # enum hawq_engine_region
ARG_KINDS = {"i32": 1, "u32": 2, "i64": 3, "f32": 4, "null": 5, "ptr": 6, "blob": 7}   # enum hawq_engine_arg
DTYPES = {torch.int8: 0, torch.uint8: 1, torch.float32: 2}           # enum hawq_engine_dtype
_HEADER = struct.Struct("<8sIIIIQII")


class UnresolvedPointer(ValueError):
    pass


def arg_codes(fn):
    """The argument signature of entry point `fn` without handle and stream, in the runtime's alphabet (engine_file.cu kEntryArgs):
    i int32, u uint32, I int64, f float, p pointer, D hawq_conv_desc, E hawq_epilogue_desc, F float[3]."""
    codes = {_lib._i32: "i", _lib._u32: "u", _lib._i64: "I", _lib._f32: "f", C.c_void_p: "p",
             C.POINTER(_lib.hawq_conv_desc): "D", C.POINTER(_lib.hawq_epilogue_desc): "E", C.POINTER(_lib._f32): "F"}
    return "".join(codes[t] for t in _lib.SIGNATURES[fn][1][1:-1])


def _align(n):
    return (n + ALIGN - 1) // ALIGN * ALIGN


def arena_layout(intervals):
    """{storage base: bytes} of the scratch storages -> ({storage base: arena offset}, arena bytes).  Overlapping address intervals
    merge into one segment whose bytes keep their relative positions, so two storages share arena bytes exactly where they shared
    device memory in the recorded run (which was valid); each segment starts at a 512-byte-aligned offset."""
    segs = []                                    # [first address, end, member bases]
    for base, n in sorted(intervals.items()):
        if segs and base < segs[-1][1]:
            segs[-1][1] = max(segs[-1][1], base + n)
            segs[-1][2].append(base)
        else:
            segs.append([base, base + n, [base]])
    place, size = {}, 0
    for start, end, members in segs:
        off = _align(size)
        for b in members:
            place[b] = off + b - start
        size = off + end - start
    return place, size


def resolve(records, inp, out, const):
    """Recorded launches (ops.recording) -> (records with every pointer as ("ptr", region, offset), arena bytes).

    inp / out: (base, bytes) of the input and output storages; const: {storage base: offset in the constants region}.  Every other
    storage is scratch and goes to the arena (arena_layout).  A pointer without a storage, or outside its storage, raises
    UnresolvedPointer naming the entry point and the argument (numbered as in the C prototype, the handle being argument 0)."""
    scratch = {}
    for fn, args in records:
        for i, a in enumerate(args):
            if a[0] != "ptr":
                continue
            _, addr, base, n = a
            if base is None or not base <= addr < base + max(n, 1):
                raise UnresolvedPointer("%s argument %d: pointer 0x%x belongs to no tensor storage the engine can place" % (fn, i + 1, addr))
            if base not in (inp[0], out[0]) and base not in const:
                scratch[base] = max(scratch.get(base, 0), n)
    place, arena = arena_layout(scratch)
    resolved = []
    for fn, args in records:
        new = []
        for a in args:
            if a[0] == "ptr":
                _, addr, base, _ = a
                if base == inp[0]:
                    region, off = "input", 0
                elif base == out[0]:
                    region, off = "output", 0
                elif base in const:
                    region, off = "const", const[base]
                else:
                    region, off = "arena", place[base]
                a = ("ptr", region, off + addr - base)
            new.append(a)
        resolved.append((fn, new))
    return resolved, arena


def _encode_arg(a):
    kind = ARG_KINDS[a[0]]
    if a[0] == "i32":
        return struct.pack("<Bi", kind, a[1])
    if a[0] == "u32":
        return struct.pack("<BI", kind, a[1])
    if a[0] == "i64":
        return struct.pack("<Bq", kind, a[1])
    if a[0] == "f32":
        return struct.pack("<Bf", kind, a[1])
    if a[0] == "null":
        return struct.pack("<B", kind)
    if a[0] == "ptr":
        return struct.pack("<BBQ", kind, REGIONS[a[1]], a[2])
    return struct.pack("<BI", kind, len(a[1])) + a[1]


def plan_bytes(input_dtype, input_shape, output_shape, residual_bits, constants, arena_bytes, sequences):
    """A plan file: input binding (torch dtype, 4-d shape), output binding [N, classes] fp32, residual bits of the fast sequence,
    the constants region (bytes), the arena size and {sequence kind: resolved records}."""
    elem = 4 if input_dtype == torch.float32 else 1
    n_in = elem
    for d in input_shape:
        n_in *= d
    body = [struct.pack("<ii4qq2q", DTYPES[input_dtype], residual_bits, *input_shape, n_in, *output_shape),
            struct.pack("<Q", len(constants)), constants, struct.pack("<Q", arena_bytes), struct.pack("<I", len(sequences))]
    for kind, records in sorted(sequences.items()):
        body.append(struct.pack("<II", kind, len(records)))
        for fn, args in records:
            body.append(struct.pack("<HH", _lib.ENGINE_ENTRIES.index(fn), len(args)))
            body += [_encode_arg(a) for a in args]
    body = b"".join(body)
    return _HEADER.pack(b"HAWQPLAN", _lib.ENGINE_FORMAT, 1, 9, 0, len(body), zlib.crc32(body), 0) + body


# ------------------------------------------------------------------------------------------------ saving a CompiledModel
def _cache_tensors(obj, found):
    """CUDA tensors held by a plan cache (nested dicts, lists and tuples), by storage base."""
    if torch.is_tensor(obj):
        if obj.is_cuda:
            found[obj.untyped_storage().data_ptr()] = obj
    elif isinstance(obj, dict):
        for v in obj.values():
            _cache_tensors(v, found)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _cache_tensors(v, found)
    return found


def _storage_bytes(t):
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage()).cpu().numpy().tobytes()


def save(eng, path):
    """CompiledModel.save: see the module docstring.  Builds the fallback graphs the engine has not built yet."""
    from .engine import _BUILD_LOCK
    from . import ops
    if eng.resize is not None:
        raise NotImplementedError("save: an engine with resize= grows its pixel arena and recaptures; plan files do not cover it")
    if eng.gather:
        raise NotImplementedError("save: an engine with gather=True all-gathers over NCCL inside its graph; plan files do not cover it")
    keys = {SEQ_FAST: eng.residual_bits, SEQ_SAFE: "safe"}
    if eng.residual_bits == 16:
        keys[SEQ_INT32] = 32
    with torch.no_grad():
        for key in keys.values():
            if key not in eng.launches:
                eng._build(32, key=key)
    dev, idx = eng.device, eng.device.index
    records, outs, consts = {}, {}, {}
    with _BUILD_LOCK, ops.using_handle(idx, eng._handle), torch.no_grad():
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for kind, key in sorted(keys.items()):
                with ops.recording() as rec:
                    out = eng._forward(eng.bits_of[key], key != "safe")
                if len(rec) != eng.launches[key]:
                    raise RuntimeError("save: %d launches recorded for sequence %r, the engine's graph has %d" % (len(rec), key, eng.launches[key]))
                st = out.untyped_storage()
                if out.dtype != torch.float32 or out.dim() < 2 or out.storage_offset() != 0 or st.nbytes() != out.numel() * 4:
                    raise RuntimeError("save: the logits of sequence %r do not fill their own fp32 storage" % (key,))
                records[kind], outs[kind] = rec, (st.data_ptr(), st.nbytes(), tuple(out.shape[:2]))
                for plans in eng._plans + [[m.__dict__["_hawq_cache"] for m in eng.model.modules() if "_hawq_cache" in m.__dict__]]:
                    _cache_tensors(plans, consts)
                del out
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
    if len({o[2] for o in outs.values()}) != 1:
        raise RuntimeError("save: the sequences' logits differ in shape")
    inp_t = eng.static_in
    ist = inp_t.untyped_storage()
    inp = (ist.data_ptr(), ist.nbytes())
    # the constants each sequence uses, each storage once, at 512-byte-aligned offsets
    used = []
    for rec in records.values():
        for _, args in rec:
            for a in args:
                if a[0] == "ptr" and a[2] in consts and a[2] not in used:
                    used.append(a[2])
    const_off, blob = {}, bytearray()
    for base in used:
        blob += bytes(_align(len(blob)) - len(blob))
        const_off[base] = len(blob)
        blob += _storage_bytes(consts[base])
    sequences, arena = {}, 0
    for kind, rec in records.items():
        sequences[kind], a = resolve(rec, inp, outs[kind][:2], const_off)
        arena = max(arena, a)
    data = plan_bytes(inp_t.dtype, tuple(inp_t.shape), outs[SEQ_FAST][2], eng.residual_bits, bytes(blob), arena, sequences)
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


# ------------------------------------------------------------------------------------------------ loading
def check(data):
    """hawq_engine_check of a plan file's bytes: its hawq_engine_info (raises HawqError on a malformed file)."""
    info = _lib.hawq_engine_info()
    _lib.check(_lib.load().hawq_engine_check(data, len(data), C.byref(info)))
    return info


class _Owner:
    """Owns one hawq_engine; the tensors over its bindings keep it alive."""

    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        if self.ptr:
            _lib.load().hawq_engine_destroy(self.ptr)
            self.ptr = None


class _DeviceArray:
    def __init__(self, ptr, shape, typestr, owner):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2, "strides": None}
        self.owner = owner


_TYPESTR = {0: "|i1", 1: "|u1", 2: "<f4"}


class LoadedEngine:
    """A plan file loaded by the library's runtime.  ``static_in`` / ``out`` are tensors over the engine's input and output
    bindings; ``__call__`` is the exact forward (CompiledModel.__call__), ``run_async`` one fast replay without a check."""

    def __init__(self, path, device=0):
        with open(path, "rb") as f:
            data = f.read()
        lib = _lib.load()
        ptr = C.c_void_p()
        _lib.check(lib.hawq_engine_load(int(device), data, len(data), C.byref(ptr)))
        self._owner = _Owner(ptr)
        self.device = torch.device("cuda", int(device))
        info = self.info()
        self.static_in = torch.as_tensor(_DeviceArray(lib.hawq_engine_input(ptr), info.input_shape[:], _TYPESTR[info.input_dtype], self._owner),
                                         device=self.device)
        self.out = torch.as_tensor(_DeviceArray(lib.hawq_engine_output(ptr), info.output_shape[:], "<f4", self._owner), device=self.device)
        self.residual_bits = info.residual_bits
        self.launches = {"fast": info.launches[SEQ_FAST], "int32": info.launches[SEQ_INT32], "safe": info.launches[SEQ_SAFE]}

    def info(self):
        info = _lib.hawq_engine_info()
        _lib.check(_lib.load().hawq_engine_get_info(self._owner.ptr, C.byref(info)))
        return info

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def run_async(self, x=None):
        """Enqueue one fast replay on the current stream (no host sync, no overflow check); returns the output tensor."""
        with torch.cuda.device(self.device):
            if x is not None:
                self.static_in.copy_(x, non_blocking=True)
            _lib.check(_lib.load().hawq_engine_enqueue(self._owner.ptr, self._stream()))
        return self.out

    def status(self):
        """The status word of the last replay (read it after synchronising the stream run_async used)."""
        v = C.c_int32()
        _lib.check(_lib.load().hawq_engine_status(self._owner.ptr, C.byref(v)))
        return int(v.value)

    def __call__(self, x=None):
        """Exact forward (hawq_engine_run): the fast replay, then the int32 or safe one when its status word asks for it."""
        with torch.cuda.device(self.device):
            if x is not None:
                self.static_in.copy_(x, non_blocking=True)
            flags = C.c_int32()
            rc = _lib.load().hawq_engine_run(self._owner.ptr, self._stream(), C.byref(flags))
        if rc == _lib.ERR_RESULT_INVALID:
            raise RuntimeError("hawq_b200: HAWQ_FLAG_BAD_RATIO raised (a dyadic ratio > 1 reached the fast kernel): results invalid")
        _lib.check(rc)
        return self.out

    @property
    def fallbacks(self):
        return int(self.info().fallbacks)

    @property
    def gpu_launches(self):
        return self.launches["fast"]


def load_engine(path, device=0):
    """Load a plan file written by CompiledModel.save onto cuda:`device` (see LoadedEngine)."""
    return LoadedEngine(path, device)
