"""Plan files without a GPU: the Python writer against the library's device-free checker (hawq_engine_check), every kind of malformed
file rejected with HAWQ_ERR_BAD_ARG, the runtime's entry table against the ctypes bindings and the launches of ops.py, the pointer
resolution and arena layout of CompiledModel.save on synthetic storages, and the dependencies of the standalone runner.  No plan is
ever loaded onto a device here."""
import ast
import ctypes
import os
import re
import struct
import subprocess
import zlib

import pytest
import torch

from hawq_b200 import _lib, engine_file as ef
from hawq_b200.build import RUNNER, build_library, build_runner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# synthetic storages (base, bytes): input int8 [2, 8, 8, 64], output fp32 [2, 10], one constant table, scratch
INP = (0x7f0000000000, 2 * 8 * 8 * 64)
OUT = (0x7f0000100000, 2 * 10 * 4)
CHAN = (0x7f0000200000, 64 * 16)
A = (0x7f0000300000, 2 * 8 * 8 * 64 * 4)        # int32 activations
B = (0x7f0000300000 + 4096, 2 * 8 * 8 * 64)     # allocated inside A's bytes once A was freed (the allocator's reuse)
POOL = (0x7f0000400000, 2 * 64)


@pytest.fixture(scope="module")
def lib():
    build_library()
    return _lib.load()


def ptr(storage, off=0):
    return ("ptr", storage[0] + off, storage[0], storage[1])


def rec(fn, *vals):
    """A recorded launch of `fn` (ops.recording's form): each value typed by the entry's signature"""
    kinds = {"i": "i32", "u": "u32", "I": "i64", "f": "f32"}
    args = []
    for code, v in zip(ef.arg_codes(fn), vals):
        if code == "p":
            args.append(("null",) if v is None else v)
        elif code in kinds:
            args.append((kinds[code], v))
        else:
            args.append(("blob", v))
    assert len(args) == len(ef.arg_codes(fn))
    return fn, args


def recording():
    """requant of the input into A, requant of A into B (aliasing A's old bytes), the pooled tail into POOL"""
    return [rec("hawq_requant", 128, 64, 32, ptr(INP), ptr(CHAN), 0, 0, 32, -2 ** 31, 2 ** 31 - 1, ptr(A)),
            rec("hawq_requant", 128, 64, 32, ptr(A), ptr(CHAN), 1, 1, 8, -128, 127, ptr(B)),
            rec("hawq_avgpool_requant", 2, 64, 1, 32, ptr(B), 2 ** 30, 31, -128, 127, ptr(POOL))]


def plan(sequences=None, const=b"\x01" * CHAN[1], residual_bits=16):
    if sequences is None:
        recs, arena = ef.resolve(recording(), INP, OUT, {CHAN[0]: 0})
        sequences = {ef.SEQ_FAST: recs, ef.SEQ_INT32: recs[:2], ef.SEQ_SAFE: recs[:1]}
    else:
        arena = 1 << 20
    return ef.plan_bytes(torch.int8, (2, 8, 8, 64), (2, 10), residual_bits, const, arena, sequences)


def reseal(data):
    """data with its header's body length and checksum recomputed (a structurally altered file that still passes the checksum)"""
    body = data[40:]
    return data[:24] + struct.pack("<QII", len(body), zlib.crc32(body), 0) + body


def rejected(data):
    with pytest.raises(_lib.HawqError) as e:
        ef.check(data)
    assert e.value.code == _lib.ERR_BAD_ARG
    return str(e.value)


def test_hand_built_plan_is_accepted_with_its_sizes(lib):
    info = ef.check(plan())
    assert (info.input_dtype, info.residual_bits) == (0, 16)
    assert list(info.input_shape) == [2, 8, 8, 64] and info.input_bytes == INP[1]
    assert list(info.output_shape) == [2, 10]
    assert info.constant_bytes == CHAN[1]
    assert info.arena_bytes == ef._align(A[1]) + POOL[1]       # A and B share one segment; POOL starts at the next 512-byte offset
    assert list(info.launches) == [3, 2, 1] and info.fallbacks == 0


def test_every_truncation_is_rejected(lib):
    data = plan()
    for n in range(len(data)):
        rejected(data[:n])


@pytest.mark.parametrize("offset,what", [(0, "magic"), (8, "format"), (12, "ABI"), (16, "compute capability"), (32, "checksum"),
                                         (200, "checksum")])
def test_flipped_header_field_or_body_byte_is_rejected(lib, offset, what):
    data = bytearray(plan())
    data[offset] ^= 0x01
    msg = rejected(bytes(data))
    assert what.split()[0].lower() in msg.lower() or what == "compute capability" and "compute" in msg


def test_unknown_entry_id_is_rejected(lib, monkeypatch):
    monkeypatch.setattr(_lib, "ENGINE_ENTRIES", _lib.ENGINE_ENTRIES + ("hawq_unknown",))
    fn, args = rec("hawq_pack_i4", 64, ptr(INP), ptr(OUT))
    recs, _ = ef.resolve([("hawq_unknown", args)], INP, OUT, {})
    assert "unknown entry id 17" in rejected(plan({ef.SEQ_FAST: recs, ef.SEQ_SAFE: recs}, residual_bits=32))


def test_wrong_argument_kind_or_count_is_rejected(lib):
    good, _ = ef.resolve(recording(), INP, OUT, {CHAN[0]: 0})
    fn, args = good[0]
    for bad in ([("i32", 128)] + args[1:], args[:-1], args + [("null",)], args[:3] + [("i32", 0)] + args[4:],
                args[:10] + [("blob", b"\0" * 8)]):
        rejected(plan({ef.SEQ_FAST: [(fn, bad)], ef.SEQ_SAFE: good}, residual_bits=32))
    # a descriptor of the wrong size
    conv = rec("hawq_conv2d", b"\0" * 40, bytes(68), ptr(INP), ptr(CHAN), ptr(CHAN), None, None, None, ptr(OUT), None)
    recs, _ = ef.resolve([conv], INP, OUT, {CHAN[0]: 0})
    assert "blob" in rejected(plan({ef.SEQ_FAST: recs, ef.SEQ_SAFE: recs}, residual_bits=32))


def test_pointer_past_its_region_is_rejected(lib):
    good, _ = ef.resolve(recording(), INP, OUT, {CHAN[0]: 0})
    fn, args = good[0]
    for region, off in [("const", CHAN[1]), ("input", INP[1]), ("output", OUT[1] + 4096), ("arena", 1 << 20)]:
        bad = args[:3] + [("ptr", region, off)] + args[4:]
        assert "outside its region" in rejected(plan({ef.SEQ_FAST: [(fn, bad)], ef.SEQ_SAFE: good}, residual_bits=32))


def test_region_larger_than_the_file_is_rejected(lib):
    data = bytearray(plan())
    at = 40 + struct.calcsize("<ii4qq2q")                        # the constants' byte count
    assert struct.unpack_from("<Q", data, at)[0] == CHAN[1]
    struct.pack_into("<Q", data, at, len(data))
    assert "past the file" in rejected(reseal(bytes(data)))
    struct.pack_into("<Q", data, at, 2 ** 63)
    rejected(reseal(bytes(data)))


def test_sequences_must_match_the_stream_width(lib):
    recs, _ = ef.resolve(recording(), INP, OUT, {CHAN[0]: 0})
    rejected(plan({ef.SEQ_FAST: recs, ef.SEQ_SAFE: recs}, residual_bits=16))                    # 16-bit without int32
    rejected(plan({ef.SEQ_FAST: recs, ef.SEQ_INT32: recs, ef.SEQ_SAFE: recs}, residual_bits=32))
    rejected(plan({ef.SEQ_FAST: recs, ef.SEQ_INT32: recs}, residual_bits=16))                   # no safe sequence
    ef.check(plan({ef.SEQ_FAST: recs, ef.SEQ_SAFE: recs}, residual_bits=32))


def _launched_by_ops():
    tree = ast.parse(open(os.path.join(ROOT, "hawq_b200", "ops.py")).read())
    return {node.args[1].value for node in ast.walk(tree) if isinstance(node, ast.Call) and getattr(node.func, "id", None) == "_launch"}


def test_entry_table_bindings_and_ops_agree(lib):
    """The header's entry ids are _lib.ENGINE_ENTRIES in order, that is every entry point ops.py launches, and the runtime accepts a
    record of each with the argument kinds of its ctypes signature."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hawq_b200.h")).read(), flags=re.S)
    body = re.search(r"enum hawq_engine_entry\s*{(.*?)}", header, re.S).group(1)
    ids = {"hawq_" + name.lower(): int(v) for name, v in re.findall(r"HAWQ_ENTRY_(\w+)\s*=\s*(\d+)", body)}
    assert ids.pop("hawq_count") == len(_lib.ENGINE_ENTRIES)
    assert ids == {name: i for i, name in enumerate(_lib.ENGINE_ENTRIES)}
    assert set(_lib.ENGINE_ENTRIES) == _launched_by_ops()
    assert set(_lib.ENGINE_ENTRIES) <= set(_lib.SIGNATURES)
    blobs = {"D": bytes(ctypes.sizeof(_lib.hawq_conv_desc)), "E": bytes(ctypes.sizeof(_lib.hawq_epilogue_desc)), "F": bytes(12)}
    for fn in _lib.ENGINE_ENTRIES:
        vals = [ptr(INP) if c == "p" else blobs[c] if c in blobs else 0 for c in ef.arg_codes(fn)]
        recs, _ = ef.resolve([rec(fn, *vals)], INP, OUT, {})
        ef.check(plan({ef.SEQ_FAST: recs, ef.SEQ_SAFE: recs}, residual_bits=32))


def test_overlapping_scratch_shares_arena_bytes():
    place, size = ef.arena_layout({1000: 600, 1200: 100, 1500: 300, 5000: 50, 5040: 100, 9000: 8})
    assert place[1000] == 0 and place[1200] - place[1000] == 200 and place[1500] - place[1000] == 500   # one segment [1000, 1800)
    assert place[5000] == 1024 and place[5040] - place[5000] == 40                                      # [5000, 5140)
    assert place[9000] == 1536 and size == 1536 + 8
    assert all(place[b] % 512 == 0 for b in (1000, 5000, 9000))


def test_resolve_places_every_region():
    recs, arena = ef.resolve(recording(), INP, OUT, {CHAN[0]: 512})
    assert recs[0][1][3] == ("ptr", "input", 0) and recs[0][1][4] == ("ptr", "const", 512)
    assert recs[0][1][10] == ("ptr", "arena", 0) and recs[1][1][10] == ("ptr", "arena", 4096)     # B keeps its place inside A
    assert recs[2][1][9] == ("ptr", "arena", ef._align(A[1])) and arena == ef._align(A[1]) + POOL[1]
    assert recs[0][0] == "hawq_requant" and recs[0][1][0] == ("i64", 128)


def test_unresolvable_pointer_names_entry_and_argument():
    bad = rec("hawq_requant", 128, 64, 32, ("ptr", 0x1234, None, None), ptr(CHAN), 0, 0, 32, 0, 1, ptr(A))
    with pytest.raises(ef.UnresolvedPointer, match=r"hawq_requant argument 4"):
        ef.resolve([bad], INP, OUT, {CHAN[0]: 0})
    outside = rec("hawq_requant", 128, 64, 32, ptr(INP), ptr(CHAN), 0, 0, 32, 0, 1, ("ptr", A[0] + A[1], A[0], A[1]))
    with pytest.raises(ef.UnresolvedPointer, match=r"hawq_requant argument 11"):
        ef.resolve([outside], INP, OUT, {CHAN[0]: 0})


def test_runner_needs_neither_python_nor_torch(lib):
    build_runner()
    r = subprocess.run(["readelf", "-d", RUNNER], capture_output=True, text=True, check=True)
    needed = re.findall(r"\(NEEDED\)\s+Shared library: \[([^\]]+)\]", r.stdout)
    assert "libhawq_b200.so" in needed
    assert not [n for n in needed if re.match(r"lib(python|torch|c10)", n)], needed
