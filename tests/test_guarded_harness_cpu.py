"""The guarded-call harness of the kernel parity tests (tests/util.guarded_call), driven on the CPU with fake kernels: a correct
kernel passes, and each way a kernel can put bytes in the wrong place, or read them from there, is reported by argument and
region."""
import numpy as np
import pytest
import torch

from tests.util import MIN_GUARD_BYTES, PAYLOAD_ALIGN, POISON, guarded_call

N = 1000   # int32 elements: 4000 payload bytes, not a multiple of the payload alignment


def whole_allocation(t):
    """the uint8 allocation behind a payload view and the payload's byte offset in it: what a kernel's pointer arithmetic reaches"""
    return torch.empty(0, dtype=torch.uint8).set_(t.untyped_storage()), t.storage_offset() * t.element_size()


def model(x):
    return x * 3 + 1


def correct(x, out, unused):
    out.copy_(model(x))


def skips_one_byte(x, out, unused):
    want = model(x).view(torch.uint8)
    o = out.view(torch.uint8)
    o[:17] = want[:17]
    o[18:] = want[18:]


def writes_past_the_end(x, out, unused):
    correct(x, out, unused)
    buf, off = whole_allocation(out)
    buf[off + out.numel() * 4] = 0


def writes_before_the_start(x, out, unused):
    correct(x, out, unused)
    buf, off = whole_allocation(out)
    buf[off - 1] = 0


def modifies_its_input(x, out, unused):
    correct(x, out, unused)
    x[5] += 1


def writes_an_unused_buffer(x, out, unused):
    correct(x, out, unused)
    unused[0] = 0


def reads_past_the_input(x, out, unused):
    """a broken read predicate: the element one past the end of x joins the last output (zero padding would hide it)"""
    buf, off = whole_allocation(x)
    past = buf[off + x.numel() * 4:off + x.numel() * 4 + 4].view(torch.int32)
    correct(x, out, unused)
    out[-1] += past[0]


def call(kernel, x=None):
    x = torch.arange(-N // 2, N // 2, dtype=torch.int32) if x is None else x
    args = dict(x=x, out=torch.zeros(N, dtype=torch.int32), unused=torch.full((64,), POISON, dtype=torch.uint8))
    return guarded_call(kernel, args, dict(out=model(x)), "cpu", guard_bytes=1000)


def test_a_correct_kernel_passes():
    outs, problems = call(correct)
    assert problems == []
    assert torch.equal(outs["out"], model(torch.arange(-N // 2, N // 2, dtype=torch.int32)))


def test_an_output_of_zeros_must_still_be_written():
    """every expected byte is 0 here; a kernel that writes nothing is still caught"""
    x = torch.full((N,), -1, dtype=torch.int32)
    args = dict(x=x, out=torch.zeros(N, dtype=torch.int32), unused=torch.zeros(8, dtype=torch.uint8))
    _, problems = guarded_call(lambda x, out, unused: None, args, dict(out=torch.zeros(N, dtype=torch.int32)), "cpu")
    assert problems == ["out payload: %d bad bytes, first at payload offset 0" % (4 * N)]


@pytest.mark.parametrize("kernel, problem", [
    (skips_one_byte, "out payload: 1 bad bytes, first at payload offset 17"),
    (writes_past_the_end, "out tail: 1 bad bytes, first at payload offset %d" % (4 * N)),
    (writes_before_the_start, "out head: 1 bad bytes, first at payload offset -1"),
    (modifies_its_input, "x payload: 1 bad bytes, first at payload offset 20"),
    (writes_an_unused_buffer, "unused payload: 1 bad bytes, first at payload offset 0"),
    (reads_past_the_input, "out payload: 4 bad bytes, first at payload offset %d" % (4 * N - 4)),
])
def test_each_misplaced_byte_is_reported(kernel, problem):
    _, problems = call(kernel)
    assert problems == [problem]


def test_layout_and_poison():
    seen = {}

    def record(x, out, unused):
        for k, t in (("x", x), ("out", out), ("unused", unused)):
            seen[k] = whole_allocation(t)
        correct(x, out, unused)

    call(record)
    for name, (buf, off) in seen.items():
        assert off % PAYLOAD_ALIGN == 0 and off >= MIN_GUARD_BYTES, name
        assert buf.numel() - off - {"x": 4 * N, "out": 4 * N, "unused": 64}[name] >= MIN_GUARD_BYTES, name
    b = np.full(4, POISON, dtype=np.uint8)
    assert b.view(np.int8)[0] != 0 and POISON & 0xF and POISON >> 4           # int8 and both nibbles
    assert b[:2].view(np.int16)[0] > 0                                         # int16 (the max-pool input is >= 0)
    assert b.view(np.float32)[0] > 1e16                                        # float32
