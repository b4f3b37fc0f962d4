"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import hashlib
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# (arch, scheme) of every ResNet network golden (net_<arch>_<scheme>.npz, written by tests/golden/make_golden.py)
RESNET_GOLDENS = sorted(tuple(f[len("net_"):-len(".npz")].split("_", 1)) for f in os.listdir(GOLDEN)
                        if f.startswith("net_resnet") and f.endswith(".npz"))


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


def load_net_golden(arch, scheme):
    g = load_golden("net_%s_%s.npz" % (arch, scheme))
    meta = json.loads(str(g["meta"]))
    return g["logits"], meta


def sha_i32(a):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a).astype(np.int32)).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------ guarded kernel calls
# Every tensor argument of a guarded call lives in its own allocation [head guard | payload | tail guard].  The guards hold
# POISON, a byte that changes a result wherever a kernel reads it: nonzero as int8 and in both nibbles, positive as int16 (0x5B5B;
# the max-pool input is >= 0) and large as float32 (about 6e16).  A guard spans at least one 128-row tile of the call's widest
# row, so a kernel that overruns by a whole ragged tile stays inside the allocation and is reported instead of faulting.
POISON = 0x5B
MIN_GUARD_BYTES = 64 << 10
PAYLOAD_ALIGN = 256          # every payload keeps the 16-byte alignment the kernels' vector accesses need


def raw_bytes(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


class Guarded:
    """A copy of tensor `src` on `device` inside one allocation [head guard | payload | tail guard].  `payload` has src's dtype
    and shape; `expect` is the whole allocation as it must be after the call: poison in both guards, src's bytes in the payload
    unless expect_output() names other ones."""

    def __init__(self, name, src, device, guard_bytes):
        self.name = name
        self.nbytes = src.numel() * src.element_size()
        self.head = -(-max(guard_bytes, MIN_GUARD_BYTES) // PAYLOAD_ALIGN) * PAYLOAD_ALIGN
        self.buf = torch.full((2 * self.head + self.nbytes,), POISON, dtype=torch.uint8, device=device)
        self.payload = self.buf[self.head:self.head + self.nbytes].view(src.dtype).view(src.shape)
        self.payload.copy_(src)
        self.expect = self.buf.clone()

    def expect_output(self, want):
        """After the call the payload must hold want's bytes.  Until then it holds their bitwise complement, so that every byte
        the call leaves unwritten differs, whatever the data."""
        w = raw_bytes(want).to(self.buf.device)
        assert w.numel() == self.nbytes, (self.name, w.numel(), self.nbytes)
        self.expect[self.head:self.head + self.nbytes] = w
        self.buf[self.head:self.head + self.nbytes] = torch.bitwise_not(w)

    def problems(self):
        """One line per region (head, payload, tail) whose bytes differ from `expect`: the count and the first offset, in bytes
        from the start of the payload (negative in the head guard)."""
        bad = self.buf != self.expect
        if not bool(bad.any()):
            return []
        out = []
        for region, lo, hi in (("head", 0, self.head), ("payload", self.head, self.head + self.nbytes),
                               ("tail", self.head + self.nbytes, self.buf.numel())):
            idx = torch.nonzero(bad[lo:hi]).reshape(-1)
            if idx.numel():
                out.append("%s %s: %d bad bytes, first at payload offset %d"
                           % (self.name, region, idx.numel(), lo + int(idx[0]) - self.head))
        return out


def guarded_call(launch, args, expected, device, guard_bytes=0):
    """Calls launch(**args) with every tensor argument copied into its own Guarded allocation on `device`.  expected maps the
    output names to the tensors the call must produce; every other tensor is an input, or a pointer the call must ignore, and
    must keep its bytes.  Returns ({output name: payload}, problems): problems lists every guard byte that changed, every output
    byte that differs from expected (raw bytes: NaN semantics do not matter) and every input byte that changed."""
    arenas = {k: Guarded(k, v, device, guard_bytes) for k, v in args.items() if torch.is_tensor(v)}
    for k, want in expected.items():
        arenas[k].expect_output(want)
    launch(**{k: arenas[k].payload if k in arenas else v for k, v in args.items()})
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)
    return {k: arenas[k].payload for k in expected}, [p for a in arenas.values() for p in a.problems()]


def golden_act_ranges(meta):
    return {k: (v["x_min"], v["x_max"]) for k, v in meta["acts"].items()}


def build_fakequant(arch, scheme, meta=None):
    """Oracle fake-quant net on the seed-0 synthetic model, act ranges from the golden file (like loading a checkpoint)."""
    from oracle import fakequant as fq
    from hawq_b200.synthetic import synthetic_float_resnet, synthetic_batch
    from hawq_b200.bit_config import get_bit_config
    net = synthetic_float_resnet(arch, 0)
    m = fq.FakeQuantResNet(arch, net, get_bit_config(arch, scheme))
    if meta is not None:
        m.load_act_ranges(golden_act_ranges(meta))
        m.freeze()
    return m
