"""The network and engine harness of the tests: frozen models built from the goldens, the oracles they are checked against, the
int8 network input, recorded forwards, the size goldens, the MobileNetV2 (and ResNet-18) scenarios that calibrated models never
produce, and the network-level checks that several test modules run.  Importing it touches neither the GPU nor the library."""
import json
import os

import numpy as np
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200.synthetic import synthetic_batch, synthetic_float_mobilenetv2, synthetic_float_resnet
from oracle import fakequant as fq
from oracle import int_ref as ir
from tests import abi_model as am
from tests.kernel_harness import DEV
from tests.util import GOLDEN, build_fakequant, golden_act_ranges, load_golden, load_net_golden, sha_i32

SCHEMES = ["uniform8", "uniform4", "modelsize_0.5", "bops_0.5"]
# resize units whose identity input is 4-bit and whose last convolution's input is 8-bit: with packed nibbles the two 1x1 inputs
# have different widths, so the dual kernel is declined there (identity RAW_I32 conv + RESIDUAL conv instead)
MIXED_WIDTH_RESIZE = {("resnet50", "modelsize_0.25"): 1, ("resnet50", "latency_0.25"): 1}


def golden_model(arch, scheme, meta, shrink=None):
    """Frozen model on the golden ranges; ``shrink`` = (QuantAct name, factor) scales that activation's range."""
    q = hb.build_synthetic_qresnet(arch, scheme, act_ranges=golden_act_ranges(meta))
    if shrink is not None:
        act = dict(q.named_modules())[shrink[0]]
        act.x_min.mul_(shrink[1])
        act.x_max.mul_(shrink[1])
    return q


def _oracle(arch, scheme, meta, shrink=None):
    fqm = build_fakequant(arch, scheme, meta)
    if shrink is not None:
        a = fqm.acts[shrink[0]]
        a.x_min, a.x_max = a.x_min * shrink[1], a.x_max * shrink[1]
    return fqm


def int8_input(x, scale):
    """float NCHW batch -> int8 NHWC network input (CPU), quantised like the reference's quant_input at `scale`"""
    return torch.from_numpy(ir.quantize_input(x.numpy(), np.float32(scale)).astype(np.int8))


def _eager(q, x, **mode):
    """One eager frozen forward of the int8 NHWC CUDA batch x under qtensor.engine_mode(**mode); returns (logits, status word)."""
    n, h, w, c = x.shape
    hb.ops.reset_status(0)
    with torch.no_grad(), qtensor.engine_mode(**mode):
        out = q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=x.view(-1), bits=8, signed=True), x.device))
    torch.cuda.synchronize()
    return out, hb.ops.get_status(0)


def nhwc(a):
    return a.transpose(0, 2, 3, 1) if a.ndim == 4 else a


def run_engine(q, x):
    """Frozen forward on the CPU ABI model; returns (logits, {QuantAct name: output IntActivation})."""
    rec = {}
    for name, m in q.named_modules():
        if isinstance(m, hb.QuantAct):
            m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name, out[0]))
    with torch.no_grad():
        y = q(x)
    return y, rec


def int_oracle(scheme, ranges, x, net=None):
    o = fq.FakeQuantMobileNetV2(net if net is not None else synthetic_float_mobilenetv2(0), hb.get_bit_config("mobilenetv2_w1", scheme))
    o.load_act_ranges(ranges)
    o.freeze()
    yf = o(x, trace=True)
    return o, yf, ir.IntMobileNetV2(o.harvest())


def assert_rows(got, want, what=None):
    """Logits `got` (array or tensor) equal the oracle's `want` row for row; the message names the first rows that differ."""
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert got.shape == want.shape and np.array_equal(got, want), \
        "%srows differing from the oracle: %s" % (what + ": " if what else "", np.nonzero((got != want).any(axis=1))[0][:16].tolist())


# ------------------------------------------------------------------------------------------------ size goldens
SIZE_GOLDENS = sorted(f for f in os.listdir(GOLDEN) if f.startswith("size_") and f.endswith(".npz"))


def load_size_golden(name):
    """(logits, meta, float input) of one size golden"""
    g = load_golden(name)
    meta = json.loads(str(g["meta"]))
    return g["logits"], meta, synthetic_batch(*meta["input"])


def oracle_for(meta, x):
    """(FakeQuant oracle after a traced forward on x, its logits, integer restatement) for the golden's network"""
    arch, scheme = meta["arch"], meta["scheme"]
    if arch == "mobilenetv2_w1":
        o, yf, net = int_oracle(scheme, golden_act_ranges(meta), x)
        return o, yf.numpy(), net
    o = build_fakequant(arch, scheme, meta)
    yf = o(x, trace=True)
    return o, yf.numpy(), ir.IntResNet(o.harvest())


def assert_mobilenet_logits(y, want, logits_g):
    """the integer restatement exactly; the reference's fp32 classifier sums (tests/test_mobilenetv2_cpu.py) closely, same classes"""
    assert np.array_equal(y, want)
    assert np.allclose(y, logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(y.argmax(1), logits_g.argmax(1))


def engine_outputs(q, x):
    """Frozen forward; returns (logits, {QuantAct name: output}, {residual unit name + '.quant_act_int32': unit output}).  A residual
    QuantAct's output is pending until the unit's ReLU; the unit output is that QuantAct's integers after the ReLU."""
    acts, units = {}, {}
    hooks = []
    for name, m in q.named_modules():
        d = units if isinstance(m, hb.q_resnet.QResidualUnit) else acts if isinstance(m, hb.QuantAct) else None
        if d is not None:
            key = name + ".quant_act_int32" if d is units else name
            hooks.append(m.register_forward_hook(lambda mod, inp, out, key=key, d=d: d.__setitem__(key, out[0])))
    with torch.no_grad():
        y = q(x)
    for h in hooks:
        h.remove()
    return y, acts, units


def check_engine_against_golden(y, acts, units, meta, logits_g, net, x):
    """Every concrete QuantAct output hashes to the golden's sha and keeps its padded channels 0; every residual-unit output equals
    the integer restatement's stream after the ReLU (the restatement's own integers are pinned to the golden in
    test_oracle_reproduces_the_golden); ResNet logits bit-equal to the golden, MobileNetV2 logits as assert_mobilenet_logits."""
    y = y.cpu().numpy()
    assert y.shape == logits_g.shape
    assert set(acts) == set(meta["acts"])
    mobilenet = meta["arch"] == "mobilenetv2_w1"
    concrete = {k: t for k, t in acts.items() if mobilenet or t.node.kind == "int"}
    assert len(concrete) + len(units) >= len(meta["acts"]) - 2, (len(concrete), len(units), len(meta["acts"]))
    for name, t in concrete.items():
        got = nhwc(t.int_tensor().cpu().numpy())
        assert list(got.shape) == meta["acts"][name]["shape"], name
        assert sha_i32(got) == meta["acts"][name]["sha"], name
    assert_padded_channels_zero(concrete)
    if mobilenet:
        assert not units
        assert_mobilenet_logits(y, net(x.numpy()), logits_g)
        return
    net(x.numpy(), trace=True)
    for name, t in units.items():
        got, want = nhwc(t.int_tensor().cpu().numpy()), np.maximum(net.trace[name], 0)
        assert np.array_equal(got.reshape(want.shape), want), (name, int((got.reshape(want.shape) != want).sum()))
    assert np.array_equal(y, logits_g)


# ------------------------------------------------------------------------------------------------ MobileNetV2 and ResNet-18 scenarios
# dead channels: two of a stride-1 depthwise conv2, one of a stride-2 depthwise conv2, one of an expansion conv1, one of a residual
# projection conv3.  Channel 3 of stage2.unit2.conv2 has a positive folded bias under seed 0; the channels in POSITIVE get one.
DEAD = {"features.stage2.unit2.conv2": (3, 10), "features.stage3.unit1.conv2": (5,), "features.stage3.unit2.conv1": (7,),
        "features.stage3.unit2.conv3": (2,)}
POSITIVE = {("features.stage3.unit2.conv1", 7), ("features.stage3.unit2.conv3", 2)}
DEAD_RESNET18 = {"features.stage1.unit1.body.conv1": (5,), "features.stage2.unit2.body.conv2": (9,)}
POSITIVE_RESNET18 = {("features.stage1.unit1.body.conv1", 5), ("features.stage2.unit2.body.conv2", 9)}

# ReLU6 sites whose cap is made to bind: (QuantAct, its convolution in the float model, the QuantAct feeding that convolution)
CAP_SITES = [("quant_act_int32", "features.init_block", "quant_input"),
             ("features.stage2.unit1.quant_act1", "features.stage2.unit1.conv1", "features.stage2.unit1.quant_act"),
             ("features.stage2.unit2.quant_act2", "features.stage2.unit2.conv2", "features.stage2.unit2.quant_act1"),
             ("features.stage3.unit1.quant_act2", "features.stage3.unit1.conv2", "features.stage3.unit1.quant_act1"),
             ("quant_act_int32_final", "features.final_block", "quant_act_before_final_block")]
# (scheme, a4_container) of the dead-channel and cap scenarios
TABLES = [("uniform8", 8), ("uniform4", 8), ("uniform4", 4)]


def submodule(net, name):
    for part in name.split("."):
        net = getattr(net, part)
    return net


def dead_float_net(arch="mobilenetv2_w1"):
    """The seed-0 float model with the DEAD channels' weights zeroed (the POSITIVE ones get folded bias 4 > 0)."""
    net = synthetic_float_mobilenetv2(0) if arch == "mobilenetv2_w1" else synthetic_float_resnet(arch, 0)
    dead, positive = (DEAD, POSITIVE) if arch == "mobilenetv2_w1" else (DEAD_RESNET18, POSITIVE_RESNET18)
    with torch.no_grad():
        for name, chans in dead.items():
            cb = submodule(net, name)
            for c in chans:
                cb.conv.weight[c] = 0
                if (name, c) in positive:
                    cb.bn.running_mean[c] = 0
                    cb.bn.bias[c] = 4.0
    return net


def capped_float_net():
    """The seed-0 float model with the BN weight of every CAP_SITES convolution scaled by 16 (used with x_max = 8 there)."""
    net = synthetic_float_mobilenetv2(0)
    with torch.no_grad():
        for _, conv, _ in CAP_SITES:
            submodule(net, conv).bn.weight.mul_(16.0)
    return net


def capped_ranges(ranges):
    ranges = dict(ranges)
    for act, _, _ in CAP_SITES:
        ranges[act] = (ranges[act][0], 8.0)
    return ranges


def frozen(arch, scheme, net, ranges):
    """Quantized graph of float model `net` with the bit table stamped and activation ranges loaded (as from a checkpoint), frozen."""
    q = hb.quantize_arch_dict[arch](net)
    assert hb.stamp_bit_config(q, hb.get_bit_config(arch, scheme)) == len(hb.get_bit_config(arch, scheme))
    q.eval()
    for name, m in q.named_modules():
        if isinstance(m, hb.QuantAct):
            m.x_min.fill_(ranges[name][0])
            m.x_max.fill_(ranges[name][1])
    hb.freeze_model(q)
    return q


def assert_padded_channels_zero(rec):
    for name, t in rec.items():
        n = t.node
        if n.cs > n.shape[1]:
            v = am.decode(n.data.cpu(), n.bits, n.signed).reshape(-1, n.cs)
            assert not v[:, n.shape[1]:].any(), name


def assert_quantacts_equal(rec, trace):
    """Every recorded QuantAct output (NCHW integers) equals the oracle's trace; names the first differing channel."""
    assert set(rec) == set(trace)
    for name, t in rec.items():
        got, want = t.int_tensor().cpu().numpy(), trace[name].numpy()
        if not np.array_equal(got, want):
            d = np.argwhere(got != want)
            n, c = d[0][:2]
            raise AssertionError("%s: %d values differ, first at image %d channel %d: %d, reference %d"
                                 % (name, len(d), n, c, got[tuple(d[0])], want[tuple(d[0])]))


def mobilenet_case(scheme, net_fn, ranges_fn=None, batch=2):
    """(frozen model, float input, FakeQuantMobileNetV2 after a traced forward, IntMobileNetV2) of a modified seed-0 model."""
    _, meta = load_net_golden("mobilenetv2_w1", scheme)
    ranges = golden_act_ranges(meta)
    if ranges_fn is not None:
        ranges = ranges_fn(ranges)
    x = synthetic_batch(*meta["input"]) if batch == 2 else synthetic_batch(batch, 11)
    o, _, net = int_oracle(scheme, ranges, x, net_fn())
    return frozen("mobilenetv2_w1", scheme, net_fn(), ranges), x, o, net


def cap_binding(rec, net):
    """Per CAP_SITES QuantAct: the number of channels whose largest output sits on its ReLU6 cap strictly below the clamp's hi."""
    counts = {}
    for act, conv, prev in CAP_SITES:
        key = "init_block" if conv == "features.init_block" else conv
        w_sf, a_prev = net.convs[key]["w_sf"], net.acts[prev]["scale"]
        m, e = ir.dyadic_vec(ir.requant_ratio(a_prev, w_sf, net.acts[act]["scale"]))
        hi = ir.clamp_range(net.acts[act]["bits"], net.acts[act]["mode"])[1]
        cap = ir.requant(ir.relu6_cap(a_prev, w_sf), m, e)
        got = nhwc(rec[act].int_tensor().cpu().numpy()).reshape(-1, len(cap)).max(axis=0)
        counts[act] = int(((cap < hi) & (got == cap)).sum())
    return counts


def resnet18_dead_case():
    """(frozen ResNet-18 uniform4 with DEAD_RESNET18, golden input, FakeQuantResNet after a traced forward, its logits)."""
    _, meta = load_net_golden("resnet18", "uniform4")
    ranges = golden_act_ranges(meta)
    x = synthetic_batch(*meta["input"])
    fqm = fq.FakeQuantResNet("resnet18", dead_float_net("resnet18"), hb.get_bit_config("resnet18", "uniform4"))
    fqm.load_act_ranges(ranges)
    fqm.freeze()
    want = fqm(x, trace=True).numpy()
    for name, c in [("stage1.unit1.quant_convbn1", 5), ("stage2.unit2.quant_convbn2", 9)]:
        assert int(fqm.harvest()["convs"][name]["bias_integer"][c]) == 2 ** 31, name
    return frozen("resnet18", "uniform4", dead_float_net("resnet18"), ranges), x, fqm, want


def run_resnet(q, x):
    """Forward with every concrete QuantAct output and every unit output (the residual stream after its ReLU) recorded, NCHW."""
    acts, units = {}, {}
    for name, m in q.named_modules():
        d = units if isinstance(m, hb.q_resnet.QResidualUnit) else acts if isinstance(m, hb.QuantAct) else None
        if d is not None:
            m.register_forward_hook(lambda mod, inp, out, name=name, d=d: d.__setitem__(name, out[0]))
    with torch.no_grad():
        y = q(x)
    got = {name: t.int_tensor().cpu().numpy() for name, t in acts.items() if t.node.kind == "int"}   # a pending residual (before
    got.update({name + ".quant_act_int32": t.int_tensor().cpu().numpy() for name, t in units.items()})   # its ReLU): the unit output
    return y, got


def assert_resnet_equal(got, trace):
    checked = 0
    for name, want in trace.items():
        if name in got:
            want = want.numpy()
            if name.endswith("quant_act_int32") and name != "quant_act_int32":
                want = np.maximum(want, 0)
            assert np.array_equal(got[name], want), (name, int((got[name] != want).sum()))
            checked += 1
    assert checked >= len(trace) - 2, (checked, len(trace))


# ------------------------------------------------------------------------------------------------ network-level checks
def checked_eager(q, q_in):
    """One eager pass over int8 input in the mode the compiled graph runs (residual_bits 16, checked), every QuantAct output recorded."""
    rec = {}
    hooks = [m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name, out[0]))
             for name, m in q.named_modules() if isinstance(m, hb.QuantAct)]
    n, h, w, c = q_in.shape
    ops.reset_status(0)
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        y = q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device))
    torch.cuda.synchronize()
    for hk in hooks:
        hk.remove()
    assert ops.get_status(0) & 7 == 0
    return y, rec


def compiled_logits(q, q_in):
    eng = hb.compile_model(q, q_in)
    out = eng(q_in).cpu().numpy()
    assert eng.fallbacks == 0
    return out


CHUNK = 16          # images per oracle pass: a full IntMobileNetV2 trace is about 1 GB per 16 images


def check_every_row(q, net, batch, containers, monkeypatch, hw=224):
    """Compiled logits of synthetic_batch(batch, 11, hw) against IntMobileNetV2 on every row, and every QuantAct of every image of a
    checked eager pass, per 4-bit container; the oracle runs CHUNK images at a time."""
    x = synthetic_batch(batch, 11, hw)
    q_in = int8_input(x, net.acts["quant_input"]["scale"]).to(DEV)
    runs = []
    for a4 in containers:
        monkeypatch.setattr(qtensor.config, "a4_container", a4)
        logits = compiled_logits(q, q_in)
        _, rec = checked_eager(q, q_in)
        assert_padded_channels_zero(rec)
        got = {}
        for name, t in rec.items():
            v = t.int_tensor().to(torch.int32)
            got[name] = v.permute(0, 2, 3, 1) if v.dim() == 4 else v
        got.setdefault("quant_input", q_in)                 # an int8 input passes quant_input unchanged
        runs.append((a4, logits, got))
        del rec
    for i in range(0, batch, CHUNK):
        want = net(x[i:i + CHUNK].numpy(), trace=True)
        for a4, logits, got in runs:
            assert_rows(logits[i:i + CHUNK], want)
            assert set(got) == set(net.trace), (a4, set(got) ^ set(net.trace))
            for name, w in net.trace.items():
                g = got[name][i:i + CHUNK].cpu().numpy()
                assert np.array_equal(g.reshape(w.shape), w), (a4, name, i, int((g.reshape(w.shape) != w).sum()))


def check_benchmarked_configuration_matches_oracle_on_every_row(arch, scheme, batch, a4_container, monkeypatch, hw=224):
    """The configuration bench.py times (CUDA graph, fused kernels, uint16 stream) at the benchmarked batch size against the
    oracle (the reference's fake-quant forward restated on the CPU, oracle/fakequant.py): ALL rows of the logits bit-equal, and the
    integers of the residual stream at the end of stage 1 and of the last stage (eager pass with the same kernels) equal too.
    Many row tiles per channel block and full-size pipelines are only reached at this size.  hw: the input size (synthetic_batch)."""
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    _, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(batch, 11, hw)
    fqm = build_fakequant(arch, scheme, meta)
    n_stage = len(fqm.units_per_stage)
    probes = ["stage1.unit%d.quant_act_int32" % fqm.units_per_stage[0], "stage%d.unit%d.quant_act_int32" % (n_stage, fqm.units_per_stage[-1])]
    want_logits = fqm(x, trace=probes).numpy()
    want = {k: np.maximum(v.numpy(), 0) for k, v in fqm.trace.items()}            # the stream is stored after the unit's ReLU
    s_in = np.float32(meta["acts"]["quant_input"]["scale"])
    q_in = torch.from_numpy(ir.quantize_input(x.numpy(), s_in).astype(np.int8)).to(DEV)      # NHWC int8
    q = golden_model(arch, scheme, meta)
    eng = hb.compile_model(q, q_in)
    got = eng(q_in).cpu().numpy()
    assert eng.fallbacks == 0
    assert got.shape == want_logits.shape and np.array_equal(got, want_logits), \
        "rows differing from the oracle: %s" % np.nonzero((got != want_logits).any(axis=1))[0][:16].tolist()
    # residual-stream integers, eager pass through the same kernels
    rec = {}
    for name, m in q.named_modules():
        if isinstance(m, hb.q_resnet.QResidualUnit) and (name + ".quant_act_int32") in want:
            m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name + ".quant_act_int32", out[0]))
    n, h, w, c = q_in.shape
    hb.ops.reset_status(0)
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device))
    torch.cuda.synchronize()
    assert hb.ops.get_status(0) & 7 == 0
    assert set(rec) == set(want)
    for name, t in rec.items():
        g = t.int_tensor().cpu().numpy()
        assert np.array_equal(g, want[name]), (name, int((g != want[name]).sum()))
