"""MobileNetV2 (and one ResNet-18) networks that calibrated synthetic models never produce, through the host engine with the kernels
replaced by the ABI model, batch 2: "dead" channels (all float weights 0) whose bias integer is the reference's 2^31, and ReLU6 caps
that bind at every kind of site (stem, expansion, both depthwise strides, final block).  Every QuantAct integer tensor must equal the
reference's float arithmetic (oracle/fakequant.py) and the logits the exact integer restatement (oracle/int_ref.py).  The scenario
builders here are shared with tests/test_mobilenetv2_edges_gpu.py."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200.synthetic import synthetic_batch, synthetic_float_mobilenetv2, synthetic_float_resnet
from oracle import fakequant as fq
from oracle import int_ref as ir
from tests import abi_model as am
from tests import abi_model_mobilenetv2 as amm
from tests.test_mobilenetv2_engine_cpu import int_oracle, load, nhwc, run_engine
from tests.util import golden_act_ranges, load_net_golden

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
    _, meta = load(scheme)
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


def test_reference_bias_quantiser_gives_a_dead_channel_2_pow_31():
    """The 32-bit bias quantiser (quant_sym = SymmetricQuantFunction + linear_quantize) clamps in fp32 to [-2^31, 2^31 - 1], and
    2^31 - 1 is not an fp32 value: a positive folded bias over a weight scale clamped to 1e-8 / n becomes exactly 2^31, a negative
    one -2^31."""
    x = torch.tensor([0.25, -0.25, 1e-12])
    sf = torch.full((3,), 1e-8 / 127 * 0.05)
    assert fq.quant_sym(x, 32, sf).to(torch.float64).tolist() == [2.0 ** 31, -2.0 ** 31, 0.0]
    _, meta = load("uniform4")
    o, _, _ = int_oracle("uniform4", golden_act_ranges(meta), synthetic_batch(*meta["input"]), dead_float_net())
    convs = o.harvest()["convs"]
    for name, c in [("features.stage2.unit2.conv2", 3)] + sorted(POSITIVE):
        assert int(convs[name]["bias_integer"][c]) == 2 ** 31, (name, c)


def test_make_chan_never_wraps_a_bias():
    """2^31 on a channel whose accumulator is identically 0 is stored exactly as (2^30, m, e - 1); without that knowledge, with
    e - 1 < 31 (a promise made from the original pairs would break) or beyond -2^31, make_chan raises."""
    m, e = 1717986918, 61
    t = ops.make_chan([2 ** 31, 5, -2 ** 31], [m, m, m], [e, e, e], zero_acc=[True, False, False]).numpy()
    assert t[:, 0].tolist() == [2 ** 30, 5, -2 ** 31] and t[:, 2].tolist() == [e - 1, e, e]
    assert t[:, 1].view(np.uint32).tolist() == [m] * 3
    assert ops.rhe_requant_host(2 ** 30, m, e - 1) == ir.requant(np.array([2 ** 31]), m, e)[0]     # RHE(2^31 * m / 2^e), exactly
    t = ops.make_chan([2 ** 31], [0], [1], zero_acc=[True]).numpy()       # ratio 0: the output is 0 whatever the bias
    assert t[0, :3].tolist() == [0, 0, 1]
    for bias, zero_acc, ee, raw in [([2 ** 31], None, 61, False), ([2 ** 31], [False], 61, False), ([2 ** 31], [True], 31, False),
                                    ([-2 ** 31 - 1], [True], 61, False), ([2 ** 31], [True], 61, True)]:
        with pytest.raises(OverflowError, match="leaves int32"):
            ops.make_chan(bias, [m], [ee], zero_acc=zero_acc, raw=raw)


def test_int_oracle_follows_the_reference_on_a_2_pow_31_bias():
    """The integer restatement accepts the dead channel's accumulator 2^31 (requant) and still refuses an accumulator that leaves
    int32 on a channel with a weight."""
    assert ir.requant(np.array([2 ** 31]), 2 ** 31, 62)[0] == 1
    with pytest.raises(AssertionError, match="leaves int32"):
        ir.requant(np.array([2 ** 31 + 1]), 1, 1)
    w = np.zeros((2, 1, 1, 1), dtype=np.int64)
    w[1] = 1
    y = ir.conv_bias(np.zeros((1, 2), dtype=np.int64), w, np.array([2 ** 31, 0]))
    assert y.tolist() == [[2 ** 31, 0]]
    with pytest.raises(AssertionError, match="leaves int32"):
        ir.conv_bias(np.ones((1, 2), dtype=np.int64), w, np.array([0, 2 ** 31 - 1]))


@pytest.mark.parametrize("scheme,a4_container", TABLES)
def test_dead_channels_equal_the_reference(scheme, a4_container, monkeypatch):
    amm.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    q, x, o, net = mobilenet_case(scheme, dead_float_net)
    y, rec = run_engine(q, x)
    assert_quantacts_equal(rec, o.trace)
    assert_padded_channels_zero(rec)
    assert np.array_equal(y.numpy(), net(x.numpy()))


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


def test_dead_channels_resnet18(monkeypatch):
    am.install_cpu_backend(monkeypatch)
    q, x, fqm, want = resnet18_dead_case()
    y, got = run_resnet(q, x)
    assert_resnet_equal(got, fqm.trace)
    assert np.array_equal(y.numpy(), want)
    assert np.array_equal(y.numpy(), ir.IntResNet(fqm.harvest())(x.numpy()))


@pytest.mark.parametrize("scheme,a4_container", TABLES)
def test_relu6_caps_bind_at_every_kind_of_site(scheme, a4_container, monkeypatch):
    amm.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    q, x, o, net = mobilenet_case(scheme, capped_float_net, capped_ranges)
    y, rec = run_engine(q, x)
    assert_quantacts_equal(rec, o.trace)
    assert np.array_equal(y.numpy(), net(x.numpy()))
    counts = cap_binding(rec, net)
    assert all(counts.values()), counts
