"""MobileNetV2 (and one ResNet-18) networks that calibrated synthetic models never produce, through the host engine with the kernels
replaced by the ABI model, batch 2: "dead" channels (all float weights 0) whose bias integer is the reference's 2^31, and ReLU6 caps
that bind at every kind of site (stem, expansion, both depthwise strides, final block).  Every QuantAct integer tensor must equal the
reference's float arithmetic (oracle/fakequant.py) and the logits the exact integer restatement (oracle/int_ref.py).  The scenario
builders are in tests/engine_harness.py, shared with tests/test_mobilenetv2_edges_gpu.py."""
import numpy as np
import pytest
import torch

from hawq_b200 import ops, qtensor
from hawq_b200.synthetic import synthetic_batch
from oracle import fakequant as fq
from oracle import int_ref as ir
from tests import abi_model as am
from tests.engine_harness import (POSITIVE, TABLES, assert_padded_channels_zero, assert_quantacts_equal, assert_resnet_equal, cap_binding,
                                  capped_float_net, capped_ranges, dead_float_net, int_oracle, mobilenet_case, resnet18_dead_case, run_engine,
                                  run_resnet)
from tests.util import golden_act_ranges, load_net_golden


def test_reference_bias_quantiser_gives_a_dead_channel_2_pow_31():
    """The 32-bit bias quantiser (quant_sym = SymmetricQuantFunction + linear_quantize) clamps in fp32 to [-2^31, 2^31 - 1], and
    2^31 - 1 is not an fp32 value: a positive folded bias over a weight scale clamped to 1e-8 / n becomes exactly 2^31, a negative
    one -2^31."""
    x = torch.tensor([0.25, -0.25, 1e-12])
    sf = torch.full((3,), 1e-8 / 127 * 0.05)
    assert fq.quant_sym(x, 32, sf).to(torch.float64).tolist() == [2.0 ** 31, -2.0 ** 31, 0.0]
    _, meta = load_net_golden("mobilenetv2_w1", "uniform4")
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
    am.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    q, x, o, net = mobilenet_case(scheme, dead_float_net)
    y, rec = run_engine(q, x)
    assert_quantacts_equal(rec, o.trace)
    assert_padded_channels_zero(rec)
    assert np.array_equal(y.numpy(), net(x.numpy()))


def test_dead_channels_resnet18(monkeypatch):
    am.install_cpu_backend(monkeypatch)
    q, x, fqm, want = resnet18_dead_case()
    y, got = run_resnet(q, x)
    assert_resnet_equal(got, fqm.trace)
    assert np.array_equal(y.numpy(), want)
    assert np.array_equal(y.numpy(), ir.IntResNet(fqm.harvest())(x.numpy()))


@pytest.mark.parametrize("scheme,a4_container", TABLES)
def test_relu6_caps_bind_at_every_kind_of_site(scheme, a4_container, monkeypatch):
    am.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    q, x, o, net = mobilenet_case(scheme, capped_float_net, capped_ranges)
    y, rec = run_engine(q, x)
    assert_quantacts_equal(rec, o.trace)
    assert np.array_equal(y.numpy(), net(x.numpy()))
    counts = cap_binding(rec, net)
    assert all(counts.values()), counts
