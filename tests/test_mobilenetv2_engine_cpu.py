"""The frozen MobileNetV2 forward through the host engine (qtensor.py) with the kernels replaced by the ABI model (tests/abi_model.py):
every QuantAct integer tensor against the reference-generated goldens, the logits against the exact integer restatement, zero padded
channels, and ReLU6 caps that bind."""
import numpy as np
import pytest

import hawq_b200 as hb
from hawq_b200 import qtensor
from hawq_b200.synthetic import synthetic_batch, synthetic_float_mobilenetv2
from oracle import int_ref as ir
from tests import abi_model as am
from tests.engine_harness import SCHEMES, int_oracle, nhwc, run_engine
from tests.util import golden_act_ranges, load_net_golden, sha_i32


@pytest.mark.parametrize("a4_container", [8, 4])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_every_quantact_and_the_logits_match(scheme, a4_container, monkeypatch):
    am.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    logits_g, meta = load_net_golden("mobilenetv2_w1", scheme)
    x = synthetic_batch(*meta["input"])
    q = hb.build_synthetic_qresnet("mobilenetv2_w1", scheme, act_ranges=golden_act_ranges(meta))
    y, rec = run_engine(q, x)
    assert set(rec) == set(meta["acts"])
    for name, t in rec.items():
        assert sha_i32(nhwc(t.int_tensor().numpy())) == meta["acts"][name]["sha"], name
        n = t.node
        if n.cs != n.shape[1]:                                 # every padded channel of every stored tensor is 0
            v = am.decode(n.data, n.bits, n.signed).reshape(-1, n.cs)
            assert not v[:, n.shape[1]:].any(), name
    _, _, net = int_oracle(scheme, golden_act_ranges(meta), x)
    want = net(x.numpy())
    assert np.array_equal(y.numpy(), want)
    # the reference's classifier sums in fp32 (see tests/test_mobilenetv2_cpu.py): close to its logits, same classes
    assert np.allclose(y.numpy(), logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(y.numpy().argmax(1), logits_g.argmax(1))


def test_relu6_caps_that_bind_equal_the_reference_arithmetic(monkeypatch):
    """With calibrated ranges the ReLU6 cap never binds (the synthetic activations stay below 2).  Behind a few ReLU6 the
    convolution's BN scale is multiplied by 16 and the activation range set to x_max = 8, so values above 6 reach ReLU6 and its cap
    binds below the clamp; the engine must still give the reference's float arithmetic's integers (FakeQuantMobileNetV2) at every
    QuantAct."""
    am.install_cpu_backend(monkeypatch)
    scheme = "uniform8"
    _, meta = load_net_golden("mobilenetv2_w1", scheme)
    ranges = golden_act_ranges(meta)
    narrowed = ["features.stage2.unit1.quant_act1", "features.stage2.unit2.quant_act2", "features.stage4.unit3.quant_act2",
                "features.stage5.unit1.quant_act1"]

    def float_net():
        net = synthetic_float_mobilenetv2(0)
        for name in narrowed:
            unit = net.features
            for part in name.split(".")[1:-1]:
                unit = getattr(unit, part)
            getattr(unit, "conv" + name[-1]).bn.weight.data.mul_(16.0)
        return net

    for name in narrowed:
        ranges[name] = (ranges[name][0], 8.0)
    x = synthetic_batch(*meta["input"])
    q = hb.q_mobilenetv2_w1(float_net())
    assert hb.stamp_bit_config(q, hb.get_bit_config("mobilenetv2_w1", scheme)) > 0
    q.eval()
    for name, m in q.named_modules():
        if isinstance(m, hb.QuantAct):
            m.x_min.fill_(ranges[name][0])
            m.x_max.fill_(ranges[name][1])
    hb.freeze_model(q)
    y, rec = run_engine(q, x)
    o, yf, net = int_oracle(scheme, ranges, x, float_net())
    for name, t in rec.items():
        assert np.array_equal(t.int_tensor().numpy(), o.trace[name].numpy()), name
    assert np.array_equal(y.numpy(), net(x.numpy()))
    # at least one channel of a narrowed activation sits on a cap below the clamp
    binding = 0
    for name in narrowed:
        unit, act = name.rsplit(".", 1)
        conv = "%s.conv%s" % (unit, act[-1])
        a_prev = net.acts[unit + (".quant_act" if act == "quant_act1" else ".quant_act1")]["scale"]
        a = net.acts[name]
        m, e = ir.dyadic_vec(ir.requant_ratio(a_prev, net.convs[conv]["w_sf"], a["scale"]))
        hi = ir.clamp_range(a["bits"], a["mode"])[1]
        cap = ir.requant(ir.relu6_cap(a_prev, net.convs[conv]["w_sf"]), m, e)
        got = nhwc(rec[name].int_tensor().numpy()).reshape(-1, len(cap)).max(axis=0)
        binding += int(((cap < hi) & (got == cap)).sum())
    assert binding > 0
