"""-m gpu: CompiledModel's fallback paths on MobileNetV2, and two networks compiled on one device.  The signed int32 stream's
RESIDUAL launches run under the HAWQ_EP_RATIOS_LE_2P20 promise in checked mode, so a requantised term that leaves int32 raises
HAWQ_FLAG_REQUANT_OVERFLOW and __call__ replays the saturating "safe" graph: here built for a network with depthwise and 3x3-stem
launches and int32 streams, taken from __call__ and from inside a pipelined run.  Each result is compared with an exact reference:
the golden logits and IntMobileNetV2 where the fast path holds, an eager forward in the safe graph's mode where it saturates."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops
from hawq_b200._lib import EP_RATIOS_LE_2P20
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests.engine_harness import _eager, int8_input, int_oracle
from tests.kernel_harness import DEV, kernel_count
from tests.util import golden_act_ranges, load_net_golden

pytestmark = pytest.mark.gpu
SCHEME = "uniform8"
P = "features.stage3.unit2"          # a case-1 unit: 32 -> 32 channels at 28 x 28, its input as the identity
Z = P + ".quant_act_int32"


def shrunk_ranges(meta, f):
    r = golden_act_ranges(meta)
    r[Z] = (r[Z][0] * f, r[Z][1] * f)
    return r


def launch_ratios(meta, f):
    """main (per channel), identity and next-unit low-bit-copy ratios of P's RESIDUAL launch with Z's range scaled by f."""
    _, _, net = int_oracle(SCHEME, shrunk_ranges(meta, f), synthetic_batch(2, 5))
    s = {k: v["scale"] for k, v in net.acts.items()}
    return [ir.requant_ratio(s[P + ".quant_act2"], net.convs[P + ".conv3"]["w_sf"], s[Z]),
            ir.requant_ratio(s["features.stage3.unit1.quant_act_int32"], np.float32(1.0), s[Z]),
            ir.requant_ratio(s[Z], np.float32(1.0), s["features.stage3.unit3.quant_act"])], net


def shrunk_case(log2_ratio):
    """(meta, ranges, IntMobileNetV2, the model) with Z's range shrunk until the largest ratio of P's launch is 2^log2_ratio; asserts
    that the launch keeps the LE_2P20 promise."""
    _, meta = load_net_golden("mobilenetv2_w1", SCHEME)
    r0 = max(float(r.max()) for r in launch_ratios(meta, 1.0)[0][:2])
    f = r0 / 2.0 ** log2_ratio
    ratios, net = launch_ratios(meta, f)
    assert 1 < max(float(r.max()) for r in ratios) <= 2.0 ** 20
    assert ops.ratio_flags(*[tuple(v.tolist() for v in ir.dyadic_vec(r)) for r in ratios]) == EP_RATIOS_LE_2P20
    ranges = shrunk_ranges(meta, f)
    return meta, ranges, net, hb.build_synthetic_qresnet("mobilenetv2_w1", SCHEME, act_ranges=ranges)


def test_requant_overflow_replays_the_saturating_graph():
    """P's largest ratio at 2^19: main terms leave int32, the eager checked pass raises flag 4, and eng(x) takes one fallback to the
    safe graph, whose logits equal an eager forward with residual_bits=32, fast_kernels=False.  Building the safe graph runs the
    forward three times through the launchers (warm-up, second pass, capture), each with 17 depthwise and 1 stem launch."""
    _, _, net, q = shrunk_case(19)
    x = int8_input(synthetic_batch(2, 5), net.acts["quant_input"]["scale"]).to(DEV)
    _, status = _eager(q, x, residual_bits=16, checked=True)
    assert status & 4, status
    eng = hb.compile_model(q, x)
    before = [kernel_count(1), kernel_count(2)]
    got = eng(x).clone()
    torch.cuda.synchronize()
    assert eng.fallbacks == 1 and "safe" in eng.graphs
    assert [kernel_count(1) - before[0], kernel_count(2) - before[1]] == [3 * 17, 3 * 1]
    want, status = _eager(q, x, residual_bits=32, fast_kernels=False)
    assert status & 7 == 0
    assert torch.equal(got, want)
    assert torch.equal(eng(x), want) and eng.fallbacks == 2           # the safe graph is built once and replayed


def test_run_pipelined_takes_the_saturating_fallback_for_every_batch():
    """run_pipelined over 6 batches of 8 (the fourth scaled by 1.3) with P's largest ratio at 2^19.  No shrink of P's range
    separates batches here: on the integer model, with the ratio at 2^15 no batch of 8 raises flag 4, not even one at the int8
    extremes, and from 2^15.5 every batch does.  So every batch raises it (asserted with the eager status word), the pipeline takes
    the safe graph once per batch while the next batch is already enqueued, and every yielded tensor equals eng(x) of its batch and
    an eager forward in the safe graph's mode."""
    _, _, net, q = shrunk_case(19)
    xs = [synthetic_batch(8, 400 + i) * (1.3 if i == 3 else 1.0) for i in range(6)]
    hosts = [int8_input(x, net.acts["quant_input"]["scale"]).pin_memory() for x in xs]
    devs = [h.to(DEV) for h in hosts]
    flags = [_eager(q, x, residual_bits=16, checked=True)[1] & 7 for x in devs]
    assert flags == [4] * len(xs), flags
    eng = hb.compile_model(q, devs[0])
    got = [y.clone() for y in eng.run_pipelined(hosts)]
    assert eng.fallbacks == len(xs)
    assert len(got) == len(hosts)
    for i, (x, g) in enumerate(zip(devs, got)):
        assert torch.equal(g, eng(x).cpu()), "batch %d: pipelined result differs from eng(x)" % i
        assert torch.equal(g, _eager(q, x, residual_bits=32, fast_kernels=False)[0].cpu()), "batch %d: differs from the eager safe mode" % i


def test_mobilenetv2_and_resnet50_replayed_alternately_on_one_stream():
    """A MobileNetV2 engine and a ResNet-50 engine compiled on one device share its default handle, SM count and kernel attributes;
    replayed alternately on one stream, three rounds, each equals its golden logits (MobileNetV2: exactly IntMobileNetV2, and the
    reference's fp32-summed logits closely) and raises no flag."""
    logits_r, meta_r = load_net_golden("resnet50", "uniform8")
    xr = int8_input(synthetic_batch(*meta_r["input"]), meta_r["acts"]["quant_input"]["scale"]).to(DEV)
    qr = hb.build_synthetic_qresnet("resnet50", "uniform8", act_ranges=golden_act_ranges(meta_r))
    logits_m, meta_m = load_net_golden("mobilenetv2_w1", SCHEME)
    xm_f = synthetic_batch(*meta_m["input"])
    _, _, net = int_oracle(SCHEME, golden_act_ranges(meta_m), xm_f)
    want_m = net(xm_f.numpy())
    assert np.allclose(want_m, logits_m, rtol=2e-6, atol=2e-7) and np.array_equal(want_m.argmax(1), logits_m.argmax(1))
    xm = int8_input(xm_f, net.acts["quant_input"]["scale"]).to(DEV)
    qm = hb.build_synthetic_qresnet("mobilenetv2_w1", SCHEME, act_ranges=golden_act_ranges(meta_m))
    em = hb.compile_model(qm, xm)
    er = hb.compile_model(qr, xr)
    rounds = []
    for _ in range(3):
        rounds.append((em.run_async(xm).clone(), em.flag.clone(), er.run_async(xr).clone(), er.flag.clone()))
    torch.cuda.synchronize()
    for k, (ym, fm, yr, fr) in enumerate(rounds):
        assert (int(fm), int(fr)) == (0, 0), k
        assert np.array_equal(ym.cpu().numpy(), want_m), "round %d: MobileNetV2" % k
        assert np.array_equal(yr.cpu().numpy(), logits_r), "round %d: ResNet-50" % k
