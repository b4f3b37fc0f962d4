"""-m gpu: the documented paths of CompiledModel (hawq_b200/engine.py) beyond one plain replay, each against an exact reference:
the pipelined call with an overflowing batch in the middle, the saturating "safe" graph taken when a requantised term leaves
int32, and the resize units built without the dual kernel (HAWQ_B200_DUAL=0)."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import qtensor
from hawq_b200._lib import EP_RATIOS_LE_2P20
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests.engine_harness import _eager, _oracle, golden_model, int8_input
from tests.kernel_harness import DEV, kernel_count
from tests.util import load_net_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("arch,scheme", [("resnet18", "bops_0.25"), ("resnet50", "modelsize_0.5")])
def test_run_pipelined_is_exact_with_an_overflowing_batch(arch, scheme):
    """run_pipelined over 7 distinct batches of 8, of which only batch 4 (every input at the int8 extremes) pushes the uint16
    residual stream past 65535; stage2.unit2's 16-bit range is shrunk to 0.75, which the other batches still fit.  Every yielded
    tensor equals eng(x) of its batch and the oracle's logits, the overflowing batch takes the exact fallback inside the pipeline
    (while batch 5 is already enqueued) exactly once, and a yielded tensor stays unchanged while the next batch is processed,
    however long that takes.  Repeated with ``post`` (argmax on the device) in a fresh engine."""
    _, meta = load_net_golden(arch, scheme)
    shrink = ("stage2.unit2.quant_act_int32", 0.75)
    q = golden_model(arch, scheme, meta, shrink)
    xs = [synthetic_batch(8, 100 + i) * (1000.0 if i == 4 else 1.0) for i in range(7)]
    fqm = _oracle(arch, scheme, meta, shrink)
    want = [fqm(x).numpy() for x in xs]
    hosts = [int8_input(x, meta["acts"]["quant_input"]["scale"]).pin_memory() for x in xs]
    devs = [h.to(DEV) for h in hosts]
    overflow = [_eager(q, x, residual_bits=16, checked=True)[1] & 1 for x in devs]
    assert overflow == [0, 0, 0, 0, 1, 0, 0], overflow

    for post in (None, lambda t: t.argmax(1)):
        eng = hb.compile_model(q, devs[0])
        got, kept = [], None
        for i, y in enumerate(eng.run_pipelined(hosts, post=post)):
            got.append(y.clone())
            torch.cuda.synchronize()              # whatever the pipeline enqueued for the next batch has run
            if kept is not None:
                assert torch.equal(kept[0], kept[1]), "the tensor yielded for batch %d changed once batch %d was yielded" % (i - 1, i)
            kept = (y, got[-1])
        assert eng.fallbacks == 1
        assert len(got) == len(hosts)
        for i, (x, g) in enumerate(zip(devs, got)):
            exact = eng(x).cpu()
            exact = exact if post is None else post(exact)
            assert torch.equal(g, exact), "batch %d: pipelined result differs from eng(x)" % i
            assert np.array_equal(g.numpy(), want[i] if post is None else want[i].argmax(1)), "batch %d differs from the oracle" % i


def test_requant_overflow_replays_the_saturating_graph():
    """A ratio > 1 term that leaves int32 under the HAWQ_EP_RATIOS_LE_2P20 promise raises HAWQ_FLAG_REQUANT_OVERFLOW; __call__
    then replays the "safe" graph (no ratio promises: generic saturating kernels, no dual launches) once, and its logits equal an
    eager forward in the same mode (int32 stream, fast_kernels=False).  stage2.unit2's 16-bit range is shrunk until the largest ratio
    of its residual launch is 2^19: every ratio of the launch, the next unit's low-bit copy included, stays <= 2^20, so the promise
    holds, and main terms exceed 2^31.  Not compared with the oracle: past int32 these kernels saturate, the reference does not."""
    arch, scheme, p = "resnet18", "uniform8", "stage2.unit2"
    _, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(2, 5)

    def launch_ratios(shrink=None):
        """main (per channel), identity and low-bit-copy ratios of p's residual launch"""
        fqm = _oracle(arch, scheme, meta, shrink)
        fqm(x)
        h = fqm.harvest()
        a, w_sf = h["acts"], h["convs"][p + ".quant_convbn2"]["w_sf"].numpy()
        s = {k: a[k]["scale"].numpy() for k in (p + ".quant_act1", "stage2.unit1.quant_act_int32", p + ".quant_act_int32",
                                                "stage3.unit1.quant_act")}
        z = s[p + ".quant_act_int32"]
        return [ir.requant_ratio(s[p + ".quant_act1"], w_sf, z), ir.requant_ratio(s["stage2.unit1.quant_act_int32"], np.float32(1.0), z),
                ir.requant_ratio(z, np.float32(1.0), s["stage3.unit1.quant_act"])]

    r0 = max(float(r.max()) for r in launch_ratios()[:2])
    shrink = (p + ".quant_act_int32", r0 / 2.0 ** 19)
    ratios = launch_ratios(shrink)
    assert 1 < max(float(r.max()) for r in ratios) <= 2.0 ** 20
    assert hb.ops.ratio_flags(*[tuple(v.tolist() for v in ir.dyadic_vec(r)) for r in ratios]) == EP_RATIOS_LE_2P20
    q = golden_model(arch, scheme, meta, shrink)
    q_in = int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV)
    _, status = _eager(q, q_in, residual_bits=16, checked=True)
    assert status & 4, status
    eng = hb.compile_model(q, q_in)
    got = eng(q_in).clone()
    assert eng.fallbacks == 1
    want, _ = _eager(q, q_in, residual_bits=32, fast_kernels=False)
    assert torch.equal(got, want)


@pytest.mark.parametrize("arch,scheme", [("resnet50", "uniform4"), ("resnet50", "bops_0.25")])
def test_resize_units_without_the_dual_kernel(arch, scheme, monkeypatch):
    """qtensor.config.dual = False (HAWQ_B200_DUAL=0) at residual_bits = 16: the resize units run as a RAW_I32 identity convolution
    plus a RESIDUAL convolution; the CUDA-graph logits equal those of the dual build, for the golden batch and a batch of 32, and no
    dual kernel is launched while this engine is compiled and run."""
    logits_g, meta = load_net_golden(arch, scheme)
    q = golden_model(arch, scheme, meta)
    xg = synthetic_batch(*meta["input"])
    s_in = meta["acts"]["quant_input"]["scale"]
    batches = [int8_input(xg, s_in).to(DEV), int8_input(torch.cat([xg, synthetic_batch(30, 77) * 1.3]), s_in).to(DEV)]
    dual = []
    for x in batches:
        before = kernel_count(4)
        dual.append(hb.compile_model(q, x)(x).clone())
        assert kernel_count(4) > before
    monkeypatch.setattr(qtensor.config, "dual", False)
    before = kernel_count(4)
    for x, want in zip(batches, dual):
        eng = hb.compile_model(q, x)
        got = eng(x)
        assert eng.fallbacks == 0
        assert torch.equal(got, want)
    torch.cuda.synchronize()
    assert kernel_count(4) == before
    assert np.array_equal(dual[0].cpu().numpy(), logits_g)
