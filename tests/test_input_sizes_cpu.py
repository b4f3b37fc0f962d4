"""Input sizes other than 224 x 224 (tests/golden/size_<arch>_<scheme>_<H>x<W>.npz, made by the unmodified reference with the parity
batch drawn at H x W; same model, same calibration at 224).  Any input whose last feature map is 7 x 7 runs: 193 gives odd maps in
every stage (97, 49, 25, 13, 7), H != W gives unequal ones.  The oracle reproduces these goldens, and so does the host engine
(qtensor.py, which plans every launch from the input's shape) with its kernels replaced by the ABI model (tests/abi_model.py)."""
import json

import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import qtensor
from hawq_b200.build import build_library
from tests import abi_model as am
from tests.engine_harness import SIZE_GOLDENS, check_engine_against_golden, engine_outputs, load_size_golden, nhwc, oracle_for
from tests.util import golden_act_ranges, load_golden, sha_i32


def test_the_size_goldens():
    """Odd and unequal maps in every stage, both ResNet families and MobileNetV2, and the ResNet goldens left to the 224 tests."""
    hws = set()
    for name in SIZE_GOLDENS:
        _, meta, x = load_size_golden(name)
        n, c, h, w = x.shape
        assert name == "size_%s_%s_%dx%d.npz" % (meta["arch"], meta["scheme"], h, w)
        assert (h, w) != (224, 224) and meta["acts"]["quant_input"]["shape"] == [n, h, w, 3]
        hws.add((h, w))
    assert {(193, 193), (193, 224), (224, 193), (200, 216)} <= hws
    assert {load_size_golden(f)[1]["arch"] for f in SIZE_GOLDENS} == {"resnet18", "resnet50", "mobilenetv2_w1"}
    assert not any(f.startswith("net_") for f in SIZE_GOLDENS)


@pytest.mark.parametrize("name", SIZE_GOLDENS)
def test_oracle_reproduces_the_golden(name):
    """The FakeQuant oracle gives the reference's integers at every QuantAct and its logits; the integer restatement its integers,
    and its logits (ResNet) or their fp32-summed approximation (MobileNetV2).  The activation ranges are the 224 golden's: one
    model serves every input size."""
    logits_g, meta, x = load_size_golden(name)
    arch, scheme = meta["arch"], meta["scheme"]
    ranges_224 = json.loads(str(load_golden("net_%s_%s.npz" % (arch, scheme))["meta"]))["acts"]
    assert golden_act_ranges(meta) == {k: (v["x_min"], v["x_max"]) for k, v in ranges_224.items()}
    o, yf, net = oracle_for(meta, x)
    assert np.array_equal(yf, logits_g)
    assert set(o.trace) >= set(meta["acts"])
    for k, v in meta["acts"].items():
        t = o.trace[k]
        assert sha_i32(nhwc(t.numpy() if torch.is_tensor(t) else t)) == v["sha"], k
    yi = net(x.numpy(), trace=True)
    for k, v in meta["acts"].items():
        assert sha_i32(net.trace[k].reshape(v["shape"])) == v["sha"], k
    if arch == "mobilenetv2_w1":
        assert np.allclose(yi, logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(yi.argmax(1), logits_g.argmax(1))
    else:
        assert np.array_equal(yi, logits_g)


@pytest.fixture(scope="module")
def _lib():
    build_library()


@pytest.mark.parametrize("name", SIZE_GOLDENS)
def test_host_engine_on_the_abi_model_matches_the_golden(name, _lib, monkeypatch):
    """The uint16 stream with 4-bit activations in byte containers on one half of the goldens, the int32 stream with packed nibbles
    on the other."""
    logits_g, meta, x = load_size_golden(name)
    i = SIZE_GOLDENS.index(name)
    am.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "residual_bits", 16 if i % 2 == 0 else 32)
    monkeypatch.setattr(qtensor.config, "a4_container", 8 if i % 2 == 0 else 4)
    q = hb.build_synthetic_qresnet(meta["arch"], meta["scheme"], act_ranges=golden_act_ranges(meta))
    y, acts, units = engine_outputs(q, x)
    _, _, net = oracle_for(meta, x)
    check_engine_against_golden(y, acts, units, meta, logits_g, net, x)
