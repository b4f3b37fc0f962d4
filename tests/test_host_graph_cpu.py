"""Host logic of the product (quant modules, lazy fusion in qtensor.py, parameter preparation, descriptors) on CPU:
the C-ABI launchers are replaced by the numpy ABI model (tests/abi_model.py), everything else is the product code.
Checked against the reference-generated goldens (bit-equal logits) and the oracle's full activation tensors."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200.build import build_library
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests import abi_model
from tests.util import RESNET_GOLDENS, build_fakequant, golden_act_ranges, load_net_golden, sha_i32


@pytest.fixture(scope="session", autouse=True)
def _lib():
    build_library()


def _hook_outputs(q):
    rec = {}
    hooks = []
    for name, m in q.named_modules():
        if isinstance(m, hb.QuantAct) or isinstance(m, hb.q_resnet.QResidualUnit):
            hooks.append(m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name, out[0])))
    return rec, hooks


@pytest.mark.parametrize("arch,scheme,res_bits,a4_container",
                         [(a, s) + ((16, 8) if i % 2 == 0 else (32, 4)) for i, (a, s) in enumerate(RESNET_GOLDENS)])
def test_frozen_graph_matches_golden(monkeypatch, arch, scheme, res_bits, a4_container):
    """a4_container: 4-bit activations stored one per byte (default) or as packed nibbles - same integers either way.  The
    goldens alternate between the uint16 stream with byte containers and the int32 stream with packed nibbles."""
    abi_model.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    logits_g, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(*meta["input"])
    # oracle trace (full tensors), itself pinned to the golden checksums
    fqm = build_fakequant(arch, scheme, meta)
    fqm(x, trace=False)
    net_i = ir.IntResNet(fqm.harvest())
    li = net_i(x.numpy(), trace=True)
    assert np.array_equal(li, logits_g)
    for k, v in meta["acts"].items():
        assert sha_i32(net_i.trace[k].reshape(v["shape"])) == v["sha"], k

    q = hb.build_synthetic_qresnet(arch, scheme, act_ranges=golden_act_ranges(meta))
    rec, hooks = _hook_outputs(q)
    monkeypatch.setattr(qtensor.config, "residual_bits", res_bits)
    with torch.no_grad():
        out = q(x)
    assert out.dtype == torch.float32 and tuple(out.shape) == (x.shape[0], 1000)
    assert np.array_equal(out.numpy(), logits_g)
    checked = 0
    for name, t in rec.items():
        if not isinstance(t, hb.IntActivation):
            continue
        if name in net_i.trace:                                  # QuantAct outputs
            want = net_i.trace[name]
            if t.node.kind != "int":
                continue                                         # pending residual (pre-ReLU): checked via the unit output
            got = t.int_tensor().numpy()
            got = got.transpose(0, 2, 3, 1) if got.ndim == 4 else got
            assert np.array_equal(got.reshape(want.shape), want), name
            checked += 1
        else:                                                    # unit outputs = ReLU(quant_act_int32)
            want = np.maximum(net_i.trace[name + ".quant_act_int32"], 0)
            got = t.int_tensor().numpy().transpose(0, 2, 3, 1)
            assert np.array_equal(got, want), name
            checked += 1
    assert checked >= len(meta["acts"]) - 2
    for h in hooks:
        h.remove()
    if res_bits == 16:
        # the mode CompiledModel runs: checked, so the 4-bit schemes may promise ratios <= 2^20 too.  Every bottleneck resize
        # unit takes the dual kernel; ResNet-18's resize units are 3x3 and never do
        duals = []
        monkeypatch.setattr(ops, "conv2d_dual", lambda *a, **kw: (duals.append(a), abi_model.conv2d_dual(*a, **kw)))
        with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
            out = q(x)
        assert np.array_equal(out.numpy(), logits_g)
        assert len(duals) == (0 if arch == "resnet18" else 4)


def test_frozen_requires_cuda():
    q = hb.build_synthetic_qresnet("resnet18", "uniform8", calib_batch=1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        q(synthetic_batch(1, 1))


def test_state_dict_keys_match_reference_layout():
    q = hb.build_synthetic_qresnet("resnet50", "uniform8", calib_batch=1)
    keys = set(q.state_dict().keys())
    for k in ("quant_input.x_min", "quant_init_convbn.conv.weight", "quant_init_convbn.bn.running_var",
              "quant_init_convbn.convbn_scaling_factor", "quant_init_convbn.weight_integer",
              "stage1.unit1.quant_identity_convbn.bias_integer", "stage4.unit3.quant_act_int32.act_scaling_factor",
              "stage2.unit1.quant_act.pre_weight_scaling_factor", "quant_output.fc_scaling_factor",
              "quant_output.weight_integer", "quant_output.bias_integer", "quant_output.weight"):
        assert k in keys, k
    names = dict(q.named_modules())
    for name in hb.get_bit_config("resnet50", "bops_0.5"):
        assert name in names, name
