"""The oracle restatements (oracle/fakequant.py, oracle/int_ref.py) against the golden vectors that
tests/golden/make_golden.py produced by running the unmodified reference.  CPU only."""
import json

import numpy as np
import pytest
import torch

from oracle import fakequant as fq
from oracle import int_ref as ir
from tests.util import RESNET_GOLDENS, load_golden, load_net_golden, sha_i32, build_fakequant
from hawq_b200.synthetic import synthetic_batch


def test_batch_frexp_kat():
    g = load_golden("kat_requant.npz")
    for r, m, e in zip(g["frexp_ratio"], g["frexp_m"], g["frexp_e"]):
        assert ir.dyadic(r) == (int(m), int(e))
    m2, e2 = fq.batch_frexp(torch.from_numpy(g["frexp_ratio"]))
    assert np.array_equal(m2.numpy(), g["frexp_m"]) and np.array_equal(e2.numpy().astype(np.int64), g["frexp_e"])
    assert ir.dyadic(0.25) == (1073741824, 32) and ir.dyadic(0.3) == (1288490189, 32)   # SURVEY A.7


def test_case0_kat():
    g = load_golden("kat_requant.npz")
    specs = json.loads(str(g["c0_specs"]))
    for i, sp in enumerate(specs):
        acc = g["c0_%d_acc" % i]                                  # [N,C,H,W]
        m, e = ir.dyadic_vec(ir.requant_ratio(g["c0_%d_a_sf" % i], g["c0_%d_w_sf" % i], g["c0_%d_z_sf" % i]))
        lo, hi = ir.clamp_range(sp["bits"], sp["mode"])
        a = acc.transpose(0, 2, 3, 1)
        want = g["c0_%d_q" % i].transpose(0, 2, 3, 1)
        assert np.array_equal(np.clip(ir.requant(a, m, e), lo, hi), want)
        assert np.array_equal(np.clip(ir.requant_fp64(a, m, e), lo, hi), want)


def test_survey_a7_vectors():
    g = load_golden("kat_requant.npz")
    for ratio, acc, q in json.loads(str(g["a7"])):
        m, e = ir.dyadic_vec(ir.requant_ratio(1.0, np.float32(ratio), 1.0))
        assert ir.requant(np.array(acc), m, e).reshape(-1).tolist() == q
    # ties go to even (the reference is NOT TVM's round-half-up): acc=8, ratio 1/16 -> 0
    m, e = ir.dyadic_vec([1.0 / 16])
    assert ir.requant(np.array([8, 24, -8, -24]), m, e).tolist() == [0, 2, 0, -2]


def test_case1_kat():
    g = load_golden("kat_requant.npz")
    for i in range(3):
        acc = g["c1_%d_acc" % i].transpose(0, 2, 3, 1)
        idn = g["c1_%d_id" % i].transpose(0, 2, 3, 1)
        z_sf = g["c1_%d_z_sf" % i]
        m1, e1 = ir.dyadic_vec(ir.requant_ratio(g["c1_%d_id_sf" % i], g["c1_%d_id_w_sf" % i], z_sf))
        m2, e2 = ir.dyadic_vec(ir.requant_ratio(g["c1_%d_a_sf" % i], g["c1_%d_w_sf" % i], z_sf))
        got = ir.requant(idn, m1, e1) + ir.requant(acc, m2, e2)
        assert np.array_equal(got, g["c1_%d_q" % i].transpose(0, 2, 3, 1))


def test_module_kats():
    g = load_golden("kat_modules.npz")
    # input quantisation
    for bits, mode in [(8, 'symmetric'), (4, 'asymmetric')]:
        q = ir.quantize_input(g["act_in_%d_x" % bits], g["act_in_%d_scale" % bits][0], bits, mode)
        assert np.array_equal(q, g["act_in_%d_q" % bits].transpose(0, 2, 3, 1))
    # folded-BN conv: fakequant restatement reproduces weight_integer / bias_integer / accumulators
    for tag in ("bnconv_a", "bnconv_b"):
        cin, cout, k, s, p, wb = [int(v) for v in g[tag + "_cfg"]]
        conv = torch.nn.Conv2d(cin, cout, k, s, p, bias=False)
        bn = torch.nn.BatchNorm2d(cout)
        with torch.no_grad():
            conv.weight.copy_(torch.from_numpy(g[tag + "_conv_w"]))
            mean, var, w, b = [torch.from_numpy(v) for v in g[tag + "_bn"]]
            bn.running_mean.copy_(mean); bn.running_var.copy_(var); bn.weight.copy_(w); bn.bias.copy_(b)
        st = fq.ConvBnState(conv, bn, wbits=wb)
        a_sf = torch.from_numpy(g[tag + "_a_sf"])
        xi = torch.from_numpy(g[tag + "_x_int"]).float()
        with torch.no_grad():
            st(xi * a_sf, a_sf)
        assert np.array_equal(st.weight_integer.long().numpy(), g[tag + "_w_int"])
        assert np.array_equal(st.bias_integer.long().numpy(), g[tag + "_b_int"])
        assert np.array_equal(st.w_sf.numpy(), g[tag + "_w_sf"])
        acc = ir.conv2d_nhwc(g[tag + "_x_int"].transpose(0, 2, 3, 1), g[tag + "_w_int"].transpose(0, 2, 3, 1), s, p) + g[tag + "_b_int"]
        assert np.array_equal(acc, g[tag + "_acc"].transpose(0, 2, 3, 1))
    # plain conv with bias
    conv = torch.nn.Conv2d(8, 8, 3, 1, 1, bias=True)
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(g["conv_w"])); conv.bias.copy_(torch.from_numpy(g["conv_b"]))
    st = fq.ConvState(conv, wbits=8)
    a_sf = torch.from_numpy(g["conv_a_sf"])
    with torch.no_grad():
        st(torch.from_numpy(g["conv_x_int"]).float() * a_sf, a_sf)
    assert np.array_equal(st.weight_integer.long().numpy(), g["conv_w_int"])
    assert np.array_equal(st.bias_integer.long().numpy(), g["conv_b_int"])
    acc = ir.conv2d_nhwc(g["conv_x_int"].transpose(0, 2, 3, 1), g["conv_w_int"].transpose(0, 2, 3, 1), 1, 1) + g["conv_b_int"]
    assert np.array_equal(acc, g["conv_acc"].transpose(0, 2, 3, 1))
    # linear
    lin = torch.nn.Linear(32, 10)
    with torch.no_grad():
        lin.weight.copy_(torch.from_numpy(g["lin_w"])); lin.bias.copy_(torch.from_numpy(g["lin_b"]))
    st = fq.LinearState(lin, wbits=8)
    a_sf = torch.from_numpy(g["lin_a_sf"])
    with torch.no_grad():
        y = st(torch.from_numpy(g["lin_x_int"]).float() * a_sf, a_sf)
    assert np.array_equal(st.weight_integer.long().numpy(), g["lin_w_int"])
    assert np.array_equal(st.bias_integer.long().numpy(), g["lin_b_int"])
    assert np.array_equal(y.numpy(), g["lin_y"])
    acc = ir.linear(g["lin_x_int"], g["lin_w_int"]) + g["lin_b_int"]
    scale = (g["lin_w_sf"] * g["lin_a_sf"][0]).astype(np.float32)
    assert np.array_equal(acc.astype(np.float32) * scale, g["lin_y"])
    # average pool incl. negative sums
    q = ir.avgpool_trunc(g["pool_x_int"].transpose(0, 2, 3, 1), 7)
    assert np.array_equal(q, g["pool_q"].transpose(0, 2, 3, 1))


@pytest.mark.parametrize("arch,scheme", RESNET_GOLDENS)
def test_network_golden(arch, scheme):
    """Whole network: fakequant and int_ref reproduce the reference's activation integers (sha256 over every
    QuantAct output), integer weights and bit-equal logits."""
    torch.set_num_threads(max(1, torch.get_num_threads()))
    logits, meta = load_net_golden(arch, scheme)
    m = build_fakequant(arch, scheme, meta)
    x = synthetic_batch(*meta["input"])
    l_fq = m(x, trace=True)
    assert np.array_equal(l_fq.numpy(), logits)
    for k, v in meta["acts"].items():
        a = m.trace[k].numpy()
        a = a.transpose(0, 2, 3, 1) if a.ndim == 4 else a
        assert sha_i32(a) == v["sha"], k
        assert abs(float(m.acts[k].scale) - v["scale"]) == 0
    h = m.harvest()
    for k, v in meta["convs"].items():
        assert sha_i32(h["convs"][k]["weight_integer"].numpy().transpose(0, 2, 3, 1)) == v["w_sha"], k
        assert sha_i32(h["convs"][k]["bias_integer"].numpy()) == v["b_sha"], k
    net_i = ir.IntResNet(h)
    l_int = net_i(x.numpy(), trace=True)
    assert np.array_equal(l_int, logits)
    for k, v in meta["acts"].items():
        assert sha_i32(net_i.trace[k].reshape(v["shape"])) == v["sha"], k
