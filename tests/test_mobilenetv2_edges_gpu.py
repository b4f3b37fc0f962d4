"""-m gpu: MobileNetV2 on the real kernels where its first tests were thin.  The whole network at the benchmarked batches, every image
and every QuantAct against the exact integer restatement; dead channels (bias integer 2^31) and ReLU6 caps that bind at every kind
of site against the reference's float arithmetic, eager and compiled; the signed stream's RESIDUAL epilogue with its low-bit copy on
the residual-projection geometries; the depthwise and stem kernels on non-square, tiny and ragged shapes, in guarded, poisoned
buffers (run_both)."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200._lib import EPI_RESIDUAL, dyadic
from hawq_b200.synthetic import synthetic_batch
from tests.engine_harness import (TABLES, assert_padded_channels_zero, assert_quantacts_equal, assert_resnet_equal, assert_rows,
                                  cap_binding, capped_float_net, capped_ranges, check_every_row, compiled_logits, dead_float_net,
                                  int8_input, int_oracle, mobilenet_case, resnet18_dead_case, run_engine, run_resnet)
from tests.kernel_harness import DEV, IO, check_stem3x3_non_square, dw_rect, out_buf, rand_act, run_both
from tests.util import golden_act_ranges, load_net_golden

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ every image at the benchmarked batches
EVERY_ROW = [("uniform8", 128, (8,)), ("uniform4", 128, (8, 4)), ("modelsize_0.5", 128, (8,)), ("bops_0.5", 128, (8, 4)),
             ("uniform8", 8, (8,)), ("uniform4", 8, (8,))]


@pytest.mark.parametrize("scheme,batch,containers", EVERY_ROW)
def test_benchmarked_batches_every_image_and_quantact(scheme, batch, containers, monkeypatch):
    _, meta = load_net_golden("mobilenetv2_w1", scheme)
    _, _, net = int_oracle(scheme, golden_act_ranges(meta), synthetic_batch(*meta["input"]))
    q = hb.build_synthetic_qresnet("mobilenetv2_w1", scheme, act_ranges=golden_act_ranges(meta))
    check_every_row(q, net, batch, containers, monkeypatch)


def test_benchmark_tool_model_every_image_and_quantact(monkeypatch):
    """The model tools/bench_mobilenetv2.py times: default calibration, its own activation ranges handed to the oracle."""
    q = hb.build_synthetic_qresnet("mobilenetv2_w1", "uniform8")
    ranges = {name: (float(m.x_min), float(m.x_max)) for name, m in q.named_modules() if isinstance(m, hb.QuantAct)}
    _, _, net = int_oracle("uniform8", ranges, synthetic_batch(2, 5))
    assert np.float32(qtensor._frozen_scale(q.quant_input)) == net.acts["quant_input"]["scale"]
    check_every_row(q, net, 128, (8,), monkeypatch)


# ------------------------------------------------------------------------------------------------ dead channels, binding caps
def eager_and_compiled(q, x, o, net):
    """The eager CUDA pass (float input) against the FakeQuant trace and IntMobileNetV2; the compiled graph's logits too."""
    y, rec = run_engine(q, x.to(DEV))
    assert_quantacts_equal(rec, o.trace)
    assert_padded_channels_zero(rec)
    want = net(x.numpy())
    assert np.array_equal(y.cpu().numpy(), want)
    assert_rows(compiled_logits(q, int8_input(x, net.acts["quant_input"]["scale"]).to(DEV)), want)
    return rec


@pytest.mark.parametrize("scheme,a4_container", TABLES)
def test_dead_channels_eager_and_compiled(scheme, a4_container, monkeypatch):
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    eager_and_compiled(*mobilenet_case(scheme, dead_float_net))


def test_dead_channels_resnet18_eager_and_compiled():
    q, x, fqm, want = resnet18_dead_case()
    y, got = run_resnet(q, x.to(DEV))
    assert_resnet_equal(got, fqm.trace)
    assert np.array_equal(y.cpu().numpy(), want)
    assert_rows(compiled_logits(q, int8_input(x, fqm.acts["quant_input"].scale.item()).to(DEV)), want)


@pytest.mark.parametrize("batch", [2, 24])
@pytest.mark.parametrize("scheme,a4_container", TABLES)
def test_relu6_caps_bind_eager_and_compiled(scheme, a4_container, batch, monkeypatch):
    """24 images: the depthwise launches end with a ragged CTA.  Per site, at least one channel sits on a cap below the clamp."""
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    q, x, o, net = mobilenet_case(scheme, capped_float_net, capped_ranges, batch)
    rec = eager_and_compiled(q, x, o, net)
    counts = cap_binding(rec, net)
    print("binding caps", scheme, a4_container, batch, counts)
    assert all(counts.values()), counts


# ------------------------------------------------------------------------------------------------ the signed stream's RESIDUAL epilogue
# MobileNetV2's residual projections (stored Cin -> stored Cout at H = W) and the logical Cout whose padded channels must stay 0
RES_GEOMS = [(192, 64, 56, 24), (192, 64, 28, 32), (384, 64, 14, 64), (576, 128, 14, 96), (960, 192, 7, 160)]


@pytest.mark.parametrize("flags", [0, 1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", RES_GEOMS)
def test_signed_stream_residual_with_low_copy(geom, a_bits, flags):
    """res_kind 0, res_bits 32, y_bits 32, relu 0 with a low-bit copy (every MobileNetV2 residual unit): signed residual operands, many
    negative, a power-of-two low ratio so that negative y land on RHE ties, 3 images so that the last row tile is ragged."""
    cin, cout, h, cout_l = geom
    n = 3
    r = np.random.RandomState(cin + cout + h + 11 * a_bits + 101 * flags)
    numel = n * h * h * cout
    x = rand_act(r, n * h * h * cin, a_bits)
    wt = np.zeros((cout, 1, 1, cin), dtype=np.int8)
    wt[:cout_l] = r.randint(-8, 8, size=(cout_l, 1, 1, cin))
    wt = torch.from_numpy(wt)
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    me = [dyadic(float(np.exp(r.uniform(np.log(1e-3), np.log(2e-2))))) for _ in range(cout_l)]
    chan = ops.make_chan(list(r.randint(-3000, 3000, size=cout_l)) + [0] * (cout - cout_l),
                         [m for m, _ in me] + [0] * (cout - cout_l), [e for _, e in me] + [1] * (cout - cout_l))
    d = ops.conv_desc(n, h, h, cin, cout, 1, 1, 1, 0, a_bits)
    for res_ratio in (0.37, 1.37):
        res = r.randint(-4000, 4000, size=numel)
        res[::7] = r.randint(-32768, 32768, size=len(res[::7]))
        res = res.reshape(-1, cout)
        res[:, cout_l:] = 0
        for low_bits, low_clamp, low_e in [(8, (-128, 127), 34), (4, (0, 15), 33)]:
            ep = ops.epilogue(EPI_RESIDUAL, relu=0, res_kind=0, res_bits=32, res_me=dyadic(res_ratio), y_bits=32, low_bits=low_bits,
                              low_me=(2 ** 30, low_e), low_clamp=low_clamp, flags=flags)
            args = dict(x=x, desc=d, ep=ep, w=wt, chan=chan, res=torch.from_numpy(res.reshape(-1).astype(np.int32)),
                        out=out_buf(numel, 32), out_low=out_buf(numel, low_bits))
            cs, gs = run_both("conv2d", args, ["out", "out_low"])
            for a, b in zip(cs, gs):
                assert torch.equal(a, b), (geom, a_bits, flags, res_ratio, low_bits)
            y = gs[0].numpy().reshape(-1, cout)
            assert (y[:, :cout_l] < 0).mean() > 0.2 and not y[:, cout_l:].any()
            low = gs[1].numpy().view(np.uint8) if low_bits == 4 else gs[1].numpy()
            assert not low.reshape(-1, cout // (8 // low_bits) if low_bits == 4 else cout)[:, cout_l // (2 if low_bits == 4 else 1):].any()


# ------------------------------------------------------------------------------------------------ depthwise and stem shapes
DW_SHAPES = [(1, 1), (1, 17), (17, 1), (2, 9), (9, 2), (3, 5), (7, 8), (8, 16), (15, 33), (33, 15)]


@pytest.mark.parametrize("hw", DW_SHAPES)
def test_dwconv_non_square_and_tiny(hw):
    hh, ww = hw
    r = np.random.RandomState(hh * 100 + ww)
    i = 0
    for c in (16, 48, 80, 1008):
        for stride in (1, 2):
            for io in IO:
                dw_rect(r, 2, hh, ww, c, stride, io, i % 3)
                i += 1


@pytest.mark.parametrize("hw", [(3, 5), (7, 8), (2, 9)])
def test_dwconv_strips_of_one_cta_span_many_images(hw):
    """Images of a few output rows and one 8-column strip each: one CTA's 256 strips cover dozens of images, the last CTA ragged."""
    hh, ww = hw
    r = np.random.RandomState(7 * hh + ww)
    for stride in (1, 2):
        for k, io in enumerate(IO):
            dw_rect(r, 77, hh, ww, 48, stride, io, k % 3)


STEM_SHAPES = [(1, 1), (1, 300), (300, 1), (6, 257), (5, 258), (223, 224), (224, 223)]


@pytest.mark.parametrize("hw", STEM_SHAPES)
def test_stem3x3_non_square(hw):
    check_stem3x3_non_square(hw)
