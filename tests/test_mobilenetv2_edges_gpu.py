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
from oracle import int_ref as ir
from tests import abi_model as am
from tests.test_kernels_gpu import out_buf, rand_act
from tests.test_mobilenetv2_edges_cpu import (TABLES, assert_padded_channels_zero, assert_quantacts_equal, assert_resnet_equal,
                                              cap_binding, capped_float_net, capped_ranges, dead_float_net, mobilenet_case,
                                              resnet18_dead_case, run_resnet)
from tests.test_mobilenetv2_engine_cpu import int_oracle, load, run_engine
from tests.test_mobilenetv2_gpu import IO, act_in, chan_for, run_both
from tests.util import golden_act_ranges

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def int_input(x, scale):
    """NHWC int8 network input on the device, quantised like the reference's quant_input."""
    return torch.from_numpy(ir.quantize_input(x.numpy(), np.float32(scale)).astype(np.int8)).to(DEV)


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


def assert_rows(got, want):
    assert got.shape == want.shape and np.array_equal(got, want), \
        "rows differing from the oracle: %s" % np.nonzero((got != want).any(axis=1))[0][:16].tolist()


# ------------------------------------------------------------------------------------------------ every image at the benchmarked batches
EVERY_ROW = [("uniform8", 128, (8,)), ("uniform4", 128, (8, 4)), ("modelsize_0.5", 128, (8,)), ("bops_0.5", 128, (8, 4)),
             ("uniform8", 8, (8,)), ("uniform4", 8, (8,))]
CHUNK = 16          # images per oracle pass: a full IntMobileNetV2 trace is about 1 GB per 16 images


def check_every_row(q, net, batch, containers, monkeypatch, hw=224):
    """Compiled logits of synthetic_batch(batch, 11, hw) against IntMobileNetV2 on every row, and every QuantAct of every image of a
    checked eager pass, per 4-bit container; the oracle runs CHUNK images at a time."""
    x = synthetic_batch(batch, 11, hw)
    q_in = int_input(x, net.acts["quant_input"]["scale"])
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


@pytest.mark.parametrize("scheme,batch,containers", EVERY_ROW)
def test_benchmarked_batches_every_image_and_quantact(scheme, batch, containers, monkeypatch):
    _, meta = load(scheme)
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
    assert_rows(compiled_logits(q, int_input(x, net.acts["quant_input"]["scale"])), want)
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
    assert_rows(compiled_logits(q, int_input(x, fqm.acts["quant_input"].scale.item())), want)


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


def pow2_chan(r, c):
    """Power-of-two ratios 2^-k (m = 2^30, e = 30 + k): with relu 0 negative accumulators land on RHE ties."""
    k = r.randint(1, 12, size=c)
    return ops.make_chan(r.randint(-64, 64, size=c) * 2 ** 6, [2 ** 30] * c, list(30 + k), [2 ** 31 - 1] * c)


def dw_rect(r, n, hh, ww, c, stride, io, variant):
    """variant 0: random data, ReLU6 caps on some channels; 1: power-of-two ratios, relu 0; 2: x = w = -128 (int8 inputs; 15 in a
    4-bit input), power-of-two ratios, relu 0."""
    a_bits, kind, out_bits, clamp = io
    ho, wo = (hh - 1) // stride + 1, (ww - 1) // stride + 1
    if variant == 2:
        v = -128 if kind == "s8" else 15
        x = torch.full((n * hh * ww * c,), v, dtype=torch.int8) if a_bits == 8 else torch.from_numpy(am.pack_i4(np.full(n * hh * ww * c, 15)))
        w = torch.full((3, 3, c), -128, dtype=torch.int8)
    else:
        x = act_in(r, n * hh * ww * c, kind, a_bits)
        w = torch.from_numpy(r.randint(-128, 128, size=(3, 3, c)).astype(np.int8))
    relu = 2 if variant == 0 else 0
    chan = chan_for(r, c, 0.9, clamp, "some") if variant == 0 else pow2_chan(r, c)
    args = dict(x=x, n=n, hh=hh, ww=ww, c=c, stride=stride, a_bits=a_bits, w=w, chan=chan, relu=relu, out_bits=out_bits, clamp=clamp,
                out=out_buf(n * ho * wo * c, out_bits))
    (cm,), (g,) = run_both("dwconv3x3", args, ["out"])
    assert torch.equal(cm, g), (n, hh, ww, c, stride, io, variant)


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
    """Wo = 129 (W 257, 258): three 64-column tiles, the last one pixel wide.  x = w = -128 with power-of-two ratios, then random data
    with ReLU6 caps and a low-bit copy."""
    hh, ww = hw
    r = np.random.RandomState(hh + 3 * ww)
    n = 2
    ho, wo = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
    clamp = (-32768, 32767)
    for variant, (relu, y_bits, low) in enumerate([(0, 32, (8, (2 ** 30, 40))), (2, 16, (4, dyadic(0.002))), (1, 32, None)]):
        wt = np.zeros((64, 3, 3, 4), dtype=np.int8)
        if variant == 0:
            x = torch.full((n * hh * ww * 3,), -128, dtype=torch.int8)
            wt[:32, :, :, :3] = -128
            k = r.randint(4, 14, size=64)
            chan = ops.make_chan(r.randint(-2 ** 20, 2 ** 20, size=64), [2 ** 30] * 64, list(30 + k), [2 ** 31 - 1] * 64)
        else:
            x = torch.from_numpy(r.randint(-128, 128, size=n * hh * ww * 3).astype(np.int8))
            wt[:32, :, :, :3] = r.randint(-128, 128, size=(32, 3, 3, 3))
            chan = chan_for(r, 64, 0.9, clamp, "some", bias_span=30000)
        low_bits, lm = (low[0], low[1]) if low else (0, (0, 1))
        low_clamp = (-128, 127) if low_bits == 8 else (0, 15)
        args = dict(x=x, w=torch.from_numpy(wt), chan=chan, relu=relu, clamp=clamp, n=n, hh=hh, ww=ww, y_bits=y_bits,
                    y=out_buf(n * ho * wo * 64, y_bits), low_bits=low_bits, low_me=lm, low_clamp=low_clamp,
                    out_low=out_buf(n * ho * wo * 64, low_bits) if low_bits else None)
        cm, g = run_both("stem3x3", args, ["y", "out_low"] if low_bits else ["y"])
        for a, b in zip(cm, g):
            assert torch.equal(a, b), (hw, variant)
