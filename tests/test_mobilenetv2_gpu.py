"""-m gpu: the MobileNetV2 kernels against the ABI model (guarded, pre-poisoned buffers through run_both), REQUANT with ReLU6 caps
on the convolution kernel, and the whole frozen network (eager and compiled) against the reference-generated goldens and the
exact integer restatement."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200._lib import EPI_REQUANT, dyadic
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests.engine_harness import SCHEMES, int_oracle, nhwc, run_engine
from tests.kernel_harness import DEV, IO, act_in, chan_for, out_buf, rand_act, run_both
from tests.util import golden_act_ranges, load_net_golden, sha_i32

pytestmark = pytest.mark.gpu


# every depthwise geometry of MobileNetV2-1.0 at 224 x 224: (stored C, input H = W, stride)
DW_GEOMS = [(64, 112, 1), (128, 112, 2), (192, 56, 1), (192, 56, 2), (192, 28, 1), (384, 28, 2), (384, 14, 1), (576, 14, 1),
            (576, 14, 2), (960, 7, 1)]


def dw_case(r, n, h, c, stride, io, ratio_hi=0.9, caps="some", relu=2, saturate=False, clamp=None):
    a_bits, kind, out_bits, oclamp = io
    clamp = clamp or oclamp
    ho = (h - 1) // stride + 1
    x = act_in(r, n * h * h * c, kind, a_bits)
    w = torch.from_numpy(r.randint(-128, 128, size=(3, 3, c)).astype(np.int8))
    chan = chan_for(r, c, ratio_hi, clamp, caps, saturate=saturate)
    args = dict(x=x, n=n, hh=h, ww=h, c=c, stride=stride, a_bits=a_bits, w=w, chan=chan, relu=relu, out_bits=out_bits, clamp=clamp,
                out=out_buf(n * ho * ho * c, out_bits))
    (cm,), (g,) = run_both("dwconv3x3", args, ["out"])
    assert torch.equal(cm, g), (n, h, c, stride, io, ratio_hi, caps, relu)


@pytest.mark.parametrize("geom", DW_GEOMS)
def test_dwconv_every_mobilenetv2_geometry(geom):
    c, h, s = geom
    r = np.random.RandomState(c * 7 + h + s)
    for i, io in enumerate(IO):
        dw_case(r, 2 if h >= 56 else 3, h, c, s, io, ratio_hi=0.9 if i % 2 == 0 else 40.0, caps="some" if i % 3 else "none")


@pytest.mark.parametrize("io", IO)
@pytest.mark.parametrize("ratio_hi", [0.9, 3000.0])
def test_dwconv_ratios_caps_and_saturation(io, ratio_hi):
    r = np.random.RandomState(int(ratio_hi) + io[0] + io[2])
    for caps, relu, saturate in [("some", 2, False), ("none", 2, True), ("some", 1, False), ("none", 0, True)]:
        dw_case(r, 2, 19, 48, 1 + (relu % 2), io, ratio_hi, caps, relu, saturate)
    lo = io[3][0] if io[3][0] >= 0 else -3
    dw_case(r, 2, 9, 32, 2, io, ratio_hi, "some", 2, clamp=(lo, lo))          # lo = hi


def test_dwconv_more_ctas_than_two_waves_ragged():
    """30 x 56 x 56 x 192: 11 760 column strips -> 46 CTAs per channel group (the last one ragged) x 12 groups, over two waves."""
    r = np.random.RandomState(5)
    for io in (IO[0], IO[2]):
        dw_case(r, 30, 56, 192, 1, io)


@pytest.mark.parametrize("w", [224, 97, 5])
def test_stem3x3(w):
    r = np.random.RandomState(w)
    n = 2 if w == 224 else 3
    h = w if w != 5 else 7
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = torch.from_numpy(r.randint(-128, 128, size=n * h * w * 3).astype(np.int8))
    wt = np.zeros((64, 3, 3, 4), dtype=np.int8)
    wt[:32, :, :, :3] = r.randint(-128, 128, size=(32, 3, 3, 3))
    for ratio_hi, caps, relu, y_bits, low in [(0.9, "some", 2, 16, (8, 0.01)), (0.9, "none", 2, 32, None), (40.0, "some", 2, 16, (4, 0.002)),
                                              (0.9, "some", 1, 32, (8, 3.0)), (5.0, "none", 0, 32, None)]:
        clamp = (-32768, 32767)
        chan = chan_for(r, 64, ratio_hi, clamp, caps, bias_span=30000, saturate=relu == 0)
        low_bits, lm = (low[0], dyadic(low[1])) if low else (0, (0, 1))
        low_clamp = (-128, 127) if low_bits == 8 else (0, 15)
        args = dict(x=x, w=torch.from_numpy(wt), chan=chan, relu=relu, clamp=clamp, n=n, hh=h, ww=w, y_bits=y_bits,
                    y=out_buf(n * ho * wo * 64, y_bits), low_bits=low_bits, low_me=lm, low_clamp=low_clamp,
                    out_low=out_buf(n * ho * wo * 64, low_bits) if low_bits else None)
        cm, g = run_both("stem3x3", args, ["y", "out_low"] if low_bits else ["y"])
        for a, b in zip(cm, g):
            assert torch.equal(a, b), (w, ratio_hi, caps, relu, y_bits, low)


@pytest.mark.parametrize("geom", [(2, 8, 8, 64, 128, 1, 1, 1, 0), (3, 7, 7, 64, 192, 3, 3, 1, 1), (2, 9, 9, 128, 64, 1, 1, 2, 0)])
@pytest.mark.parametrize("a_bits", [8, 4])
def test_conv_requant_relu6_caps(geom, a_bits):
    """REQUANT with relu 2 on the convolution kernel: BN 128 (Cout 128) and 64 (Cout 64 / 192), all output widths, caps on some
    channels; relu 1 on the same channels must ignore the caps."""
    n, h, w, cin, cout, kh, kw, s, p = geom
    r = np.random.RandomState(sum(geom) + a_bits)
    ho, wo = (h + 2 * p - kh) // s + 1, (w + 2 * p - kw) // s + 1
    x = rand_act(r, n * h * w * cin, a_bits)
    wt = torch.from_numpy(r.randint(-128, 128, size=(cout, kh, kw, cin)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
    d = ops.conv_desc(n, h, w, cin, cout, kh, kw, s, p, a_bits)
    for out_bits, clamp in [(8, (-128, 127)), (4, (0, 15)), (16, (-32768, 32767)), (32, (-2 ** 31, 2 ** 31 - 1))]:
        chan = chan_for(r, cout, 1e-2 if out_bits <= 8 else 0.9, clamp if out_bits <= 16 else (0, 100000), "some")
        for relu in (2, 1):
            ep = ops.epilogue(EPI_REQUANT, relu=relu, out_bits=out_bits, clamp=clamp, flags=1)
            (cm,), (g,) = run_both("conv2d", dict(x=x, desc=d, ep=ep, w=wt, chan=chan, out=out_buf(n * ho * wo * cout, out_bits)), ["out"])
            assert torch.equal(cm, g), (geom, a_bits, out_bits, relu)


@pytest.mark.parametrize("a4_container", [8, 4])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_network_eager_and_compiled(scheme, a4_container, monkeypatch):
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    logits_g, meta = load_net_golden("mobilenetv2_w1", scheme)
    xg = synthetic_batch(*meta["input"])
    _, _, net = int_oracle(scheme, golden_act_ranges(meta), xg)
    want = net(xg.numpy(), trace=True)
    q = hb.build_synthetic_qresnet("mobilenetv2_w1", scheme, act_ranges=golden_act_ranges(meta))
    # eager frozen forward on CUDA: every QuantAct tensor, the logits
    y, rec = run_engine(q, xg.to(DEV))
    assert set(rec) == set(meta["acts"])
    for name, t in rec.items():
        got = nhwc(t.int_tensor().cpu().numpy())
        assert sha_i32(got) == meta["acts"][name]["sha"], name
        assert np.array_equal(got.reshape(net.trace[name].shape), net.trace[name]), name
    assert np.array_equal(y.cpu().numpy(), want)
    assert np.allclose(want, logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(want.argmax(1), logits_g.argmax(1))
    # compiled graph, batch 128 whose first two images are the golden inputs
    B = 128
    x = torch.cat([xg, synthetic_batch(B - xg.shape[0], 77) * 1.3], dim=0)
    s_in = np.float32(meta["acts"]["quant_input"]["scale"])
    q_in = torch.from_numpy(ir.quantize_input(x.numpy(), s_in).astype(np.int8)).to(DEV)
    lib = hb._lib.load()
    eng = hb.compile_model(q, q_in)
    before = (lib.hawq_debug_kernel_count(1), lib.hawq_debug_kernel_count(2))
    out1 = eng(q_in).clone()
    after = (lib.hawq_debug_kernel_count(1), lib.hawq_debug_kernel_count(2))
    out2 = eng().clone()
    torch.cuda.synchronize()
    assert torch.equal(out1, out2)
    assert np.array_equal(out1[:2].cpu().numpy(), want)
    assert after == before                                  # a graph replay does not go through the launchers
    n0 = (lib.hawq_debug_kernel_count(1), lib.hawq_debug_kernel_count(2))
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        n, h, w, c = q_in.shape
        out_e = q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device))
    torch.cuda.synchronize()
    assert (lib.hawq_debug_kernel_count(1) - n0[0], lib.hawq_debug_kernel_count(2) - n0[1]) == (17, 1)
    assert torch.equal(out_e, out1)
    # fp32 and uint8 inputs, the pipelined call
    eng_f = hb.compile_model(q, x.to(DEV))
    assert torch.equal(eng_f(x.to(DEV)), out1)
    u8 = torch.randint(0, 256, (8, 224, 224, 3), generator=torch.Generator().manual_seed(3), dtype=torch.uint8)
    eng_u = hb.compile_model(q, u8.to(DEV))
    from hawq_b200.engine import IMAGENET_MEAN, IMAGENET_STD
    xf = u8.permute(0, 3, 1, 2).to(torch.float32).div(255)
    xf = xf.sub(torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)).div(torch.tensor(IMAGENET_STD).view(1, 3, 1, 1))
    with torch.no_grad():
        assert torch.equal(eng_u(u8.to(DEV)), q(xf.to(DEV)))
    batches = [q_in.cpu().pin_memory(), torch.flip(q_in, [0]).cpu().pin_memory()]
    outs = [o.clone() for o in eng.run_pipelined(batches)]
    assert torch.equal(outs[0], out1.cpu()) and torch.equal(outs[1], eng(batches[1].to(DEV)).cpu())
