"""-m gpu: the engine at input sizes other than 224 x 224.  The networks take any input whose last feature map is 7 x 7 (193 to 224
pixels per side, square or not); the engine plans every launch from the input's shape.  At 193 every map is odd (97, 49, 25, 13, 7),
and H != W gives unequal maps everywhere, so these sizes reach resize units with odd-height identity inputs, strided convolutions and
bottleneck tails on odd maps, and the stem, depthwise and input kernels at shapes no 224 input produces.

The kernels run against the ABI model in guarded, poisoned buffers (run_both); the networks against the reference-generated goldens
tests/golden/size_*.npz (tests/test_input_sizes_cpu.py pins the oracle and the host engine to them) and the in-repo oracle."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import _lib, ops, qtensor
from hawq_b200._lib import EPI_RESIDUAL, dyadic
from hawq_b200.synthetic import synthetic_batch
from tests.engine_harness import (MIXED_WIDTH_RESIZE, SIZE_GOLDENS, check_benchmarked_configuration_matches_oracle_on_every_row,
                                  check_engine_against_golden, check_every_row, engine_outputs, golden_model, int8_input,
                                  load_size_golden, oracle_for)
from tests.kernel_harness import (DEV, IO, check_conv1x1_requant_and_residual, check_conv_raw_and_dequant_geoms, check_conv_requant,
                                  check_conv_residual, check_stem3x3_non_square, check_stem_and_pool, dw_rect, images_for_three_tiles,
                                  make_chan, out_buf, rand_act, run_both)
from tests.util import golden_act_ranges, load_net_golden

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ resize units, odd identity inputs
# ResNet-50 resize units with a stride-2 identity: stage -> (Cin = bottleneck width, Cin2 = unit input channels, Cout)
R50_RESIZE = {2: (128, 256, 512), 3: (256, 512, 1024), 4: (512, 1024, 2048)}
# (stage, Ho, Wo, H2, W2): the identity input H2 x W2 of the networks at 193 x 193, 193 x 224 and 200 x 216
DUAL_ODD = [(3, 13, 13, 25, 25),     # odd H2, odd W2
            (4, 7, 7, 13, 13),
            (2, 25, 28, 49, 56),     # odd H2, even W2
            (3, 13, 14, 25, 27),
            (4, 7, 7, 13, 14),       # odd H2, even W2
            (2, 25, 25, 50, 49)]     # even H2, odd W2: W2 < H2


@pytest.mark.parametrize("flag", [1, 2])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("case", DUAL_ODD)
def test_conv_dual_odd_identity_inputs(case, a_bits, flag):
    """hawq_conv2d_dual on identity inputs of odd height or width (H2 = 2 Ho - 1 or W2 = 2 Wo - 1): bit-exact vs the ABI model's
    RAW_I32 identity conv + res_kind-1 RESIDUAL conv, and the dual kernel (hawq_debug_kernel_count family 4) takes every launch."""
    stage, ho, wo, h2, w2 = case
    cin, cin2, cout = R50_RESIZE[stage]
    assert (h2 - 1) // 2 + 1 == ho and (w2 - 1) // 2 + 1 == wo and (h2 % 2 or w2 % 2)
    n = images_for_three_tiles(ho * wo, cout)
    r = np.random.RandomState(4001 + sum(v * (i + 3) for i, v in enumerate(case)) * 4 + a_bits + flag)
    numel = n * ho * wo * cout
    x = rand_act(r, n * ho * wo * cin, a_bits)
    x2 = rand_act(r, n * h2 * w2 * cin2, a_bits)
    wt = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8))
    wt2 = torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin2)).astype(np.int8))
    if a_bits == 4:
        ops.permute_weights_for_i4(wt)
        ops.permute_weights_for_i4(wt2)
    hi = 0.9 if flag == 1 else 30.0
    chan = make_chan(r, cout, bias_mag=3000, ratio_lo=1e-2, ratio_hi=hi)
    chan2 = make_chan(r, cout, bias_mag=3000, ratio_lo=1e-2, ratio_hi=hi)
    d = ops.conv_desc(n, ho, wo, cin, cout, 1, 1, 1, 0, a_bits, 1)
    d2 = ops.conv_desc(n, h2, w2, cin2, cout, 1, 1, 2, 0, a_bits, 1)
    wg, wg2 = ops.upload_weights(wt, DEV), ops.upload_weights(wt2, DEV)
    for low_bits in (8, 4, 0):
        ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, low_bits=low_bits, low_me=dyadic(0.003),
                          low_clamp=(0, 15) if low_bits == 4 else (-128, 127), flags=flag)
        args = dict(x=x, desc=d, ep=ep, w=wt, chan=chan, desc2=d2, x2=x2, w2=wt2, chan2=chan2, out=out_buf(numel, 16),
                    out_low=out_buf(numel, low_bits) if low_bits else None)
        keys = ["out"] + (["out_low"] if low_bits else [])
        before = _lib.load().hawq_debug_kernel_count(4)
        cs, gs = run_both("conv2d_dual", args, keys, gpu_overrides=dict(w=wg, w2=wg2))
        assert _lib.load().hawq_debug_kernel_count(4) == before + 1, "conv_dual did not take this launch"
        for a, b, k_ in zip(cs, gs, keys):
            assert torch.equal(a, b), (case, a_bits, flag, low_bits, k_)


# ------------------------------------------------------------------------------------------------ conv_igemm on odd and unequal maps
@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(9, 25, 28, 512, 256, 1, 1, 2, 0),     # ResNet-50 stage-3 conv1 at 193 x 224: 13 x 14 out
                                  (7, 25, 27, 128, 256, 3, 3, 2, 1),     # ResNet-18 stage-3 conv1 at 200 x 216
                                  (5, 49, 49, 256, 128, 1, 1, 2, 0)])    # ResNet-50 stage-2 conv1 at 193 x 193
def test_strided_conv_requant_odd_maps(geom, a_bits, tc):
    check_conv_requant(geom, a_bits, tc)


@pytest.mark.parametrize("a_bits", [8, 4])
def test_resnet18_strided_identity_raw(a_bits):
    """ResNet-18's 1x1/2 identity convolution (RAW_I32) from 25 x 27"""
    check_conv_raw_and_dequant_geoms((7, 25, 27, 128, 256, 1, 1, 2, 0), a_bits)


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("geom", [(7, 13, 14, 256, 256, 3, 3, 1, 1),     # ResNet-18 stage-3 conv2 + identity (res_kind 0 and 1)
                                  (None, 13, 13, 256, 1024, 1, 1, 1, 0),  # ResNet-50 bottleneck tails at 193 and 193 x 224
                                  (None, 25, 28, 128, 512, 1, 1, 1, 0)])
def test_residual_odd_maps(geom, a_bits, tc):
    """RESIDUAL epilogues on odd maps; a batch of None gives every CTA of the tail kernel at least three row tiles"""
    n, h, w, cin, cout = geom[:5]
    check_conv_residual((n or images_for_three_tiles(h * w, cout),) + geom[1:], a_bits, tc)


@pytest.mark.parametrize("a_bits", [8, 4])
@pytest.mark.parametrize("hw", [(13, 13), (25, 28)])
def test_bottleneck_tail_odd_maps(hw, a_bits):
    h, w = hw
    mid, cout = (256, 1024) if h == 13 else (128, 512)
    check_conv1x1_requant_and_residual((images_for_three_tiles(h * w, cout), h, w, mid, cout), a_bits)


@pytest.mark.parametrize("shape", [(2, 193, 224), (1, 224, 193), (2, 200, 216), (3, 193, 193)])
def test_resnet_stem_odd_maps(shape):
    """stem_conv then maxpool_requant: 97 x 112 -> 49 x 56, 112 x 97 -> 56 x 49, 100 x 108 -> 50 x 54, 97 x 97 -> 49 x 49"""
    check_stem_and_pool(shape)


@pytest.mark.parametrize("hw", [(193, 193), (193, 224), (224, 193)])
def test_mobilenet_stem_odd_maps(hw):
    check_stem3x3_non_square(hw)


# MobileNetV2's stride-2 depthwise convolutions at 193 x 224: (stored channels, input H, W)
DW_ODD = [(128, 97, 112), (192, 49, 56), (192, 25, 28), (576, 13, 14), (128, 97, 97), (576, 13, 13), (192, 56, 49)]


@pytest.mark.parametrize("geom", DW_ODD)
def test_dwconv_stride2_odd_maps(geom):
    c, hh, ww = geom
    r = np.random.RandomState(c + 7 * hh + 11 * ww)
    for i, io in enumerate(IO):
        dw_rect(r, 3, hh, ww, c, 2, io, i % 3)


# ------------------------------------------------------------------------------------------------ networks against the size goldens

def int_activation(q_in):
    n, h, w, c = q_in.shape
    return hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device)


def golden_rows(meta, logits_g, net, xg):
    """what the compiled graph must give on the golden images: the golden logits (ResNet), the integer restatement (MobileNetV2)"""
    if meta["arch"] != "mobilenetv2_w1":
        return logits_g
    want = net(xg.numpy())
    assert np.allclose(want, logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(want.argmax(1), logits_g.argmax(1))
    return want


@pytest.mark.parametrize("name", SIZE_GOLDENS)
def test_eager_module_api_matches_size_golden(name):
    """Frozen module-by-module forward on fp32 NCHW CUDA input at residual_bits 32 and 16: every concrete QuantAct's integers hash to
    the reference's, every residual-unit output equals the oracle's stream, ResNet logits bit-equal to the reference."""
    logits_g, meta, x = load_size_golden(name)
    _, _, net = oracle_for(meta, x)
    q = golden_model(meta["arch"], meta["scheme"], meta)
    for res_bits in (32, 16):
        qtensor.config.residual_bits = res_bits
        try:
            y, acts, units = engine_outputs(q, x.to(DEV))
            torch.cuda.synchronize()
        finally:
            qtensor.config.residual_bits = 32
        assert y.is_cuda and y.dtype == torch.float32
        check_engine_against_golden(y, acts, units, meta, logits_g, net, x)


def size_a4_configs():
    out = []
    for name in SIZE_GOLDENS:
        meta = load_size_golden(name)[1]
        out += [(name, 8)] + ([(name, 4)] if any(v["bits"] == 4 for v in meta["acts"].values()) else [])
    return out


@pytest.mark.parametrize("name,a4_container", size_a4_configs())
def test_compiled_graph_matches_size_golden(name, a4_container, monkeypatch):
    """CUDA-graph engine on int8 NHWC input, batch 32 whose first two images are the golden ones: those rows equal the golden, a
    replay is idempotent, the int32-residual engine and the engine without a graph agree.  A checked eager pass at residual_bits 16
    runs every ResNet-50 resize unit as one dual kernel, except the mixed-width one under packed nibbles."""
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    logits_g, meta, xg = load_size_golden(name)
    arch, scheme = meta["arch"], meta["scheme"]
    _, _, net = oracle_for(meta, xg)
    want = golden_rows(meta, logits_g, net, xg)
    q = golden_model(meta["arch"], meta["scheme"], meta)
    B = 32
    x = torch.cat([xg, synthetic_batch(B - xg.shape[0], 77, tuple(xg.shape[2:])) * 1.3], dim=0)
    q_in = int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV)
    eng = hb.compile_model(q, q_in)
    out1 = eng(q_in).clone()
    out2 = eng().clone()
    torch.cuda.synchronize()
    assert eng.fallbacks == 0
    assert torch.equal(out1, out2)
    assert np.array_equal(out1[:2].cpu().numpy(), want)
    lib = _lib.load()
    counts = lambda: [lib.hawq_debug_kernel_count(f) for f in (1, 2, 4)]
    before = counts()
    hb.ops.reset_status(0)
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        out_e = q(int_activation(q_in))
    torch.cuda.synchronize()
    after = counts()
    assert hb.ops.get_status(0) & 7 == 0
    if arch == "resnet50":
        assert after[2] - before[2] == 4 - (MIXED_WIDTH_RESIZE.get((arch, scheme), 0) if a4_container == 4 else 0)
    elif arch == "resnet18":
        assert after[2] == before[2]
    else:                                                       # 17 depthwise launches, one 3x3 stem (as at 224)
        assert (after[0] - before[0], after[1] - before[1]) == (17, 1)
    assert torch.equal(out_e, out1)
    eng32 = hb.compile_model(q, q_in, residual_bits=32)
    assert torch.equal(eng32(q_in), out1)
    eng_e = hb.compile_model(q, q_in, use_cuda_graph=False)
    assert torch.equal(eng_e(q_in), out1)


def test_compiled_graph_uint8_pixels_with_a_tail_byte():
    """3 x 193 x 193 x 3 = 335 241 uint8 bytes, not a multiple of 4: the fused ToTensor/Normalize/quantise kernel at the head of the
    graph ends on a partial word and must still equal the torch pipeline fed to the eager model."""
    from hawq_b200.engine import IMAGENET_MEAN, IMAGENET_STD
    _, meta, _ = load_size_golden("size_resnet18_uniform8_193x193.npz")
    q = golden_model(meta["arch"], meta["scheme"], meta)
    u8 = torch.randint(0, 256, (3, 193, 193, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    assert u8.numel() % 4 == 1
    x = u8.permute(0, 3, 1, 2).to(torch.float32).div(255)
    x = x.sub(torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)).div(torch.tensor(IMAGENET_STD).view(1, 3, 1, 1))
    with torch.no_grad():
        want = q(x.to(DEV)).cpu()
    eng = hb.compile_model(q, u8.to(DEV))
    got = eng(u8.to(DEV)).cpu()
    assert torch.equal(got, want)
    assert torch.equal(eng().cpu(), want)


# ------------------------------------------------------------------------------------------------ benchmarked batch at another size
@pytest.mark.parametrize("a4_container", [8, 4])
def test_resnet50_benchmarked_batch_193x224(a4_container, monkeypatch):
    """every logits row and the stage-end residual streams of 128 images at 193 x 224 against the CPU oracle"""
    check_benchmarked_configuration_matches_oracle_on_every_row("resnet50", "uniform4", 128, a4_container, monkeypatch, hw=(193, 224))


def test_mobilenetv2_benchmarked_batch_224x193(monkeypatch):
    """every logits row and every QuantAct of 128 images at 224 x 193 against the exact integer restatement"""
    _, meta, xg = load_size_golden("size_mobilenetv2_w1_uniform4_193x224.npz")
    _, _, net = oracle_for(meta, xg)
    check_every_row(golden_model(meta["arch"], meta["scheme"], meta), net, 128, (8, 4), monkeypatch, hw=(224, 193))


# ------------------------------------------------------------------------------------------------ one model, several sizes
def test_one_model_several_input_sizes():
    """Eager forwards at 224, 193 x 224, then 224 again on one frozen model each equal their golden, and compiled engines for both
    sizes built from that model give their goldens on interleaved replays: nothing planned or allocated for one input shape is
    reused for another."""
    logits_224, meta_224 = load_net_golden("resnet50", "uniform4")
    logits_s, meta_s, x_s = load_size_golden("size_resnet50_uniform4_193x224.npz")
    assert golden_act_ranges(meta_224) == golden_act_ranges(meta_s)
    x_224 = synthetic_batch(*meta_224["input"])
    q = golden_model(meta_224["arch"], meta_224["scheme"], meta_224)
    with torch.no_grad():
        for x, want in [(x_224, logits_224), (x_s, logits_s), (x_224, logits_224)]:
            assert np.array_equal(q(x.to(DEV)).cpu().numpy(), want), tuple(x.shape)
    engines = []
    for x, want in [(x_224, logits_224), (x_s, logits_s)]:
        xb = torch.cat([x, synthetic_batch(6, 78, tuple(x.shape[2:]))], dim=0)
        q_in = int8_input(xb, meta_224["acts"]["quant_input"]["scale"]).to(DEV)
        eng = hb.compile_model(q, q_in)
        engines.append((eng, q_in, want))
    for _ in range(2):
        for eng, q_in, want in engines:
            assert np.array_equal(eng(q_in)[:2].cpu().numpy(), want)
        for eng, q_in, want in engines:
            assert np.array_equal(eng()[:2].cpu().numpy(), want)
    with torch.no_grad():
        assert np.array_equal(q(x_s.to(DEV)).cpu().numpy(), logits_s)
