"""-m gpu: whole quantized ResNets on the CUDA path against the reference-generated goldens (bit-equal logits),
the oracle's full activation tensors, and size-independent properties at the benchmark batch size."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import qtensor
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests.util import RESNET_GOLDENS, build_fakequant, golden_act_ranges, load_net_golden, sha_i32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# every golden at a4_container 8, and packed nibbles too for the schemes with 4-bit activations
A4_CONFIGS = [(a, s, 8) for a, s in RESNET_GOLDENS] + [(a, s, 4) for a, s in RESNET_GOLDENS
                                                       if any(v["bits"] == 4 for v in load_net_golden(a, s)[1]["acts"].values())]
# resize units whose identity input is 4-bit and whose last convolution's input is 8-bit: with packed nibbles the two 1x1 inputs
# have different widths, so the dual kernel is declined there (identity RAW_I32 conv + RESIDUAL conv instead)
MIXED_WIDTH_RESIZE = {("resnet50", "modelsize_0.25"): 1, ("resnet50", "latency_0.25"): 1}


def _model(arch, scheme, meta):
    return hb.build_synthetic_qresnet(arch, scheme, act_ranges=golden_act_ranges(meta))


@pytest.mark.parametrize("arch,scheme", RESNET_GOLDENS)
@pytest.mark.parametrize("res_bits", [32, 16])
def test_eager_module_api_matches_golden(arch, scheme, res_bits):
    """Frozen module-by-module forward (the drop-in API) on fp32 NCHW CUDA input: logits bit-equal to the reference."""
    logits_g, meta = load_net_golden(arch, scheme)
    q = _model(arch, scheme, meta)
    x = synthetic_batch(*meta["input"]).to(DEV)
    qtensor.config.residual_bits = res_bits
    try:
        with torch.no_grad():
            out = q(x)
    finally:
        qtensor.config.residual_bits = 32
    torch.cuda.synchronize()
    assert out.is_cuda and out.dtype == torch.float32
    assert np.array_equal(out.cpu().numpy(), logits_g)


@pytest.mark.parametrize("arch,scheme", RESNET_GOLDENS)
def test_every_activation_matches_oracle(arch, scheme):
    """Mirror of the reference's --debug-unit checks: integer equality at every QuantAct / unit boundary."""
    logits_g, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(*meta["input"])
    fqm = build_fakequant(arch, scheme, meta)
    fqm(x)
    net_i = ir.IntResNet(fqm.harvest())
    li = net_i(x.numpy(), trace=True)
    assert np.array_equal(li, logits_g)
    q = _model(arch, scheme, meta)
    rec = {}
    for name, m in q.named_modules():
        if isinstance(m, (hb.QuantAct, hb.q_resnet.QResidualUnit)):
            m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name, out[0]))
    with torch.no_grad():
        out = q(x.to(DEV))
    torch.cuda.synchronize()
    bad = []
    for name, t in rec.items():
        if not isinstance(t, hb.IntActivation) or t.node.kind != "int":
            continue
        got = t.int_tensor().cpu().numpy()
        got = got.transpose(0, 2, 3, 1) if got.ndim == 4 else got
        want = net_i.trace[name] if name in net_i.trace else np.maximum(net_i.trace[name + ".quant_act_int32"], 0)
        if not np.array_equal(got.reshape(want.shape), want):
            bad.append((name, int((got.reshape(want.shape) != want).sum())))
    assert not bad, bad[:5]
    assert np.array_equal(out.cpu().numpy(), logits_g)


@pytest.mark.parametrize("arch,scheme,a4_container", A4_CONFIGS)
def test_compiled_graph_int8_input_and_batch_invariance(arch, scheme, a4_container, monkeypatch):
    """CUDA-graph engine on int8 NHWC input at a larger batch: the first two images are the golden inputs, so their
    logits must equal the golden logits whatever else is in the batch (size-independent property); replays are idempotent.
    a4_container: 4-bit activations one per byte (default) or as packed nibbles expanded on chip - same logits.
    The uint16 stream runs each bottleneck resize unit as one dual kernel, except where the two inputs differ in width."""
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    logits_g, meta = load_net_golden(arch, scheme)
    q = _model(arch, scheme, meta)
    B = 32
    xg = synthetic_batch(*meta["input"])
    s_in = np.float32(meta["acts"]["quant_input"]["scale"])
    x = torch.cat([xg, synthetic_batch(B - xg.shape[0], 77) * 1.3], dim=0)
    q_in = torch.from_numpy(ir.quantize_input(x.numpy(), s_in).astype(np.int8)).to(DEV)      # NHWC int8
    eng = hb.compile_model(q, q_in)
    out1 = eng(q_in).clone()
    out2 = eng().clone()
    torch.cuda.synchronize()
    assert torch.equal(out1, out2)
    assert np.array_equal(out1[:2].cpu().numpy(), logits_g)
    assert eng.gpu_launches > 0
    # one eager checked forward at residual_bits = 16: one dual kernel per bottleneck resize unit of equal input widths
    duals = 0 if arch == "resnet18" else 4 - (MIXED_WIDTH_RESIZE.get((arch, scheme), 0) if a4_container == 4 else 0)
    n, h, w, c = q_in.shape
    before = hb._lib.load().hawq_debug_kernel_count(4)
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        out_e = q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device))
    torch.cuda.synchronize()
    assert hb._lib.load().hawq_debug_kernel_count(4) - before == duals
    assert torch.equal(out_e, out1)
    # exactness fallback: int32 residual graph gives the same logits
    eng32 = hb.compile_model(q, q_in, residual_bits=32)
    assert torch.equal(eng32(q_in), out1)
    # eager (no graph) agrees
    eng_e = hb.compile_model(q, q_in, use_cuda_graph=False)
    assert torch.equal(eng_e(q_in), out1)


def test_uint16_overflow_falls_back_exactly():
    """Inputs 4x hotter than the calibration batch push residual values past 65535: the uint16 graph raises the flag
    and the engine transparently re-runs with int32 residuals; the result equals the oracle."""
    arch, scheme = "resnet18", "uniform8"
    _, meta = load_net_golden(arch, scheme)
    q = _model(arch, scheme, meta)
    # force a tiny 16-bit range so that overflow certainly happens
    for name, m in q.named_modules():
        if name.endswith("quant_act_int32") and name != "quant_act_int32":
            m.x_min.mul_(0.2)
            m.x_max.mul_(0.2)
    x = synthetic_batch(2, 5)
    fqm = build_fakequant(arch, scheme, meta)
    for name, a in fqm.acts.items():
        if name.endswith("quant_act_int32") and name != "quant_act_int32":
            a.x_min, a.x_max = a.x_min * 0.2, a.x_max * 0.2
    want = fqm(x).numpy()
    eng = hb.compile_model(q, x.to(DEV))
    got = eng(x.to(DEV))
    assert eng.fallbacks == 1
    assert np.array_equal(got.cpu().numpy(), want)


def test_compiled_graph_uint8_pixels_equal_the_torch_pipeline():
    """uint8 NHWC pixels -> fused ToTensor/Normalize/quantise kernel at the head of the graph == the reference's loader pipeline
    (transforms.ToTensor + Normalize, fp32 NCHW) fed to the same frozen model; and weights reloaded in place invalidate the plan."""
    from hawq_b200.engine import IMAGENET_MEAN, IMAGENET_STD
    logits_g, meta = load_net_golden("resnet18", "uniform8")
    q = _model("resnet18", "uniform8", meta)
    g = torch.Generator().manual_seed(5)
    u8 = torch.randint(0, 256, (3, 224, 224, 3), generator=g, dtype=torch.uint8)
    x = u8.permute(0, 3, 1, 2).to(torch.float32).div(255)                               # transforms.ToTensor
    x = x.sub(torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)).div(torch.tensor(IMAGENET_STD).view(1, 3, 1, 1))   # Normalize
    with torch.no_grad():
        want = q(x.to(DEV)).cpu()
    eng = hb.compile_model(q, u8.to(DEV))
    got = eng(u8.to(DEV)).cpu()
    assert torch.equal(got, want)
    # eager plan invalidation on the CUDA path: scaling one conv's float weights in place changes the logits, restoring them
    # restores the logits (load_state_dict writes in place)
    sd = {k: v.clone() for k, v in q.state_dict().items()}
    with torch.no_grad():
        q.stage1.unit1.quant_convbn1.conv.weight.mul_(0.5)
        changed = q(x.to(DEV)).cpu()
        assert not torch.equal(changed, want)
        q.load_state_dict(sd)
        assert torch.equal(q(x.to(DEV)).cpu(), want)


# BASELINE.json configurations 1-4 at the batch sizes that are benchmarked (config 5 = config "resnet50 uniform4" per GPU)
BENCH_CONFIGS = [("resnet18", "uniform8", 8, 8), ("resnet18", "uniform4", 128, 8), ("resnet50", "uniform8", 128, 8),
                 ("resnet50", "bops_0.5", 128, 8), ("resnet50", "uniform4", 128, 8), ("resnet50", "uniform4", 128, 4), ("resnet50", "uniform8", 8, 8)]


@pytest.mark.parametrize("arch,scheme,batch,a4_container", BENCH_CONFIGS)
def test_benchmarked_configuration_matches_oracle_on_every_row(arch, scheme, batch, a4_container, monkeypatch, hw=224):
    """The configuration bench.py times (CUDA graph, fused kernels, uint16 stream) at the benchmarked batch size against the
    oracle (the reference's fake-quant forward restated on the CPU, oracle/fakequant.py): ALL rows of the logits bit-equal, and the
    integers of the residual stream at the end of stage 1 and of the last stage (eager pass with the same kernels) equal too.
    Many row tiles per channel block and full-size pipelines are only reached at this size.  hw: the input size (synthetic_batch)."""
    monkeypatch.setattr(qtensor.config, "a4_container", a4_container)
    _, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(batch, 11, hw)
    fqm = build_fakequant(arch, scheme, meta)
    n_stage = len(fqm.units_per_stage)
    probes = ["stage1.unit%d.quant_act_int32" % fqm.units_per_stage[0], "stage%d.unit%d.quant_act_int32" % (n_stage, fqm.units_per_stage[-1])]
    want_logits = fqm(x, trace=probes).numpy()
    want = {k: np.maximum(v.numpy(), 0) for k, v in fqm.trace.items()}            # the stream is stored after the unit's ReLU
    s_in = np.float32(meta["acts"]["quant_input"]["scale"])
    q_in = torch.from_numpy(ir.quantize_input(x.numpy(), s_in).astype(np.int8)).to(DEV)      # NHWC int8
    q = _model(arch, scheme, meta)
    eng = hb.compile_model(q, q_in)
    got = eng(q_in).cpu().numpy()
    assert eng.fallbacks == 0
    assert got.shape == want_logits.shape and np.array_equal(got, want_logits), \
        "rows differing from the oracle: %s" % np.nonzero((got != want_logits).any(axis=1))[0][:16].tolist()
    # residual-stream integers, eager pass through the same kernels
    rec = {}
    for name, m in q.named_modules():
        if isinstance(m, hb.q_resnet.QResidualUnit) and (name + ".quant_act_int32") in want:
            m.register_forward_hook(lambda mod, inp, out, name=name: rec.__setitem__(name + ".quant_act_int32", out[0]))
    n, h, w, c = q_in.shape
    hb.ops.reset_status(0)
    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
        q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in.view(-1), bits=8, signed=True), q_in.device))
    torch.cuda.synchronize()
    assert hb.ops.get_status(0) & 7 == 0
    assert set(rec) == set(want)
    for name, t in rec.items():
        g = t.int_tensor().cpu().numpy()
        assert np.array_equal(g, want[name]), (name, int((g != want[name]).sum()))
