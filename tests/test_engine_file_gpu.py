"""-m gpu: plan files end to end.  A CompiledModel is saved (CompiledModel.save) and loaded by the library's runtime
(hawq_b200.load_engine); the loaded engine's logits are byte-equal to the CompiledModel's and to the golden logits, on every input
route, at the golden batch and at batch 128, after the model is gone, through the int32 and saturating fallbacks, from the standalone
C runner, and next to other engines replaying on other streams."""
import gc
import os
import subprocess

import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import qtensor
from hawq_b200.build import RUNNER
from hawq_b200.synthetic import synthetic_batch
from oracle import int_ref as ir
from tests.engine_harness import _eager, _oracle, golden_model, int8_input
from tests.kernel_harness import DEV
from tests.util import golden_act_ranges, load_net_golden

pytestmark = pytest.mark.gpu

CONFIGS = [("resnet18", "uniform4", 8), ("resnet18", "uniform4", 4), ("resnet50", "uniform8", 8), ("resnet50", "bops_0.5", 8),
           ("resnet101", "uniform8", 8), ("mobilenetv2_w1", "uniform8", 8), ("mobilenetv2_w1", "uniform4", 8)]


def model(arch, scheme, meta):
    return hb.build_synthetic_qresnet(arch, scheme, act_ranges=golden_act_ranges(meta))


def saved(eng, tmp_path, name="plan.hawq"):
    path = str(tmp_path / name)
    assert eng.save(path) == os.path.getsize(path)
    return hb.load_engine(path)


def assert_launches(loaded, eng):
    assert loaded.launches["fast"] == eng.launches[eng.residual_bits] == loaded.gpu_launches
    assert loaded.launches["int32"] == (eng.launches[32] if eng.residual_bits == 16 else 0)
    assert loaded.launches["safe"] == eng.launches["safe"]


def assert_golden(y, logits_g, arch):
    """ResNets: the golden logits bit for bit; MobileNetV2 (fp32 classifier sums): as tests/engine_harness.assert_mobilenet_logits"""
    if arch == "mobilenetv2_w1":
        assert np.allclose(y, logits_g, rtol=2e-6, atol=2e-7) and np.array_equal(y.argmax(1), logits_g.argmax(1))
    else:
        assert np.array_equal(y, logits_g)


@pytest.mark.parametrize("arch,scheme,a4", CONFIGS)
def test_loaded_engine_equals_the_compiled_model(arch, scheme, a4, tmp_path, monkeypatch):
    monkeypatch.setattr(qtensor.config, "a4_container", a4)
    logits_g, meta = load_net_golden(arch, scheme)
    q = model(arch, scheme, meta)
    x = synthetic_batch(*meta["input"])
    s_in = np.float32(meta["acts"]["quant_input"]["scale"])
    g = torch.Generator().manual_seed(5)
    routes = {"int8": int8_input(x, s_in).to(DEV), "fp32": x.to(DEV),
              "uint8": torch.randint(0, 256, (2, 224, 224, 3), generator=g, dtype=torch.uint8).to(DEV)}
    for route, xin in routes.items():
        eng = hb.compile_model(q, xin)
        want = eng(xin).cpu().numpy()
        loaded = saved(eng, tmp_path, route + ".hawq")
        got = loaded(xin).cpu().numpy()
        assert np.array_equal(got, want), route
        assert loaded.fallbacks == eng.fallbacks
        assert_launches(loaded, eng)
        if route != "uint8":
            assert_golden(got, logits_g, arch)
        del loaded, eng
    big = int8_input(synthetic_batch(128, 11), s_in).to(DEV)
    eng = hb.compile_model(q, big)
    want = eng(big).cpu().numpy()
    loaded = saved(eng, tmp_path, "b128.hawq")
    assert np.array_equal(loaded(big).cpu().numpy(), want)
    assert_launches(loaded, eng)


def test_loaded_engine_outlives_the_model(tmp_path):
    """The file is all the loaded engine needs: the model, its plan caches and the CompiledModel are gone before it is loaded."""
    logits_g, meta = load_net_golden("resnet18", "uniform4")
    x = synthetic_batch(*meta["input"])
    xin = int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV)
    q = model("resnet18", "uniform4", meta)
    eng = hb.compile_model(q, xin)
    path = str(tmp_path / "plan.hawq")
    eng.save(path)
    del q, eng
    gc.collect()
    torch.cuda.empty_cache()
    fqm = _oracle("resnet18", "uniform4", meta)
    fqm(x)
    want = ir.IntResNet(fqm.harvest())(x.numpy())
    loaded = hb.load_engine(path)
    got = loaded(xin.clone()).cpu().numpy()
    assert np.array_equal(got, want) and np.array_equal(got, logits_g)


def test_int32_fallback_is_taken_once_and_exact(tmp_path):
    """stage2.unit2's 16-bit range shrunk to 0.75 (tests/test_engine_paths_gpu.py): a batch at the int8 extremes overflows the uint16
    stream, hawq_engine_run replays the int32 sequence once, and the logits equal the oracle's; a clean batch takes no fallback."""
    arch, scheme, shrink = "resnet18", "bops_0.25", ("stage2.unit2.quant_act_int32", 0.75)
    _, meta = load_net_golden(arch, scheme)
    q = golden_model(arch, scheme, meta, shrink)
    fqm = _oracle(arch, scheme, meta, shrink)
    xs = [synthetic_batch(8, 100), synthetic_batch(8, 104) * 1000.0]
    devs = [int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV) for x in xs]
    assert [_eager(q, x, residual_bits=16, checked=True)[1] for x in devs] == [0, 1]
    loaded = saved(hb.compile_model(q, devs[0]), tmp_path)
    assert np.array_equal(loaded(devs[0]).cpu().numpy(), fqm(xs[0]).numpy()) and loaded.fallbacks == 0
    assert np.array_equal(loaded(devs[1]).cpu().numpy(), fqm(xs[1]).numpy()) and loaded.fallbacks == 1


def test_requant_overflow_replays_the_safe_sequence(tmp_path):
    """The 2^19 shrink of tests/test_engine_paths_gpu.py: HAWQ_FLAG_REQUANT_OVERFLOW, the safe sequence replayed once, logits equal to
    the eager forward with an int32 stream and no ratio promises."""
    arch, scheme, p = "resnet18", "uniform8", "stage2.unit2"
    _, meta = load_net_golden(arch, scheme)
    x = synthetic_batch(2, 5)
    fqm = _oracle(arch, scheme, meta)
    fqm(x)
    h = fqm.harvest()
    a, w_sf = h["acts"], h["convs"][p + ".quant_convbn2"]["w_sf"].numpy()
    z = a[p + ".quant_act_int32"]["scale"].numpy()
    r0 = max(float(ir.requant_ratio(a[p + ".quant_act1"]["scale"].numpy(), w_sf, z).max()),
             float(ir.requant_ratio(a["stage2.unit1.quant_act_int32"]["scale"].numpy(), np.float32(1.0), z).max()))
    q = golden_model(arch, scheme, meta, (p + ".quant_act_int32", r0 / 2.0 ** 19))
    q_in = int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV)
    assert _eager(q, q_in, residual_bits=16, checked=True)[1] & 4
    loaded = saved(hb.compile_model(q, q_in), tmp_path)
    got = loaded(q_in).clone()
    assert loaded.fallbacks == 1
    want, _ = _eager(q, q_in, residual_bits=32, fast_kernels=False)
    assert torch.equal(got, want)


def test_standalone_runner_writes_the_same_logits(tmp_path):
    """tools/hawq_run.c, run without Python on its path, on a saved ResNet-18 plan and two raw int8 batches"""
    logits_g, meta = load_net_golden("resnet18", "uniform4")
    s_in = meta["acts"]["quant_input"]["scale"]
    xs = [int8_input(synthetic_batch(*meta["input"]), s_in), int8_input(synthetic_batch(2, 21), s_in)]
    eng = hb.compile_model(model("resnet18", "uniform4", meta), xs[0].to(DEV))
    loaded = saved(eng, tmp_path)
    want = np.concatenate([loaded(x.to(DEV)).cpu().numpy() for x in xs])
    assert os.path.isfile(RUNNER), "hawq_run is built by build() (hawq_b200.build.build_runner)"
    (tmp_path / "in.raw").write_bytes(b"".join(x.numpy().tobytes() for x in xs))
    env = {k: v for k, v in os.environ.items() if k not in ("PYTHONPATH", "PYTHONHOME")}
    r = subprocess.run([RUNNER, str(tmp_path / "plan.hawq"), str(tmp_path / "in.raw"), "2", str(tmp_path / "out.raw")], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.frombuffer((tmp_path / "out.raw").read_bytes(), dtype=np.float32).reshape(want.shape)
    assert np.array_equal(got, want) and np.array_equal(got[:2], logits_g)


def test_loaded_engines_keep_their_own_status_words(tmp_path):
    """Two loaded engines of one plan and the CompiledModel it came from replay at once on three streams; only the engine given the
    overflowing batch sees HAWQ_FLAG_RESIDUAL_OVERFLOW, and only it falls back."""
    arch, scheme, shrink = "resnet18", "bops_0.25", ("stage2.unit2.quant_act_int32", 0.75)
    _, meta = load_net_golden(arch, scheme)
    q = golden_model(arch, scheme, meta, shrink)
    fqm = _oracle(arch, scheme, meta, shrink)
    xs = [synthetic_batch(8, 101), synthetic_batch(8, 104) * 1000.0, synthetic_batch(8, 102)]
    devs = [int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV) for x in xs]
    eng = hb.compile_model(q, devs[0])
    path = str(tmp_path / "plan.hawq")
    eng.save(path)
    a, b = hb.load_engine(path), hb.load_engine(path)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(3)]
    for _ in range(3):
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(streams[0]):
            b.run_async(devs[0])
        with torch.cuda.stream(streams[1]):
            a.run_async(devs[1])
        with torch.cuda.stream(streams[2]):
            eng.run_async(devs[2])
        torch.cuda.synchronize()
        assert a.status() & 1 and b.status() == 0 and int(eng.flag.item()) == 0
        assert np.array_equal(b.out.cpu().numpy(), fqm(xs[0]).numpy())
        assert np.array_equal(eng.outs[eng.residual_bits].cpu().numpy(), fqm(xs[2]).numpy())
    assert np.array_equal(a(devs[1]).cpu().numpy(), fqm(xs[1]).numpy())
    assert np.array_equal(b(devs[0]).cpu().numpy(), fqm(xs[0]).numpy())
    assert (a.fallbacks, b.fallbacks, eng.fallbacks) == (1, 0, 0)
