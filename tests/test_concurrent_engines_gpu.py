"""-m gpu: several compiled engines at once on one device, each against an exact reference.  Every forward of a CompiledModel
resets a status word, lets its kernels raise sticky overflow flags in it, and copies it to ``eng.flag``; the host then takes the
exact int32 or saturating fallback.  These tests check that one engine's flags never reach another: an interleave fixed with
events (another engine's whole forward between an engine's kernels and its copy of the word), two engines replayed freely on
two streams, two threads each with its own engine (one compiling while the other runs eagerly in another execution mode), and
one fresh model compiled by two threads at once."""
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200 import ops, qtensor
from hawq_b200.synthetic import synthetic_batch
from tests.engine_harness import _eager, _oracle, assert_rows, golden_model, int8_input, int_oracle
from tests.util import golden_act_ranges, load_net_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ARCH, SCHEME = "resnet18", "bops_0.25"
SHRINK = ("stage2.unit2.quant_act_int32", 0.75)
CLEAN, OVER = (0, 1, 2), 3          # indices into the ResNet-18 batches: OVER pushes the uint16 stream past 65535


@pytest.fixture(scope="module")
def resnet():
    """ResNet-18 bops_0.25 with stage2.unit2's 16-bit range shrunk to 0.75 (as in test_engine_paths_gpu): three ordinary batches
    of 8 fit the uint16 stream, a batch at the int8 extremes does not.  Oracle logits and eager status words, computed once."""
    _, meta = load_net_golden(ARCH, SCHEME)
    xs = [synthetic_batch(8, 100 + i) for i in CLEAN] + [synthetic_batch(8, 104) * 1000.0]
    fqm = _oracle(ARCH, SCHEME, meta, SHRINK)
    want = [fqm(x).numpy() for x in xs]
    q = golden_model(ARCH, SCHEME, meta, SHRINK)
    devs = [int8_input(x, meta["acts"]["quant_input"]["scale"]).to(DEV) for x in xs]
    status = [_eager(q, x, residual_bits=16, checked=True)[1] for x in devs]
    assert [s & 1 for s in status] == [0, 0, 0, 1], status
    assert not any(s & 6 for s in status), status
    return SimpleNamespace(q=q, meta=meta, xs=devs, want=want, status=status)


@pytest.fixture(scope="module")
def mnv2():
    """MobileNetV2 uniform8 on its golden ranges, two batches of 8 and their IntMobileNetV2 logits."""
    _, meta = load_net_golden("mobilenetv2_w1", "uniform8")
    ranges = golden_act_ranges(meta)
    _, _, net = int_oracle("uniform8", ranges, synthetic_batch(*meta["input"]))
    xs = [synthetic_batch(8, 300 + i) * (1.0 + 0.3 * i) for i in range(2)]
    want = [net(x.numpy()) for x in xs]
    s_in = np.float32(net.acts["quant_input"]["scale"])
    devs = [int8_input(x, s_in).to(DEV) for x in xs]
    q = hb.build_synthetic_qresnet("mobilenetv2_w1", "uniform8", act_ranges=ranges)
    assert all(_eager(q, x, residual_bits=16, checked=True)[1] & 7 == 0 for x in devs)
    return SimpleNamespace(q=q, xs=devs, want=want)


# ------------------------------------------------------------------------------------------------ a fixed interleave
class Interleave:
    """Wraps ops.copy_status.  When engine `a` copies its status word into a.flag, the hook first runs one forward of engine `b`
    on its own stream, ordered with events between a's kernels and a's copy: a's kernels -> b's reset, kernels and copy -> a's
    copy.  Armed for one copy at a time; `b_out` holds b's logits and status word of that forward."""

    def __init__(self, monkeypatch):
        self.real = ops.copy_status
        self.stream = torch.cuda.Stream(device=DEV)
        self.armed = None
        self.b_out = None
        monkeypatch.setattr(ops, "copy_status", self.copy_status)

    def arm(self, a, b, xb):
        self.armed, self.b_out = (a, b, xb), None

    def copy_status(self, idx, dst):
        if self.armed is not None and dst is self.armed[0].flag:
            a, b, xb = self.armed
            self.armed = None
            cur = torch.cuda.current_stream(idx)
            e1 = torch.cuda.Event()
            e1.record(cur)
            with torch.cuda.stream(self.stream):
                self.stream.wait_event(e1)
                self.b_out = (b.run_async(xb).clone(), b.flag.clone())
                e2 = torch.cuda.Event()
                e2.record(self.stream)
            cur.wait_event(e2)
        self.real(idx, dst)


def test_interleave_keeps_each_engines_status_word(resnet, monkeypatch):
    """Engine A (eager: reset, launches, copy, the graph's discipline) and engine B (a CUDA graph of the same model).  B's whole
    forward on a clean batch runs after A's overflowing kernels and before A copies its word: A must still see its overflow and
    take the exact int32 fallback once, and B must not.  Then the converse, in a fresh A: B's overflowing forward inside A's clean
    one must neither raise A's flag nor change A's logits."""
    r = resnet
    clean, over = r.xs[CLEAN[0]], r.xs[OVER]
    b = hb.compile_model(r.q, clean)
    solo = {}
    for i in (CLEAN[0], OVER):
        solo[i] = b.run_async(r.xs[i]).clone()
        assert int(b.flag.item()) == r.status[i]
    a = hb.compile_model(r.q, over, use_cuda_graph=False)
    hook = Interleave(monkeypatch)

    hook.arm(a, b, clean)
    got = a(over).clone()
    torch.cuda.synchronize()
    assert hook.b_out is not None, "A's status word copy was not intercepted"
    exact = np.array_equal(got.cpu().numpy(), r.want[OVER])
    assert (a.fallbacks, exact) == (1, True), "A, overflowing, with B's clean forward inside: fallbacks %d, logits %s the oracle" \
        % (a.fallbacks, "equal" if exact else "differ from")
    assert torch.equal(hook.b_out[0], solo[CLEAN[0]]) and int(hook.b_out[1]) == r.status[CLEAN[0]]
    assert b.fallbacks == 0

    a = hb.compile_model(r.q, clean, use_cuda_graph=False)
    hook.arm(a, b, over)
    got = a(clean).clone()
    torch.cuda.synchronize()
    assert hook.b_out is not None, "A's status word copy was not intercepted"
    assert a.fallbacks == 0, "B's overflow flag reached A"
    assert_rows(got, r.want[CLEAN[0]], "A, clean, with B's overflowing forward inside")
    assert torch.equal(hook.b_out[0], solo[OVER]) and int(hook.b_out[1]) == r.status[OVER]


# ------------------------------------------------------------------------------------------------ two streams, no host sync
def test_two_engines_replayed_freely_on_two_streams(resnet, mnv2):
    """ResNet-18 (batches alternating overflowing and clean) and MobileNetV2, each on its own stream, 8 rounds of run_async with no
    host synchronisation between them.  Once both streams have drained, each round's copied flag equals its batch's eager status
    word, and each round's logits, or where the flag is raised __call__'s exact re-run, equal the oracle."""
    r, m = resnet, mnv2
    ea = hb.compile_model(r.q, r.xs[CLEAN[0]])
    eb = hb.compile_model(m.q, m.xs[0])
    sa, sb = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
    sa.wait_stream(torch.cuda.current_stream())
    sb.wait_stream(torch.cuda.current_stream())
    order_a = [OVER, CLEAN[0], OVER, CLEAN[1], OVER, CLEAN[2], OVER, CLEAN[0]]
    order_b = [0, 1] * 4
    rounds = []
    for ia, ib in zip(order_a, order_b):
        with torch.cuda.stream(sa):
            ya = (ea.run_async(r.xs[ia]).clone(), ea.flag.clone())
        with torch.cuda.stream(sb):
            yb = (eb.run_async(m.xs[ib]).clone(), eb.flag.clone())
        rounds.append((ia, ya, ib, yb))
    torch.cuda.synchronize()
    for k, (ia, (la, fa), ib, (lb, fb)) in enumerate(rounds):
        assert int(fa) == r.status[ia], "round %d: ResNet-18 flag %d, its batch's eager status %d" % (k, int(fa), r.status[ia])
        assert int(fb) == 0, "round %d: MobileNetV2 flag %d" % (k, int(fb))
        assert_rows(ea(r.xs[ia]) if int(fa) & 7 else la, r.want[ia], "round %d, ResNet-18" % k)
        assert_rows(lb, m.want[ib], "round %d, MobileNetV2" % k)
    assert ea.fallbacks == order_a.count(OVER)
    assert eb.fallbacks == 0


# ------------------------------------------------------------------------------------------------ threads
def run_threads(*targets, timeout=900):
    """Runs each target on its own thread (its own stream, started together at a barrier); re-raises the first exception."""
    barrier = threading.Barrier(len(targets), timeout=timeout)
    errors, results = [], [None] * len(targets)

    def body(i, fn):
        try:
            with torch.cuda.stream(torch.cuda.Stream(device=DEV)), torch.no_grad():
                results[i] = fn(barrier)
            torch.cuda.current_stream(DEV).synchronize()
        except BaseException as e:            # noqa: B902 - handed to the main thread
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=body, args=(i, fn), daemon=True) for i, fn in enumerate(targets)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a thread did not finish within %d s" % timeout
    if errors:
        raise errors[0]
    return results


def test_two_threads_each_with_its_own_engine(resnet, mnv2):
    """Thread 1 sits inside engine_mode(residual_bits=32, fast_kernels=False) with the dual kernel switched off for itself, and runs
    an eager MobileNetV2 engine; thread 2 meanwhile compiles the ResNet-18 engine and calls it, fallbacks included.  The execution
    mode is per thread: thread 2's launch counts per graph and its logits equal a solo compile's, and thread 1's logits equal the
    oracle."""
    r, m = resnet, mnv2
    order = [CLEAN[0], OVER, CLEAN[1], OVER, CLEAN[2]]
    solo = hb.compile_model(r.q, r.xs[CLEAN[0]])
    solo_out = [solo(r.xs[i]).cpu().numpy() for i in order]
    solo_launches = dict(solo.launches)
    assert set(solo_launches) == {16, 32} and solo.fallbacks == 2
    e1 = hb.compile_model(m.q, m.xs[0], use_cuda_graph=False)

    def eager_mobilenet(barrier):
        with qtensor.engine_mode(residual_bits=32, fast_kernels=False):
            qtensor.config.dual = False
            barrier.wait()
            return [e1(m.xs[i % 2]).cpu().numpy() for i in range(6)], e1.fallbacks

    def compile_resnet(barrier):
        barrier.wait()
        e2 = hb.compile_model(r.q, r.xs[CLEAN[0]])
        return [e2(r.xs[i]).cpu().numpy() for i in order], dict(e2.launches), e2.fallbacks

    dual = qtensor.config.dual
    (out1, fb1), (out2, launches2, fb2) = run_threads(eager_mobilenet, compile_resnet)
    assert qtensor.config.dual == dual, "thread 1's execution mode reached the main thread"
    assert fb1 == 0
    for i, y in enumerate(out1):
        assert_rows(y, m.want[i % 2], "thread 1, call %d" % i)
    assert launches2 == solo_launches
    assert fb2 == 2
    for i, y, s in zip(order, out2, solo_out):
        assert np.array_equal(y, s)
        assert_rows(y, r.want[i], "thread 2, batch %d" % i)


def test_one_fresh_model_compiled_by_two_threads(resnet):
    """Two threads compile one freshly frozen model whose integer plans do not exist yet, each for its own batch, and call it on
    that batch and on the overflowing one: every plan either thread uses is complete on the device, and all logits equal the
    oracle."""
    r = resnet
    q = golden_model(ARCH, SCHEME, r.meta, SHRINK)
    assert not any("_hawq_cache" in mod.__dict__ for mod in q.modules())

    def compile_and_run(k):
        def fn(barrier):
            barrier.wait()
            eng = hb.compile_model(q, r.xs[k])
            return [eng(r.xs[k]).cpu().numpy(), eng(r.xs[OVER]).cpu().numpy()], eng.fallbacks
        return fn

    results = run_threads(compile_and_run(CLEAN[0]), compile_and_run(CLEAN[1]))
    for k, (outs, fallbacks) in zip((CLEAN[0], CLEAN[1]), results):
        assert fallbacks == 1
        assert_rows(outs[0], r.want[k], "thread compiled for batch %d" % k)
        assert_rows(outs[1], r.want[OVER], "thread compiled for batch %d, overflowing batch" % k)
