"""SURVEY.md 8(f) rank 4: the bit-allocation ILP (hawq_b200/ilp.py) against the reference's own published results.
With the notebook's data (tests/golden/ilp_data.json, extracted from ILP.ipynb) the exact solver must reproduce the bit
configurations the reference ships in bit_config.py for every constraint type and budget."""
import itertools
import json
import os

import numpy as np
import pytest

from hawq_b200 import ilp
from hawq_b200.bit_config import get_bit_config

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = json.load(open(os.path.join(HERE, "golden", "ilp_data.json")))


def _objective_and_cost(arch, bits, constraint):
    d = DATA[arch]
    names = ilp.layer_order(arch)
    x = np.array([1.0 if bits[n] == 8 else 0.0 for n in names])
    sens = np.array(d["Hutchinson_trace"]) * (np.array(d["delta_weights_8bit_square"]) - np.array(d["delta_weights_4bit_square"]))
    c4, c8 = {"modelsize": (0.5 * np.array(d["parameters"]), np.array(d["parameters"])),
              "bops": (np.array(d["bops"]) / 64, np.array(d["bops"]) / 16),
              "latency": (np.array(d["latency_int4"]), np.array(d["latency_int8"]))}[constraint]
    return float((x * sens).sum()), float((c4 + x * (c8 - c4)).sum()), c4, c8


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
@pytest.mark.parametrize("constraint", ["modelsize", "bops", "latency"])
@pytest.mark.parametrize("fraction", [0.25, 0.5, 0.75])
def test_reproduces_published_bit_configs(arch, constraint, fraction):
    got = ilp.allocate(DATA[arch], constraint, fraction, arch)
    published = get_bit_config(arch, "%s_%s" % (constraint, fraction))
    names = ilp.layer_order(arch)
    assert set(names) <= set(published)
    obj_g, cost_g, c4, c8 = _objective_and_cost(arch, got, constraint)
    obj_p, cost_p, _, _ = _objective_and_cost(arch, published, constraint)
    limit = ilp.budget(c4, c8, fraction)
    assert cost_g <= limit + 1e-9 and cost_p <= limit + 1e-9
    for a, b in ilp.tie_pairs(arch):
        assert got[names[a]] == got[names[b]]
    if (arch, constraint, fraction) == ("resnet50", "modelsize", 0.25):
        # the one published configuration that is not optimal for the notebook's own data: ours is feasible and strictly better
        assert [n for n in names if got[n] != published[n]] == ["stage3.unit6.quant_convbn1"]
        assert obj_g < obj_p
    else:
        assert {n: got[n] for n in names} == {n: published[n] for n in names}


def test_exact_against_brute_force():
    r = np.random.RandomState(0)
    for trial in range(30):
        n = 10
        sens = -r.uniform(0.01, 1.0, n)
        c4 = r.uniform(0.1, 1.0, n)
        c8 = c4 + r.uniform(-0.2, 1.0, n)              # some layers cheaper at 8 bit
        ties = [(0, 3)] if trial % 2 else []
        limit = ilp.budget(c4, c8, r.uniform(0.2, 0.8))
        best = None
        for x in itertools.product((0, 1), repeat=n):
            if any(x[a] != x[b] for a, b in ties):
                continue
            if sum(c4[i] + x[i] * (c8[i] - c4[i]) for i in range(n)) <= limit + 1e-12:
                v = sum(x[i] * sens[i] for i in range(n))
                if best is None or v < best - 1e-15:
                    best = v
        try:
            bits = ilp.solve(sens, c4, c8, limit, ties)
        except ValueError:
            assert best is None
            continue
        x = [1 if b == 8 else 0 for b in bits]
        assert sum(c4[i] + x[i] * (c8[i] - c4[i]) for i in range(n)) <= limit + 1e-9
        assert abs(sum(x[i] * sens[i] for i in range(n)) - best) < 1e-12


def test_b200_latency_table_from_bench_detail():
    """per-launch timings of this engine (bench.py --detail of ResNet-50 uniform4 and uniform8 runs, stored in
    tests/golden/detail_resnet50_h100.json) -> the notebook's latency arrays -> re-solved."""
    det = json.load(open(os.path.join(HERE, "golden", "detail_resnet50_h100.json")))
    d4, d8 = det["uniform4"], det["uniform8"]
    l4, l8 = ilp.latency_table_from_detail(d4, d8, "resnet50", DATA["resnet50"]["parameters"])
    assert l4.shape == (52,) and l8.shape == (52,) and (l4 > 0).all() and (l8 > 0).all()
    conv4 = sum(l["ms"] for l in d4["layers"] if l["kernel"].startswith("conv"))
    assert abs(l4.sum() - conv4) < 1e-9                 # every convolution launch is accounted for exactly once
    table = dict(DATA["resnet50"], latency_int4=l4.tolist(), latency_int8=l8.tolist())
    bits = ilp.allocate(table, "latency", 0.5, "resnet50")
    assert set(bits.values()) <= {4, 8} and len(bits) == 52
