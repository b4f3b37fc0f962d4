#!/usr/bin/env python
"""Latency table of this engine + re-solved bit allocation (ILP.ipynb with this engine's timings instead of the T4 table).

usage: python tools/ilp_b200.py DETAIL_UNIFORM4.json DETAIL_UNIFORM8.json [--arch resnet50] [--out out.json]
The detail files come from `python bench.py --arch A --scheme uniform4|uniform8 --detail FILE` on the GPU."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hawq_b200 import ilp  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("detail4")
ap.add_argument("detail8")
ap.add_argument("--arch", default="resnet50")
ap.add_argument("--data", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ilp_data.json"))
ap.add_argument("--out", default="")
a = ap.parse_args()
data = json.load(open(a.data))[a.arch]
l4, l8 = ilp.latency_table_from_detail(json.load(open(a.detail4)), json.load(open(a.detail8)), a.arch, data["parameters"])
names = ilp.layer_order(a.arch)
b200 = dict(data, latency_int4=l4.tolist(), latency_int8=l8.tolist())
res = {"arch": a.arch, "unit": "ms per launch at the bench batch size (CUDA events, eager pass)", "layers": names,
       "latency_int4": l4.tolist(), "latency_int8": l8.tolist(), "sum_int4": float(l4.sum()), "sum_int8": float(l8.sum()),
       "layers_faster_at_4bit": [n for n, x, y in zip(names, l4, l8) if x < y], "allocations": {}}
for frac in (0.25, 0.5, 0.75):
    bits = ilp.allocate(b200, "latency", frac, a.arch)
    res["allocations"]["latency_%s" % frac] = {"n_8bit": sum(1 for v in bits.values() if v == 8), "bits": bits}
print("sum of conv launches: int4 %.3f ms, int8 %.3f ms; %d of %d layers are faster at 4 bit" % (res["sum_int4"], res["sum_int8"], len(res["layers_faster_at_4bit"]), len(names)))
for k, v in res["allocations"].items():
    print(k, "->", v["n_8bit"], "of", len(names), "layers at 8 bit")
if a.out:
    json.dump(res, open(a.out, "w"), indent=1)
