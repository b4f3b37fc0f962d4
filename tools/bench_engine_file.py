"""Plan files against the CompiledModel they were saved from: the replay rate of both, alternating in one process, the load time of
the plan against compile_model's, and the file's size.

    python tools/bench_engine_file.py [--steps 50] [--repeats 7] [--batch 128] [--out result.json]

Workloads: ResNet-50 and MobileNetV2-1.0, W8A8 (uniform8), int8 NHWC input.  Per repeat, one window of `steps` graph replays of
each engine (order alternating between repeats), timed with CUDA events; img/s is reported as the median and range over repeats.
The logits of a timed batch are compared between the two.  Prints one JSON line per workload, with the card's name and power limit
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import hawq_b200 as hb  # noqa: E402
from hawq_b200.synthetic import synthetic_batch  # noqa: E402
from oracle import int_ref as ir  # noqa: E402

WORKLOADS = [("resnet50", "uniform8"), ("mobilenetv2_w1", "uniform8")]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        name, limit = [v.strip() for v in r.stdout.strip().split(",")[:2]]
        return name, limit
    except Exception as e:              # the numbers stay valid without it; say so
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def window(run, x, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        run(x)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3


def bench(arch, scheme, batch, steps, repeats, tmp):
    q = hb.build_synthetic_qresnet(arch, scheme)
    scale = np.float32(hb.qtensor._frozen_scale(q.quant_input).item())
    x = torch.from_numpy(ir.quantize_input(synthetic_batch(batch, 11).numpy(), scale).astype(np.int8)).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng = hb.compile_model(q, x)
    torch.cuda.synchronize()
    t_compile = time.perf_counter() - t0
    path = os.path.join(tmp, "%s_%s.hawq" % (arch, scheme))
    size = eng.save(path)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    loaded = hb.load_engine(path)
    torch.cuda.synchronize()
    t_load = time.perf_counter() - t0
    info = loaded.info()
    runs = {"compiled": eng.run_async, "loaded": loaded.run_async}
    for run in runs.values():                 # warm-up
        window(run, x, 5)
    times = {k: [] for k in runs}
    for r in range(repeats):
        for k in (("compiled", "loaded") if r % 2 == 0 else ("loaded", "compiled")):
            times[k].append(window(runs[k], x, steps))
    same = torch.equal(eng.outs[eng.residual_bits], loaded.out)
    rate = {k: sorted(batch * steps / t for t in v) for k, v in times.items()}
    return dict(workload="%s %s b%d" % (arch, scheme, batch), logits_equal=bool(same),
                img_per_s={k: dict(median=v[len(v) // 2], min=v[0], max=v[-1]) for k, v in rate.items()},
                loaded_over_compiled=rate["loaded"][len(rate["loaded"]) // 2] / rate["compiled"][len(rate["compiled"]) // 2],
                compile_model_s=t_compile, load_engine_s=t_load, file_bytes=size, arena_bytes=int(info.arena_bytes),
                constant_bytes=int(info.constant_bytes), launches=loaded.launches, steps=steps, repeats=repeats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_engine_file needs a GPU")
    name, limit = card()
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        for arch, scheme in WORKLOADS:
            res = bench(arch, scheme, a.batch, a.steps, a.repeats, tmp)
            res.update(gpu=name, power_limit=limit)
            print(json.dumps(res), flush=True)
            results.append(res)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
