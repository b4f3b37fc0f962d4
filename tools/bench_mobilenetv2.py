"""MobileNetV2-1.0 on the integer engine: images/s of the compiled CUDA graph and a per-kernel-family breakdown.

    python tools/bench_mobilenetv2.py [--schemes uniform8,uniform4] [--batches 128,8] [--steps 30] [--warmup 5] [--repeats 5]

For each bit table and batch: a seeded synthetic model (calibrated on a seeded CPU batch), seeded int8 NHWC inputs, `CompiledModel`
graph replays timed with device events over --steps steps after --warmup, repeated --repeats times (median and range reported).
Parity: the logits of one timed batch must equal an eager run with int32 residuals and no ratio promises (exact integer
requantisation).  Breakdown (batch 128 only): one eager forward per repeat with every launch bracketed by CUDA events (ops.timer, as
bench.py --detail); per kernel family the median time per step and the achieved bytes/s of its algorithmic bytes, counted both at the
stored (zero-padded to multiples of 64) channel counts and at the model's logical ones, next to a device-to-device copy measured in
the same call.  Card name, power limit and SM clock are read in the same call."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--schemes", default="uniform8,uniform4")
    ap.add_argument("--batches", default="128,8")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--copy-gb", type=float, default=2.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import hawq_b200 as hb
    from hawq_b200 import ops, qtensor

    if not torch.cuda.is_available():
        raise SystemExit("bench_mobilenetv2 needs a GPU")
    dev = torch.device("cuda:0")

    def events_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    nbytes = int(args.copy_gb * 1e9) // 2
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    events_ms(lambda: dst.copy_(src), 3)
    copy_gbs = 2 * nbytes / events_ms(lambda: dst.copy_(src), 20) / 1e6
    del src, dst
    torch.cuda.empty_cache()

    result = {"gpu": gpu_info(), "copy_gbs": round(copy_gbs, 1), "runs": []}
    for scheme in args.schemes.split(","):
        q = hb.build_synthetic_qresnet("mobilenetv2_w1", scheme)
        s_in = float(qtensor._frozen_scale(q.quant_input))
        for batch in [int(b) for b in args.batches.split(",")]:
            g = torch.Generator().manual_seed(1000 + batch)
            xs = [torch.randn(batch, 3, 224, 224, generator=g) for _ in range(2)]
            q_in = [torch.clamp(torch.round(x * (1.0 / s_in)), -128, 127).to(torch.int8).permute(0, 2, 3, 1).contiguous().to(dev) for x in xs]
            eng = hb.compile_model(q, q_in[0])
            i = [0]

            def step():
                i[0] ^= 1
                eng.run_async(q_in[i[0]])
            events_ms(step, args.warmup)
            rates = [batch / events_ms(step, args.steps) * 1e3 for _ in range(args.repeats)]
            got = eng(q_in[0]).clone()
            n, h, w, c = q_in[0].shape
            with torch.no_grad(), qtensor.engine_mode(residual_bits=32, fast_kernels=False):
                want = q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in[0].view(-1), bits=8, signed=True), dev))
            torch.cuda.synchronize()
            run = {"scheme": scheme, "batch": batch, "img_s_median": round(statistics.median(rates), 1),
                   "img_s_range": [round(min(rates), 1), round(max(rates), 1)], "ms_per_step": round(batch / statistics.median(rates) * 1e3, 3),
                   "parity_bit_equal": bool(torch.equal(got, want)), "fallbacks": eng.fallbacks, "launches": eng.gpu_launches,
                   "clocks": gpu_info().get("clocks.sm")}
            if batch == 128:
                fam = {}
                for _ in range(args.repeats):
                    ops.timer = []
                    with torch.no_grad(), qtensor.engine_mode(residual_bits=16, checked=True):
                        q(hb.IntActivation(qtensor.Node("int", (n, c, h, w), data=q_in[0].view(-1), bits=8, signed=True), dev))
                    torch.cuda.synchronize()
                    per = {}
                    for label, info, e0, e1 in ops.timer:
                        f = per.setdefault(label, [0, 0.0, 0, 0])
                        f[0] += 1
                        f[1] += e0.elapsed_time(e1)
                        f[2] += info[1]
                        f[3] += info[2] if len(info) > 2 else info[1]
                    ops.timer = None
                    for label, f in per.items():
                        fam.setdefault(label, dict(launches=f[0], ms=[], stored_bytes=f[2], logical_bytes=f[3]))["ms"].append(f[1])
                run["families"] = {}
                for label, f in sorted(fam.items(), key=lambda kv: -statistics.median(kv[1]["ms"])):
                    ms = statistics.median(f["ms"])
                    run["families"][label] = {"launches": f["launches"], "ms": round(ms, 4), "stored_GB": round(f["stored_bytes"] / 1e9, 4),
                                              "logical_GB": round(f["logical_bytes"] / 1e9, 4),
                                              "stored_GBs": round(f["stored_bytes"] / ms / 1e6, 1),
                                              "logical_GBs": round(f["logical_bytes"] / ms / 1e6, 1),
                                              "stored_of_copy": round(f["stored_bytes"] / ms / 1e6 / copy_gbs, 3)}
            result["runs"].append(run)
            print(json.dumps(run), flush=True)
            del eng
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
