"""The evaluation transform on the device (hawq_resize_crop_quantize_u8, compile_model(..., resize=256)) against the work it takes off
the host.

    python tools/bench_eval_transform.py [--steps 50] [--warmup 5] [--repeats 5] [--host-images 64] [--e2e-batches 20]

Images: seeded noise at a size mix shaped like ImageNet val (mostly 500 x 375, 375 x 500 and 500 x 333; some 1-3 MP images; some
below 256 px).  Reports, with the card name, power limit and SM clock read in the same call:
  kernel   ms per launch at B = 8 and B = 128 (device events, median of --repeats windows of --steps launches), and the rate of
           source bytes the crops read (eval_transform.source_box) over that time;
  host     ms per image of torchvision Resize(256) + CenterCrop(224) + ToTensor + Normalize on PIL images in this process (what
           the kernel replaces), and the host cores that would take at the measured end-to-end rate (not measured without PIL);
  e2e      ResNet-50 W8A8 (uniform8) images/s at batch 128 through run_pipelined from pinned PackedImages, against the uint8-224 route
           from pinned uint8 batches (host clock around --e2e-batches batches, ending in a synchronise), the pinned host-to-device
           copy time of one ragged batch, and the parity of the resize route with the uint8-224 route on the model's crops."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def imagenet_like(r, n):
    sizes = []
    for _ in range(n):
        u = r.rand()
        if u < 0.8:
            sizes.append([(500, 375), (375, 500), (500, 333)][r.randint(3)])
        elif u < 0.9:
            mp = r.uniform(1e6, 3e6)
            a = r.uniform(0.6, 1.6)
            sizes.append((int((mp * a) ** 0.5), int((mp / a) ** 0.5)))
        else:
            sizes.append(tuple(int(v) for v in r.randint(100, 256, size=2)))
    return [r.randint(0, 256, size=(h, w, 3), dtype="uint8") for h, w in sizes]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-images", type=int, default=64)
    ap.add_argument("--e2e-batches", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    import hawq_b200 as hb
    from hawq_b200 import ops
    from hawq_b200.engine import IMAGENET_MEAN, IMAGENET_STD
    from hawq_b200.eval_transform import source_box

    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_transform needs a GPU")
    dev = torch.device("cuda:0")
    r = np.random.RandomState(0)
    pool = imagenet_like(r, 4 * 128)
    result = {"gpu": gpu_info(), "kernel": {}}

    def events_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    # ---- kernel
    for b in (8, 128):
        p = hb.collate_images(pool[:b])
        pixels, table = p.pixels.to(dev), p.table().to(dev)
        out = torch.empty(b * 224 * 224 * 3, dtype=torch.int8, device=dev)
        read = sum(rows * cols * 3 for (_, rows), (_, cols) in (source_box(int(h), int(w), 256, (224, 224)) for h, w in p.sizes.tolist()))

        def launch():
            ops.resize_crop_quantize_u8(pixels, table, 256, (224, 224), IMAGENET_MEAN, IMAGENET_STD, 0.0208, (-128, 127), out)
        events_ms(launch, args.warmup)
        ms = statistics.median(events_ms(launch, args.steps) for _ in range(args.repeats))
        result["kernel"]["b%d" % b] = {"ms": round(ms, 4), "source_MB": round(read / 1e6, 2), "packed_MB": round(p.pixels.numel() / 1e6, 2),
                                       "source_GBs": round(read / ms / 1e6, 1), "clocks.sm": gpu_info().get("clocks.sm")}
        print(json.dumps({"kernel_b%d" % b: result["kernel"]["b%d" % b]}), flush=True)

    # ---- host cost of the same transform in PIL + torchvision
    try:
        from PIL import Image
        import torchvision.transforms as T
        tf = T.Compose([T.Resize(256), T.CenterCrop(224), T.ToTensor(), T.Normalize(IMAGENET_MEAN, IMAGENET_STD)])
        pil = [Image.fromarray(a) for a in pool[:args.host_images]]
        tf(pil[0])
        t0 = time.perf_counter()
        for im in pil:
            tf(im)
        host_ms = (time.perf_counter() - t0) * 1e3 / len(pil)
        result["host"] = {"ms_per_image": round(host_ms, 3), "torch_threads": torch.get_num_threads(),
                          "cpus": len(os.sched_getaffinity(0))}
    except ImportError as e:
        result["host"] = {"not_measured": str(e)}
    print(json.dumps({"host": result["host"]}), flush=True)

    # ---- end to end: ResNet-50 W8A8, batch 128
    B = 128
    q = hb.build_synthetic_qresnet("resnet50", "uniform8")
    packed = [hb.collate_images(pool[i * B:(i + 1) * B]).pin_memory() for i in range(4)]
    eng_r = hb.compile_model(q, torch.zeros((B, 224, 224, 3), dtype=torch.uint8, device=dev), resize=256)
    crops = [torch.randint(0, 256, (B, 224, 224, 3), generator=torch.Generator().manual_seed(i), dtype=torch.uint8).pin_memory()
             for i in range(4)]
    eng_u = hb.compile_model(q, crops[0].to(dev))

    def rate(eng, batches):
        for _ in eng.run_pipelined(batches[:2]):
            pass
        t0 = time.perf_counter()
        for _ in eng.run_pipelined([batches[i % len(batches)] for i in range(args.e2e_batches)]):
            pass
        torch.cuda.synchronize()
        return args.e2e_batches * B / (time.perf_counter() - t0)
    rates = {"resize": [], "uint8_224": []}
    for _ in range(args.repeats):                               # alternate the two routes
        rates["resize"].append(rate(eng_r, packed))
        rates["uint8_224"].append(rate(eng_u, crops))
    stage = torch.empty(packed[0].pixels.numel(), dtype=torch.uint8, device=dev)
    h2d_ms = statistics.median(events_ms(lambda: stage.copy_(packed[0].pixels, non_blocking=True), 10) for _ in range(3))
    from tests import eval_transform_model as etm               # parity: the resize route == the uint8-224 route on the model's crops
    u8 = torch.from_numpy(np.stack([etm.eval_crop_u8(packed[0].image(j).numpy(), 256, (224, 224)) for j in range(B)]))
    eng_p = hb.compile_model(q, u8.to(dev))
    parity = bool(torch.equal(eng_r(packed[0]), eng_p(u8.to(dev))))
    result["e2e"] = {"arch": "resnet50", "scheme": "uniform8", "batch": B,
                     "img_s_resize_median": round(statistics.median(rates["resize"]), 1),
                     "img_s_resize_range": [round(min(rates["resize"]), 1), round(max(rates["resize"]), 1)],
                     "img_s_uint8_224_median": round(statistics.median(rates["uint8_224"]), 1),
                     "img_s_uint8_224_range": [round(min(rates["uint8_224"]), 1), round(max(rates["uint8_224"]), 1)],
                     "packed_MB_per_batch": round(statistics.mean(p.pixels.numel() for p in packed) / 1e6, 2),
                     "h2d_ms_per_batch": round(h2d_ms, 3), "recaptures": eng_r.recaptures, "fallbacks": eng_r.fallbacks,
                     "parity_bit_equal": parity, "clocks.sm": gpu_info().get("clocks.sm")}
    if "ms_per_image" in result["host"]:
        result["e2e"]["host_cores_at_resize_rate"] = round(result["host"]["ms_per_image"] * result["e2e"]["img_s_resize_median"] / 1e3, 1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
