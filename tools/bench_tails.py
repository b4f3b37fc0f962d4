"""Per-launch timing of the 16 ResNet-50 bottleneck-tail launches at batch 128 (12 RESIDUAL 1x1 convolutions with the uint16
stream, 4 resize units), against a device-to-device copy ceiling measured in the same process.

    python tools/bench_tails.py [--repo DIR] [--batch 128] [--iters 100] [--regime le_one|le_2p20|both] [--a-bits 8|4]

Each launch runs on seeded random data with the engine's geometry and epilogue (uint16 stream, 8-bit copy for the next unit except
after the last unit), with ratios inside the promised range (HAWQ_EP_RATIOS_LE_ONE, or LE_2P20 with residual ratios above 1 as in
W4A4 networks) and biases inside the window, so the FP64 epilogue runs as it does in the network.  Each launch is timed with CUDA
events over --iters back-to-back launches after a warm-up; GB/s are the algorithmic bytes of ops.conv_work (resize units: the dual
work formula of ops.conv2d_dual) over that time.  --repo selects the tree whose hawq_b200 is imported (default: this one)."""
import argparse
import json
import os
import subprocess
import sys

# (stage, H = W, mid channels, out channels, tail launches)
STAGES = [(1, 56, 64, 256, 2), (2, 28, 128, 512, 3), (3, 14, 256, 1024, 5), (4, 7, 512, 2048, 2)]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repo", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--regime", choices=["le_one", "le_2p20", "both"], default="both")
    ap.add_argument("--a-bits", type=int, choices=[8, 4], default=8)
    ap.add_argument("--copy-gb", type=float, default=2.0)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.repo))
    import numpy as np
    import torch
    from hawq_b200 import ops
    from hawq_b200._lib import EP_RATIOS_LE_2P20, EP_RATIOS_LE_ONE, EPI_RESIDUAL, dyadic

    dev = "cuda:0"
    torch.cuda.init()
    r = np.random.RandomState(2026)
    ab = args.a_bits

    def act(n_vals):
        if ab == 4:
            v = r.randint(0, 256, size=n_vals // 2).astype(np.uint8)
            return torch.from_numpy(v).to(dev)
        return torch.from_numpy(r.randint(-128, 128, size=n_vals).astype(np.int8)).to(dev)

    def weights(cout, cin):
        return ops.upload_weights(torch.from_numpy(r.randint(-8, 8, size=(cout, 1, 1, cin)).astype(np.int8)), dev)

    def chan(c, lo, hi):
        me = [dyadic(float(np.exp(r.uniform(np.log(lo), np.log(hi))))) for _ in range(c)]
        return ops.make_chan(r.randint(-2000, 2000, size=c), [m for m, _ in me], [e for _, e in me]).to(dev)

    def launches(regime):
        """[(name, thunk)] in network order"""
        wide = regime == "le_2p20"
        flag = EP_RATIOS_LE_2P20 if wide else EP_RATIOS_LE_ONE
        hi = 30.0 if wide else 0.9
        out = []
        n = args.batch
        for si, (stage, hw, mid, cout, tails) in enumerate(STAGES):
            h_in = hw * (1 if stage == 1 else 2)
            cin_id = 64 if stage == 1 else cout // 2
            m = n * hw * hw
            # resize unit: main 1x1 (mid -> cout) + identity 1x1 of stride 1 (stage 1) or 2
            d = ops.conv_desc(n, hw, hw, mid, cout, 1, 1, 1, 0, ab, 1)
            d2 = ops.conv_desc(n, h_in, h_in, cin_id, cout, 1, 1, 1 if stage == 1 else 2, 0, ab, 1)
            x, x2 = act(m * mid), act(n * h_in * h_in * cin_id)
            w, w2 = weights(cout, mid), weights(cout, cin_id)
            ch, ch2 = chan(cout, 1e-3, hi), chan(cout, 1e-3, hi)
            y = torch.empty(m * cout, dtype=torch.int16, device=dev)
            low = torch.empty(m * cout, dtype=torch.int8, device=dev)
            ep = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=1, res_bits=32, y_bits=16, low_bits=8, low_me=dyadic(0.003),
                              low_clamp=(-128, 127), flags=flag)
            out.append(("s%d resize" % stage, "conv_dual",
                        lambda a=(x, d, ep, w, ch, d2, x2, w2, ch2, y, low): ops.conv2d_dual(*a[:9], out=a[9], out_low=a[10])))
            for ti in range(tails):
                last = si == len(STAGES) - 1 and ti == tails - 1
                dt = ops.conv_desc(n, hw, hw, mid, cout, 1, 1, 1, 0, ab)
                xt, wt = act(m * mid), weights(cout, mid)
                cht = chan(cout, 1e-3, hi)
                res = torch.from_numpy(r.randint(0, 900 if wide else 40000, size=m * cout).astype(np.uint16).view(np.int16)).to(dev)
                yt = torch.empty(m * cout, dtype=torch.int16, device=dev)
                lowt = None if last else torch.empty(m * cout, dtype=torch.int8, device=dev)
                ept = ops.epilogue(EPI_RESIDUAL, relu=1, res_kind=0, res_bits=16, res_me=dyadic(1.37 if wide else 0.37), y_bits=16,
                                   low_bits=0 if last else 8, low_me=dyadic(0.0004 if wide else 0.004), low_clamp=(-128, 127), flags=flag)
                out.append(("s%d tail %d" % (stage, ti + 1), "conv_igemm",
                            lambda a=(xt, dt, ept, wt[:cout * mid], cht, res, yt, lowt): ops.conv2d(*a[:5], res=a[5], out=a[6], out_low=a[7])))
        return out

    def time_it(fn, iters):
        for _ in range(args.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    # copy ceiling: device-to-device copy, read + write counted
    nbytes = int(args.copy_gb * 1e9) // 2
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    copy_ms = time_it(lambda: dst.copy_(src), 20)
    ceiling = 2 * nbytes / copy_ms / 1e6
    del src, dst
    torch.cuda.empty_cache()

    result = {"gpu": gpu_info(), "repo": os.path.abspath(args.repo), "batch": args.batch, "a_bits": ab, "iters": args.iters,
              "copy_ceiling_gbs": round(ceiling, 1)}
    for regime in (["le_one", "le_2p20"] if args.regime == "both" else [args.regime]):
        rows, tot_ms, tot_b = [], 0.0, 0
        for name, label, fn in launches(regime):
            ops.timer = []
            fn()
            _, (_, b), _, _ = ops.timer[0]
            ops.timer = None
            ms = time_it(fn, args.iters)
            rows.append({"launch": name, "kernel": label, "ms": round(ms, 4), "MB": round(b / 1e6, 1), "GBs": round(b / ms / 1e6, 1)})
            tot_ms += ms
            tot_b += b
        ops.reset_status(0)
        torch.cuda.synchronize()
        gbs = tot_b / tot_ms / 1e6
        result[regime] = {"launches": rows, "total_ms": round(tot_ms, 3), "total_GB": round(tot_b / 1e9, 3), "GBs": round(gbs, 1),
                          "of_copy_ceiling": round(gbs / ceiling, 3)}
        for row in rows:
            print("%-6s %-12s %-10s %8.4f ms %8.1f MB %8.1f GB/s" % (regime, row["launch"], row["kernel"], row["ms"], row["MB"], row["GBs"]))
        print("%-6s total %.3f ms, %.3f GB, %.1f GB/s = %.3f of the copy ceiling (%.1f GB/s)" % (regime, tot_ms, tot_b / 1e9, gbs, gbs / ceiling, ceiling))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
