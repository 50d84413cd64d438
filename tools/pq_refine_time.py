"""Times the error-correcting FC quantizer (qcnn_pq_refine_fc) on AlexNet fc6 / fc7 / fc8 (N = 4 Din inputs) and VGG16
fc6 (N = 8192) with seeded Gaussian weights (std 1/sqrt(Din)) and inputs, started from pq_quantize_fc (iters = 20) at
the shipped AlexNet (K, d).  Per layer, from one run under torch.profiler (CUDA activities): the Gram kernel's time, the
median per sweep of the sum of kernel durations (the sweeps are split at their loss kernels), how that splits between
the per-block cooperative kernel and the trailing GEMMs, achieved fp64 TFLOP/s from shape-based flop counts
(Gram: N Din (Din + 1), the useful lower triangle; sweep: 2 Dout Din^2, its GEMM work), and the loss trace.  Then, with
the profiler off, the wall time of a whole call.  Prints the card, its power limit and max SM clock.
    python tools/pq_refine_time.py [--sweeps 3] [--layers alexnet_fc6 ...]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = {   # name: (Din, Dout, K, d, N)
    "alexnet_fc6": (9216, 4096, 32, 4, 4 * 9216),
    "alexnet_fc7": (4096, 4096, 32, 4, 4 * 4096),
    "alexnet_fc8": (4096, 1000, 16, 1, 4 * 4096),
    "vgg16_fc6": (25088, 4096, 32, 4, 8192),
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def kernels(prof):
    """(name, start us, duration us) of every CUDA kernel of the trace, in start order"""
    from torch.autograd import DeviceType
    ev = [(e.name, e.time_range.start, e.time_range.end - e.time_range.start) for e in prof.events()
          if e.device_type == DeviceType.CUDA and "pqr_" in e.name]
    return sorted(ev, key=lambda x: x[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=3)
    ap.add_argument("--layers", nargs="*", default=list(LAYERS))
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "needs a GPU"
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    print("card: %s (name, power limit, max SM clock)" % card())
    results = []
    for name in args.layers:
        Din, Dout, K, d, N = LAYERS[name]
        W = (np.random.default_rng(1).standard_normal((Dout, Din), dtype=np.float32) / np.float32(np.sqrt(Din)))
        g = torch.Generator(device="cuda").manual_seed(2)
        x = torch.randn((N, Din), generator=g, device="cuda", dtype=torch.float32)
        c0, a0, _ = q.pq_quantize_fc(ctx, W, K, d, iters=20, seed=3)
        q.pq_refine_fc(ctx, W, x[:64], c0, a0, sweeps=1)   # warm-up: module load, smem opt-in
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, _, loss = q.pq_refine_fc(ctx, W, x, c0, a0, sweeps=args.sweeps)
            torch.cuda.synchronize()
        ev = kernels(prof)
        gram = sum(t for n, _, t in ev if "pqr_gemm_kernel<true>" in n)
        ends = [i for i, (n, _, _) in enumerate(ev) if "pqr_loss_final" in n]
        sweeps, blk, trail = [], [], []
        for a, b in zip(ends[:-1], ends[1:]):
            part = ev[a + 1:b + 1]
            sweeps.append(sum(t for _, _, t in part))
            blk.append(sum(t for n, _, t in part if "pqr_block_kernel" in n))
            trail.append(sum(t for n, _, t in part if "pqr_gemm_kernel<false>" in n))
        t0 = time.perf_counter()
        q.pq_refine_fc(ctx, W, x, c0, a0, sweeps=args.sweeps)
        wall = time.perf_counter() - t0
        sweep_ms = float(np.median(sweeps)) / 1e3
        gram_ms = gram / 1e3
        r = dict(layer=name, Din=Din, Dout=Dout, K=K, d=d, N=N, gram_ms=gram_ms,
                 gram_tflops=N * Din * (Din + 1) / (gram_ms * 1e-3) / 1e12, sweep_ms=sweep_ms,
                 sweep_block_kernel_ms=float(np.median(blk)) / 1e3, sweep_gemm_ms=float(np.median(trail)) / 1e3,
                 sweep_tflops=2.0 * Dout * Din * Din / (sweep_ms * 1e-3) / 1e12, call_wall_s=wall,
                 loss=[float(v) for v in loss], loss_ratio=float(loss[-1] / loss[0]))
        results.append(r)
        print("%-12s Gram %8.2f ms (%5.1f TFLOP/s)  sweep %8.2f ms (%5.1f TFLOP/s; block kernels %.2f ms, GEMMs %.2f ms)  "
              "call %.2f s  loss x%.3f after %d sweeps"
              % (name, gram_ms, r["gram_tflops"], sweep_ms, r["sweep_tflops"], r["sweep_block_kernel_ms"],
                 r["sweep_gemm_ms"], wall, r["loss_ratio"], args.sweeps))
        print("  loss trace: " + " ".join("%.6g" % v for v in loss))
        del x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), sweeps=args.sweeps, results=results), f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
