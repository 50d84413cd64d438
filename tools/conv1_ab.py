#!/usr/bin/env python
"""conv1 of AlexNet alone (227x227x3 -> 55x55x96, 11x11 / 4, bf16x2 operands): the weight-stationary family conv_ws
(force_kernel = 7) against pq_gemm_tc mode 1 (force_kernel = 6), in one process on one GPU.

For every batch size the two families alternate, round by round; a round is `iters` back-to-back launches between CUDA
events.  Each family first runs once untimed, so that the autotuner picks its tiling for the batch size.  Per family the
tool prints the median and min-max of the per-launch time over the rounds, the executed tensor-core TFLOP/s (every MMA the
plan issues, padding included) and the useful TFLOP/s (2 x N x 55 x 55 x 96 x 363 flops of the dense layer), with the
card name, power limit and maximum SM clock.

    python tools/conv1_ab.py [--batches 1,4,40,256,1024] [--rounds 7] [--iters 20] [--out conv1_ab.json]
"""
import argparse
import ctypes
import importlib
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HI, WI, CIN, COUT, K, PAD, STRIDE = 227, 227, 3, 96, 11, 0, 4
FAMILIES = {7: "conv_ws", 6: "pq_gemm_tc mode 1"}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        lim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        lim = "unknown"
    return name, lim


def executed_macs(desc):
    """Tensor-core MACs one launch issues, from the plan string (two bf16 MMAs of K = 16 per k-step)."""
    m = re.search(r"pq_gemm_tc_ws\(.*? N=(\d+) positions=(\d+) .*?grid=(\d+) .*?ksteps=(\d+)", desc)
    if m:
        n, p, grid, ks = (float(v) for v in m.groups())
        return grid * ks * 2 * 16 * p * n
    m = re.search(r"pq_gemm_tc\(.*?NT=(\d+) .*?grid=(\d+) .*?ksteps=(\d+)", desc)
    nt, grid, ks = (float(v) for v in m.groups())
    return grid * ks * 2 * 16 * 128 * nt


def stats(v):
    v = np.asarray(v, np.float64)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,40,256,1024")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20, help="launches per round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = importlib.import_module("quantized-cnn_b200")
    name, lim = card()
    print("card: %s  power.limit, clocks.max.sm: %s" % (name, lim), flush=True)
    ctx = q.Context(0)
    rng = np.random.RandomState(1)
    ctrd = (rng.randn(1, 128, 8) / np.sqrt(CIN * K * K)).astype(np.float32)
    asmt = rng.randint(0, 128, size=(COUT, K, K, 1)).astype(np.uint8)
    bias = (rng.randn(COUT) * 0.1).astype(np.float32)
    L = q.ConvLayer(ctx, CIN, HI, WI, COUT, K, PAD, STRIDE, 1, ctrd, asmt, bias)
    ho, wo, co = L.out_dims()
    stream = torch.cuda.current_stream()
    res = dict(card=name, power_limit_and_max_sm_clock=lim, rounds=args.rounds, iters=args.iters, batches={})
    for N in [int(b) for b in args.batches.split(",")]:
        x = torch.from_numpy((np.abs(rng.randn(N, HI, WI, CIN)) * 20).astype(np.float32)).cuda()
        y = torch.empty((N, ho, wo, co), dtype=torch.float32, device="cuda")
        useful = 2.0 * N * ho * wo * co * K * K * CIN

        def launch():
            q._check(q.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(x.data_ptr()), N, ctypes.c_void_p(y.data_ptr()), 1,
                                                  ctypes.c_void_p(stream.cuda_stream)))
        plans, times = {}, {k: [] for k in FAMILIES}
        for r in range(args.rounds + 1):
            for kern in FAMILIES:
                L.set_param("force_kernel", kern)
                if r == 0:
                    launch()          # tiling chosen on the device for this batch size
                    torch.cuda.synchronize()
                    plans[kern] = L.describe(N)
                    continue
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    launch()
                b.record()
                torch.cuda.synchronize()
                times[kern].append(a.elapsed_time(b) / args.iters)
        out = {}
        for kern, fam in FAMILIES.items():
            s = stats(times[kern])
            ex = 2.0 * executed_macs(plans[kern])
            out[fam] = dict(ms=s, executed_TFLOPs=ex / (s["median"] * 1e-3) / 1e12,
                            useful_TFLOPs=useful / (s["median"] * 1e-3) / 1e12, plan=plans[kern])
            print("N=%-5d %-18s %8.4f ms (%.4f - %.4f)  executed %6.1f TFLOP/s  useful %6.1f TFLOP/s  %s"
                  % (N, fam, s["median"], s["min"], s["max"], out[fam]["executed_TFLOPs"], out[fam]["useful_TFLOPs"],
                     plans[kern].split(" smem")[0]), flush=True)
        res["batches"][str(N)] = out
        del x, y
        torch.cuda.empty_cache()
    L.close()
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
