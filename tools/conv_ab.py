#!/usr/bin/env python
"""AlexNet conv layers alone (bf16x2 operands): the weight-stationary family conv_ws (force_kernel = 7) against the
decode-at-use pq_gemm_tc (force_kernel = 6) -- mode 1 for conv1, mode 0 for conv2-conv5 -- in one process on one GPU.

For every layer and batch size the two families alternate, round by round; a round is `iters` back-to-back launches
between CUDA events.  Each family is a layer object of its own (same parameters, the family pinned once), so that its
tiling is chosen on the device by one untimed launch per batch size and no timed round re-tunes.  Per
family the tool prints the median and min-max of the per-launch time over the rounds, the executed tensor-core TFLOP/s
(every MMA the plan issues, padding included) and the useful TFLOP/s (2 x N x Ho x Wo x Cout x k^2 x Cin/grp flops of the
dense layer), the plan, and the card name, power limit and maximum SM clock.

    python tools/conv_ab.py [--layers conv1,conv2,conv3,conv4,conv5] [--batches 1,4,40,256,1024] [--rounds 7]
                            [--iters 20] [--out conv_ab.json]
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

# name: (Hi, Wi, Cin, Cout, k, pad, stride, groups, S, K, d) -- the AlexNet layers of bench.py
LAYERS = {
    "conv1": (227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8),
    "conv2": (27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8),
    "conv3": (13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8),
    "conv4": (13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8),
    "conv5": (13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8),
}
FAMILIES = {7: "conv_ws", 6: "pq_gemm_tc"}


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


def run_layer(q, ctx, name, batches, args, rng, res):
    import torch
    Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d = LAYERS[name]
    ctrd = (rng.randn(S, K, d) / np.sqrt(Cin // G * k * k)).astype(np.float32)
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    bias = (rng.randn(Cout) * 0.1).astype(np.float32)
    lay = {}
    for kern in FAMILIES:
        lay[kern] = q.ConvLayer(ctx, Cin, Hi, Wi, Cout, k, pad, stride, G, ctrd, asmt, bias)
        lay[kern].set_param("tensor_core", 2)
        lay[kern].set_param("force_kernel", kern)
    ho, wo, co = lay[7].out_dims()
    stream = torch.cuda.current_stream()
    res[name] = {}
    for N in batches:
        x = torch.from_numpy((np.abs(rng.randn(N, Hi, Wi, Cin)) * 20).astype(np.float32)).cuda()
        y = torch.empty((N, ho, wo, co), dtype=torch.float32, device="cuda")
        useful = 2.0 * N * ho * wo * co * k * k * (Cin // G)

        def launch(L):
            q._check(q.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(x.data_ptr()), N, ctypes.c_void_p(y.data_ptr()), 1,
                                                  ctypes.c_void_p(stream.cuda_stream)))
        plans, times = {}, {kern: [] for kern in FAMILIES}
        for r in range(args.rounds + 1):
            for kern in FAMILIES:
                if r == 0:
                    launch(lay[kern])          # tiling chosen on the device for this batch size
                    torch.cuda.synchronize()
                    plans[kern] = lay[kern].describe(N)
                    continue
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    launch(lay[kern])
                b.record()
                torch.cuda.synchronize()
                times[kern].append(a.elapsed_time(b) / args.iters)
        out = {}
        for kern, fam in FAMILIES.items():
            s = stats(times[kern])
            ex = 2.0 * executed_macs(plans[kern])
            out[fam] = dict(ms=s, executed_TFLOPs=ex / (s["median"] * 1e-3) / 1e12,
                            useful_TFLOPs=useful / (s["median"] * 1e-3) / 1e12, plan=plans[kern])
            print("%s N=%-5d %-11s %8.4f ms (%.4f - %.4f)  executed %6.1f TFLOP/s  useful %6.1f TFLOP/s  %s"
                  % (name, N, fam, s["median"], s["min"], s["max"], out[fam]["executed_TFLOPs"], out[fam]["useful_TFLOPs"],
                     plans[kern].split(" smem")[0]), flush=True)
        res[name][str(N)] = out
        del x, y
        torch.cuda.empty_cache()
    for L in lay.values():
        L.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", default="conv1,conv2,conv3,conv4,conv5")
    ap.add_argument("--batches", default="1,4,40,256,1024")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20, help="launches per round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    layers = args.layers.split(",")
    for name in layers:
        if name not in LAYERS:
            ap.error("unknown layer %r (known: %s)" % (name, ",".join(LAYERS)))
    q = importlib.import_module("quantized-cnn_b200")
    name, lim = card()
    print("card: %s  power.limit, clocks.max.sm: %s" % (name, lim), flush=True)
    ctx = q.Context(0)
    rng = np.random.RandomState(1)
    res = dict(card=name, power_limit_and_max_sm_clock=lim, rounds=args.rounds, iters=args.iters, layers={})
    for layer in layers:
        run_layer(q, ctx, layer, [int(b) for b in args.batches.split(",")], args, rng, res["layers"])
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
