#!/usr/bin/env python
"""AlexNet and VGG16 block-1 conv layers alone (bf16x2 operands): the weight-stationary family conv_ws (force_kernel = 7)
against the decode-at-use pq_gemm_tc (force_kernel = 6) -- mode 1 for conv1, mode 0 for conv2-conv5 and VGG16 conv1_2 --
or, for VGG16 conv1_1 (3 input channels, which pq_gemm_tc does not take), against the LUT + gather kernels
(tensor_core = 0, the tiling timed on the device), in one process on one GPU.

For every layer and batch size the two families alternate, round by round; a round is `iters` back-to-back launches
between CUDA events.  Each family is a layer object of its own (same parameters, the family pinned once), so that its
tiling is chosen on the device by one untimed launch per batch size and no timed round re-tunes.  Per
family the tool prints the median and min-max of the per-launch time over the rounds, the executed tensor-core TFLOP/s
(every MMA the plan issues, padding included) and the useful TFLOP/s (2 x N x Ho x Wo x Cout x k^2 x Cin/grp flops of the
dense layer; not given for the LUT + gather kernels), the plan, and the card name, power limit and maximum SM clock.

    python tools/conv_ab.py [--layers conv1,conv2,conv3,conv4,conv5] [--batches 1,4,40,256,1024] [--rounds 7]
                            [--iters 20] [--out conv_ab.json]
    python tools/conv_ab.py --layers vgg_conv1_1,vgg_conv1_2 --batches 1,64,256
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

# name: (Hi, Wi, Cin, Cout, k, pad, stride, groups, S, K, d) -- the AlexNet layers of bench.py, VGG16's block 1 with the
# subspaces of tests/test_oracle_vgg16.py
LAYERS = {
    "conv1": (227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8),
    "conv2": (27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8),
    "conv3": (13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8),
    "conv4": (13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8),
    "conv5": (13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8),
    "vgg_conv1_1": (224, 224, 3, 64, 3, 1, 1, 1, 1, 128, 4),
    "vgg_conv1_2": (224, 224, 64, 64, 3, 1, 1, 1, 8, 128, 8),
}
# the two sides of a layer: name -> (tensor_core, force_kernel or None)
FAMILIES = {"conv_ws": (2, 7), "pq_gemm_tc": (2, 6)}
LUT_RIVAL = {"vgg_conv1_1": {"conv_ws": (2, 7), "lut_gather": (0, None)}}


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
    if not m:
        return None   # (LUT + gather: no tensor-core GEMM)
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
    fams = LUT_RIVAL.get(name, FAMILIES)
    lay = {}
    for fam, (tc, kern) in fams.items():
        lay[fam] = q.ConvLayer(ctx, Cin, Hi, Wi, Cout, k, pad, stride, G, ctrd, asmt, bias)
        lay[fam].set_param("tensor_core", tc)
        if kern is not None:
            lay[fam].set_param("force_kernel", kern)
    ho, wo, co = lay["conv_ws"].out_dims()
    stream = torch.cuda.current_stream()
    res[name] = {}
    for N in batches:
        x = torch.from_numpy((np.abs(rng.randn(N, Hi, Wi, Cin)) * 20).astype(np.float32)).cuda()
        y = torch.empty((N, ho, wo, co), dtype=torch.float32, device="cuda")
        useful = 2.0 * N * ho * wo * co * k * k * (Cin // G)

        def launch(L):
            q._check(q.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(x.data_ptr()), N, ctypes.c_void_p(y.data_ptr()), 1,
                                                  ctypes.c_void_p(stream.cuda_stream)))
        plans, times = {}, {fam: [] for fam in fams}
        for r in range(args.rounds + 1):
            for kern in fams:
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
        for fam in fams:
            s = stats(times[fam])
            em = executed_macs(plans[fam])
            out[fam] = dict(ms=s, executed_TFLOPs=2.0 * em / (s["median"] * 1e-3) / 1e12 if em else None,
                            useful_TFLOPs=useful / (s["median"] * 1e-3) / 1e12, plan=plans[fam])
            print("%s N=%-5d %-11s %8.4f ms (%.4f - %.4f)  executed %s TFLOP/s  useful %6.1f TFLOP/s  %s"
                  % (name, N, fam, s["median"], s["min"], s["max"],
                     "%6.1f" % out[fam]["executed_TFLOPs"] if em else "     -", out[fam]["useful_TFLOPs"],
                     plans[fam].split(" smem")[0]), flush=True)
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
