#!/usr/bin/env python
"""AlexNet's FC layers alone (bf16x2 operands, byte table): the weight-stationary GEMM fc_ws (fc_ws = 1) against the
decode-at-use pq_gemm_tc mode 2 (fc_ws = 0), in one process on one GPU.

For every layer and batch size the two sides alternate, round by round; a round is `iters` back-to-back launches between
CUDA events (each launch includes the plane-image prep and, with a K-split, the reduction).  Each side is a layer object
of its own with the same parameters.  Per side the tool prints the median and min-max of the per-launch time over the
rounds, the executed tensor-core TFLOP/s (every MMA the plan issues, padding included) and the useful TFLOP/s
(2 x N x Din x Dout flops of the dense layer), the plan, and the card name, power limit and maximum SM clock.

    python tools/fc_ab.py [--layers fc6,fc7,fc8] [--batches 96,128,256,1024] [--rounds 7] [--iters 20] [--out fc_ab.json]
"""
import argparse
import ctypes
import importlib
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from conv_ab import card, stats  # noqa: E402

# name: (Din, Dout, S, K, d, NHWC source map or None) -- the AlexNet layers of bench.py
LAYERS = {
    "fc6": (9216, 4096, 2304, 32, 4, (6, 6, 256)),
    "fc7": (4096, 4096, 1024, 32, 4, None),
    "fc8": (4096, 1000, 4096, 16, 1, None),
}
SIDES = {"fc_ws": 1, "pq_gemm_tc_mode2": 0}


def executed_macs(desc):
    """Tensor-core MACs one launch issues, from the plan string (two bf16 MMAs of K = 16 per k-step)."""
    m = re.search(r"pq_gemm_tc_ws\(.*? N=(\d+) images=(\d+) .*?grid=(\d+) .*?ksteps=(\d+)", desc)
    if m:
        n, p, grid, ks = (float(v) for v in m.groups())
        return grid * ks * 2 * 16 * p * n
    m = re.search(r"pq_gemm_tc\(.*?NT=(\d+) .*?grid=(\d+) .*?ksteps=(\d+)", desc)
    if not m:
        return None
    nt, grid, ks = (float(v) for v in m.groups())
    return grid * ks * 2 * 16 * 128 * nt


def run_layer(q, ctx, name, batches, args, rng, res):
    import torch
    Din, Dout, S, K, d, nhwc = LAYERS[name]
    ctrd = (rng.randn(S, K, d) / np.sqrt(Din)).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    lay = {}
    for side, ws in SIDES.items():
        lay[side] = q.FcLayer(ctx, Din, ctrd, asmt, bias)
        if nhwc:
            lay[side].set_src_nhwc(*nhwc)
        lay[side].set_param("tensor_core", 2)
        lay[side].set_param("fc_ws", ws)
    stream = torch.cuda.current_stream()
    res[name] = {}
    for N in batches:
        x = torch.from_numpy((np.abs(rng.randn(N, Din)) * 4).astype(np.float32)).cuda()
        y = torch.empty((N, Dout), dtype=torch.float32, device="cuda")
        useful = 2.0 * N * Din * Dout

        def launch(L):
            q._check(q.lib.qcnn_fc_aprx_forward(L.h, ctypes.c_void_p(x.data_ptr()), N, ctypes.c_void_p(y.data_ptr()), 1,
                                                ctypes.c_void_p(stream.cuda_stream)))
        plans, times = {}, {side: [] for side in SIDES}
        for r in range(args.rounds + 1):
            for side in SIDES:
                if r == 0:
                    launch(lay[side])          # scratch buffers sized for this batch outside the timed rounds
                    torch.cuda.synchronize()
                    plans[side] = lay[side].describe(N)
                    continue
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    launch(lay[side])
                b.record()
                torch.cuda.synchronize()
                times[side].append(a.elapsed_time(b) / args.iters)
        out = {}
        for side in SIDES:
            s = stats(times[side])
            em = executed_macs(plans[side])
            out[side] = dict(ms=s, executed_TFLOPs=2.0 * em / (s["median"] * 1e-3) / 1e12 if em else None,
                             useful_TFLOPs=useful / (s["median"] * 1e-3) / 1e12, plan=plans[side])
            print("%s N=%-5d %-17s %8.4f ms (%.4f - %.4f)  executed %s TFLOP/s  useful %6.1f TFLOP/s  %s"
                  % (name, N, side, s["median"], s["min"], s["max"],
                     "%6.1f" % out[side]["executed_TFLOPs"] if em else "     -", out[side]["useful_TFLOPs"],
                     plans[side].split(" via ")[-1].split(" smem")[0]), flush=True)
        res[name][str(N)] = out
        del x, y
        torch.cuda.empty_cache()
    for L in lay.values():
        L.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", default="fc6,fc7,fc8")
    ap.add_argument("--batches", default="96,128,256,1024")
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
