#!/usr/bin/env python
"""Where the time of the persistent FC kernel (csrc/fc_chain.cu) goes: per-CTA clock64 stamps after every phase of every
layer, with and without an L2 flush before the launch.  AlexNet fc6/fc7/fc8 shapes, random parameters.

    python tools/fc_chain_phases.py [--reps 10]
"""
import argparse
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PH = ["x-slice", "lut", "chunk0", "gather", "publish"]


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--mhz", type=float, default=1980.0, help="SM clock the cycle stamps are converted with (H100 maximum: 1980)")
    args = ap.parse_args()
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    rng = np.random.RandomState(0)
    shapes = [(9216, 4096, 2304, 32, 4), (4096, 4096, 1024, 32, 4), (4096, 1000, 4096, 16, 1)]
    layers = []
    for (Din, Dout, S, K, d) in shapes:
        layers.append(q.FcLayer(ctx, Din, (rng.randn(S, K, d) * 0.02).astype(np.float32),
                                rng.randint(0, K, size=(Dout, S)).astype(np.uint8), (rng.randn(Dout) * 0.1).astype(np.float32)))
    G = ctx.sm_count
    stamps = torch.zeros(32 * G, dtype=torch.int64, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    cfgs = [("fc6+fc7+fc8", layers, [1, 1, 0], 9216), ("fc6", layers[:1], [1], 9216), ("fc7", layers[1:2], [1], 4096),
            ("fc8", layers[2:], [0], 4096)]
    for name, ls, relu, din in cfgs:
        x = torch.rand((1, din), dtype=torch.float32, device="cuda")
        for do_flush in (True, False):
            rows = []
            for k in range(args.reps):
                stamps.zero_()
                if do_flush:
                    flush.fill_(k & 0xFF)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                q.fc_chain_forward(ls, relu, x, stamps=stamps)
                b.record()
                torch.cuda.synchronize()
                st = stamps.cpu().numpy().reshape(G, 32).astype(np.float64)
                rows.append((a.elapsed_time(b) * 1e3, st))
            rows = rows[2:]
            ev = np.median([r[0] for r in rows])
            st = rows[len(rows) // 2][1]
            span = (st[:, 1].max() - st[:, 0].min()) / 1e3
            skew = (st[:, 0].max() - st[:, 0].min()) / 1e3
            cyc = (st[:, 3] - st[:, 2])
            print("%-12s %s  event %.2f us  span(globaltimer) %.2f us  start skew %.2f us  CTA cycles med %.0f max %.0f (%.2f us)"
                  % (name, "L2 flushed" if do_flush else "L2 warm   ", ev, span, skew, np.median(cyc), cyc.max(), cyc.max() / args.mhz))
            for l in range(len(ls)):
                parts = []
                for i, ph in enumerate(PH):
                    t = (st[:, 4 + 5 * l + i] - st[:, 2]) / args.mhz
                    parts.append("%s %.2f/%.2f" % (ph, np.median(t), t.max()))
                print("    layer %d  (us since CTA start, median/max over CTAs): %s" % (l, "  ".join(parts)))
            tc = [(st[:, 19 + i] - st[:, 2]) / args.mhz for i in range(3)]
            print("    final reduction, thread 0 (us since CTA start, median/max): enter %.2f/%.2f  all words read %.2f/%.2f  "
                  "reduced %.2f/%.2f" % tuple(x for t in tc for x in (np.median(t), t.max())))
            arr = ["issued %.2f" % np.median((st[:, 23] - st[:, 2]) / args.mhz)]
            for i in range(8):
                t = (st[:, 24 + i] - st[:, 2]) / args.mhz
                if (st[:, 24 + i] > 0).all():
                    arr.append("c%d %.2f/%.2f" % (i, np.median(t), t.max()))
            print("    chunk arrival (us since CTA start, median/max): %s" % "  ".join(arr))
    for L in layers:
        L.close()
    ctx.close()


if __name__ == "__main__":
    main()
