"""Times the k-means product quantizer (qcnn_pq_quantize_conv / _fc / _model) on AlexNet- and VGG16-shaped seeded
Gaussian dense weights at the (K, d) of the shipped AlexNet files and of the VGG16 table of tests/test_oracle_vgg16.py.
Per layer: the device time of the quantizer's kernels (torch.profiler, CUDA activities; H2D / D2H copies and the host
side excluded), median of 3 runs, and the relative reconstruction error ||W - W^|| / ||W||.  Then the wall time of
qcnn_pq_quantize_model for AlexNet, file I/O included.  Prints the card, its power limit and max SM clock.
    python tools/pq_quantize_time.py [--iters 20] [--model AlexNet VGG16]"""
import argparse
import importlib
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def tables(po):
    """model -> [(layerInd, 'conv' | 'fc', weight shape, K, d)]"""
    from test_oracle_vgg16 import VGG16_IN, vgg16_layers, vgg16_pq
    out = {}
    for name, layers, chw, pq in (("AlexNet", po.alexnet_layers(), po.ALEXNET_IN, {l: v[1:] for l, v in po.ALEXNET_PQ.items()}),
                                  ("VGG16", vgg16_layers(po), VGG16_IN, None)):
        if pq is None:
            pq = {l: v[1:] for l, v in vgg16_pq(layers).items()}
        shapes = po.infer_shapes(layers, chw)
        rows = []
        for l, L in enumerate(layers):
            h, w, c = shapes[l]
            if L["type"] == po.CONV:
                rows.append((l, "conv", (L["cnt"], c // L["grp"], L["k"], L["k"])) + tuple(pq[l]))
            elif L["type"] == po.FCNT:
                rows.append((l, "fc", (L["nod"], h * w * c)) + tuple(pq[l]))
        out[name] = rows
    return out


def dense(shape, seed):
    fan = int(np.prod(shape[1:]))
    return np.random.default_rng(seed).standard_normal(shape, dtype=np.float32) * np.float32(1.0 / np.sqrt(fan))


def decode(ctrd, asmt, cin):
    S, K, d = ctrd.shape
    g = ctrd[np.arange(S), asmt]
    g = g.reshape(g.shape[:-2] + (S * d,))[..., :cin]
    return np.moveaxis(g, -1, 1) if g.ndim == 4 else g


def kernel_ms(prof):
    tot = 0.0
    for e in prof.key_averages():
        if "pq_" in e.key:   # the quantizer's kernels; copies are named Memcpy
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    return tot / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--model", nargs="+", default=["AlexNet", "VGG16"])
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle import pyoracle as po
    q = importlib.import_module("quantized-cnn_b200")
    if not torch.cuda.is_available():
        sys.exit("pq_quantize_time.py needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print("card: %s" % (smi[0] if smi else torch.cuda.get_device_name(0)))
    ctx = q.Context(0)
    tabs = tables(po)
    for model in args.model:
        print("\n%s, iters=%d: per-layer device time of the quantizer kernels (median of %d) and ||W - W^|| / ||W||"
              % (model, args.iters, args.reps))
        total = 0.0
        for l, kind, shape, K, d in tabs[model]:
            w = dense(shape, 1000 + l)
            fn = q.pq_quantize_conv if kind == "conv" else q.pq_quantize_fc
            fn(ctx, w, K, d, iters=1)   # warm-up: module load, shared-memory opt-in
            times = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    ctrd, asmt, sse = fn(ctx, w, K, d, iters=args.iters)
                    torch.cuda.synchronize()
                times.append(kernel_ms(prof))
            ms = float(np.median(times))
            total += ms
            err = np.linalg.norm((w - decode(ctrd, asmt, shape[1])).ravel()) / np.linalg.norm(w.ravel())
            print("  layer %2d %-4s %-22s K=%3d d=%2d  %8.3f ms  rel.err %.4f  sse %.4g -> %.4g"
                  % (l, kind, "x".join(map(str, shape)), K, d, ms, err, sse[0], sse[-1]))
        print("  total %.2f ms" % total)
    if "AlexNet" in args.model:
        tmp = tempfile.mkdtemp(prefix="qcnn_pqq_")
        try:
            src, out = os.path.join(tmp, "dense"), os.path.join(tmp, "out")
            os.makedirs(src)
            os.makedirs(out)
            pq = {}
            for l, kind, shape, K, d in tabs["AlexNet"]:
                po.write_bin(os.path.join(src, "a.%s.%02d.bin" % ("convKnl" if kind == "conv" else "fcntWei", l + 1)),
                             dense(shape, 1000 + l))
                po.write_bin(os.path.join(src, "a.biasVec.%02d.bin" % (l + 1)), np.zeros(shape[0], np.float32))
                pq[l] = (K, d)
            walls = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                q.pq_quantize_model(ctx, "AlexNet", src, "a", out, "q", pq, iters=args.iters)
                walls.append(time.perf_counter() - t0)
            print("\nqcnn_pq_quantize_model AlexNet, iters=%d, wall time incl. file I/O: median %.2f s (runs: %s)"
                  % (args.iters, float(np.median(walls)), ", ".join("%.2f" % t for t in walls)))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    ctx.close()


if __name__ == "__main__":
    main()
