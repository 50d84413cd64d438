"""Per-layer CUDA-event times + chosen tilings of a PQ net at a given batch size: AlexNet (the benchmark's files) or
VGG16 (seeded synthetic parameters, the table and scales of tests/test_oracle_vgg16.py).
    python tools/layer_times.py --batch 1 [--reps 50] [--model VGG16]"""
import argparse
import importlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--tc", type=int, default=-1, help="tensor_core parameter for every PQ layer (0 strict, 1 3xTF32, 2 bf16x2)")
    ap.add_argument("--model", default="AlexNet", choices=("AlexNet", "VGG16"))
    args = ap.parse_args()
    import torch
    q = importlib.import_module("quantized-cnn_b200")
    B = args.batch
    tmp = tempfile.mkdtemp(prefix="qcnn_lt_")
    if args.model == "VGG16":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from oracle import pyoracle
        from test_oracle_vgg16 import synth_vgg16, vgg16_images
        _, params = synth_vgg16(pyoracle, seed=16)
        pyoracle.save_model(tmp, "vgg", params)
        d, pfx = tmp, "vgg"
        imgs = vgg16_images(B, 2016)
    else:
        d, pfx, what = bench.model_files(q, tmp)
        imgs = bench.lcg_images(B, 12345)
    ctx = q.Context(0)
    net = q.Net(ctx, d, pfx, args.model)
    if args.tc >= 0:
        for l in range(net.layer_count):
            if net.pq_layer(l) is not None:
                net.pq_layer(l).set_param("tensor_core", args.tc)
    img = torch.from_numpy(imgs).cuda()
    prob = torch.empty((B, 1000), dtype=torch.float32, device="cuda")
    for _ in range(5):
        net.forward(img, prob=prob)
    torch.cuda.synchronize()
    # whole-pass time without per-layer events
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        net.forward(img, prob=prob)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.reps
    print("%s batch %d: %.4f ms / forward, %.1f images/s (%d launches); %s" % (args.model, B, ms, B / ms * 1e3,
                                                                          net.launch_count(), torch.cuda.get_device_name(0)))
    net.set_profiling(True)
    acc = np.zeros(net.layer_count)
    for _ in range(args.reps):
        net.forward(img, prob=prob)
        torch.cuda.synchronize()
        acc += np.array([net.layer_time_ms(l) for l in range(net.layer_count)])
    acc /= args.reps
    for l in range(net.layer_count):
        if acc[l] > 0:
            pl = net.pq_layer(l)
            print("  layer %2d  %8.4f ms  %s" % (l, acc[l], pl.describe(B) if pl is not None else ""))
    print("  sum of layers %.4f ms" % acc.sum())
    net.close()
    ctx.close()


if __name__ == "__main__":
    main()
