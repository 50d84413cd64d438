"""Per-layer error of the conv kernel families against the CPU oracle (same metric as the parity tests).
    python tools/accuracy.py            # on an H100
"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def close(gpu, ref):
    gpu = np.asarray(gpu, np.float64)
    ref = np.asarray(ref, np.float64)
    scale = np.maximum(np.maximum(1.0, np.abs(ref)), 0.1 * np.abs(ref).max())
    return float((np.abs(gpu - ref) / scale).max()), float(np.abs(gpu - ref).max() / np.abs(ref).max())


def main():
    import torch
    import pyoracle as po
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    cases = [
        ("conv1", (2, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8), 60.0),
        ("conv2", (2, 27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8), 20.0),
        ("conv3", (2, 13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8), 20.0),
        ("conv4", (2, 13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8), 20.0),
        ("conv5", (2, 13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8), 20.0),
    ]
    for name, case, scale in cases:
        N, Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d = case
        rng = np.random.RandomState(5)
        ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
        asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
        bias = (rng.randn(Cout) * 0.1).astype(np.float32)
        x = (rng.randn(N, Hi, Wi, Cin) * scale).astype(np.float32) if name == "conv1" else \
            (np.abs(rng.randn(N, Hi, Wi, Cin)) * scale).astype(np.float32)
        L = po.conv(pad, k, Cout, G, stride)
        ref = po.conv_aprx(x, L, ctrd, asmt, bias)
        xd = torch.from_numpy(x).cuda()
        for fam in ("0", "1", "2", "4", "5", "6"):
            os.environ["QCNN_FORCE_KERNEL"] = fam
            layer = q.ConvLayer(ctx, Cin, Hi, Wi, Cout, k, pad, stride, G, ctrd, asmt, bias)
            desc = layer.describe(N).split(" ")[0]
            y = layer.forward(xd).cpu().numpy()
            e1, e2 = close(y, ref)
            print("%s family %s (%s): test metric %.3g, max|d|/max|ref| %.3g, max|ref| %.3g" % (name, fam, desc[:24], e1, e2, np.abs(ref).max()))
            layer.close()
    os.environ.pop("QCNN_FORCE_KERNEL", None)
    # FC: gather kernel (explicit nsplit) vs tensor-core path at N = 128
    for name, (Din, Dout, S, K, d) in (("fc6", (9216, 4096, 2304, 32, 4)), ("fc7", (4096, 4096, 1024, 32, 4)), ("fc8", (4096, 1000, 4096, 16, 1))):
        rng = np.random.RandomState(6)
        N = 128
        ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
        asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
        bias = (rng.randn(Dout) * 0.1).astype(np.float32)
        x = (np.abs(rng.randn(N, Din)) * 20.0).astype(np.float32)
        ref = po.fc_aprx(x, ctrd, asmt, bias)
        layer = q.FcLayer(ctx, Din, ctrd, asmt, bias)
        xd = torch.from_numpy(x).cuda()
        y = layer.forward(xd).cpu().numpy()
        print("%s tensor-core path: test metric %.3g, rel-to-max %.3g" % ((name,) + close(y, ref)))
        layer.set_param("fc_nsplit", 4)
        y = layer.forward(xd).cpu().numpy()
        print("%s gather kernel nsplit=4: test metric %.3g, rel-to-max %.3g" % ((name,) + close(y, ref)))
        layer.close()


if __name__ == "__main__":
    main()
