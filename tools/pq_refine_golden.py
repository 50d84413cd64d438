"""Writes tests/golden/pq_refine_conv_bits.npz: the results (ctrd, asmt, loss) of qcnn_pq_refine_conv and
qcnn_pq_refine_conv_target on seeded layers, so that later builds can be checked bit for bit against the build that
wrote them (tests/test_gpu_pq_stats.py).  The inputs are seeded numpy arrays (maps, targets, weights and a random
start), so they are reproduced exactly from the row table below; the results are those of one NVIDIA H100.
    python tools/pq_refine_golden.py [--root TREE] [--out tests/golden/pq_refine_conv_bits.npz]"""
import argparse
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed): padding, groups with a partial subspace, stride 4 with 3
# input channels, and AlexNet conv1 over two runs of positions
ROWS = [
    ("3x3_grp2_partial", 20, 9, 32, 3, 1, 1, 2, 16, 4, 3, 21),
    ("5x5_s2_p2", 12, 11, 24, 5, 2, 2, 1, 32, 4, 4, 21),
    ("conv1_like", 3, 63, 32, 11, 0, 4, 1, 128, 8, 6, 21),
    ("conv1_two_runs", 3, 227, 96, 11, 0, 4, 1, 32, 8, 70, 21),
]
SWEEPS = 2


def inputs(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed):
    """weights [Cout][Cg][k][k], maps NHWC, targets NHWC and a start (ctrd, asmt), all seeded numpy"""
    rng = np.random.RandomState(seed)
    Cg, S = Cin // grp, -(-(Cin // grp) // d)
    Ho = (H + 2 * pad - k) // stride + 1
    W = (rng.randn(Cout, Cg, k, k) / np.sqrt(Cg * k * k)).astype(np.float32)
    X = rng.randn(N, H, H, Cin).astype(np.float32)
    T = rng.randn(N, Ho, Ho, Cout).astype(np.float32)
    ctrd = (0.3 * rng.randn(S, K, d) / np.sqrt(Cg * k * k)).astype(np.float32)
    for m in range(S):
        ctrd[m, :, min(d, Cg - m * d):] = 0
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    return W, X, T, ctrd, asmt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT, help="tree to load quantized-cnn_b200 (and its library) from")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "pq_refine_conv_bits.npz"))
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    out = {}
    for name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed in ROWS:
        W, X, T, ctrd, asmt = inputs(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
        x, t = torch.from_numpy(X).cuda(), torch.from_numpy(T).cuda()
        c, a, loss = q.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=SWEEPS)
        ct, at, losst = q.pq_refine_conv_target(ctx, x, t, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=SWEEPS)
        out.update({name + "/ctrd": c, name + "/asmt": a, name + "/loss": loss,
                    name + "/target_ctrd": ct, name + "/target_asmt": at, name + "/target_loss": losst})
        print(name, loss, losst)
    np.savez_compressed(args.out, **out)
    ctx.close()


if __name__ == "__main__":
    main()
