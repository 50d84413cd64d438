"""Times one add of a batch to target calibration statistics (PqStats.add with y and t) for AlexNet conv1, conv2 and fc6
at batch 256, seeded Gaussian y and t.  Per layer: the median wall time of an add (the NaN / Inf scan with its
synchronisation, then the folds, up to a device synchronise) over --reps adds after a warm-up one, and, from one add
under torch.profiler (CUDA activities), the sum of its kernel durations and of its first-moment kernels (pqr_colsum_kernel,
pqrc_tapsum_kernel).  --root loads the package (and so the library) from another tree, so that a build whose adds
form no first moments can be timed by the same script.  Prints the card, its power limit and max SM clock.
    python tools/pq_stats_add_time.py [--batch 256] [--reps 20] [--root TREE]"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pq_refine_time import card   # noqa: E402

LAYERS = {   # name: FC (Din, Dout, d) or conv (Cin, H, Cout, k, pad, stride, grp, d)
    "alexnet_conv1": (3, 227, 96, 11, 0, 4, 1, 4),
    "alexnet_conv2": (96, 27, 256, 5, 2, 1, 2, 8),
    "alexnet_fc6": (9216, 4096, 8),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--root", default=ROOT, help="tree to load quantized-cnn_b200 (and its library) from")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "needs a GPU"
    q = importlib.import_module("quantized-cnn_b200")
    print("library: %s" % q.LIB_PATH)
    print("card: %s (name, power limit, max SM clock)" % card())
    ctx = q.Context(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    N, rows = args.batch, []
    for name, geo in LAYERS.items():
        if len(geo) == 3:
            Din, Dout, d = geo
            y = torch.randn((N, Din), generator=g, device="cuda")
            t = torch.randn((N, Dout), generator=g, device="cuda")
            st = q.PqStats.fc(ctx, Din, Dout, d, target=True)
        else:
            Cin, H, Cout, k, pad, stride, grp, d = geo
            Ho = (H + 2 * pad - k) // stride + 1
            y = torch.randn((N, H, H, Cin), generator=g, device="cuda")
            t = torch.randn((N, Ho, Ho, Cout), generator=g, device="cuda")
            st = q.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
        st.add(y, t)   # warm-up
        torch.cuda.synchronize()
        walls = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            st.add(y, t)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.add(y, t)
            torch.cuda.synchronize()
        ev = [(e.name, e.time_range.end - e.time_range.start) for e in prof.events() if e.device_type == DeviceType.CUDA]
        total = sum(d for n, d in ev if "pqr" in n) / 1e3
        moments = sum(d for n, d in ev if "pqr_colsum" in n or "pqrc_tapsum" in n) / 1e3
        st.close()
        del y, t
        row = dict(layer=name, batch=N, add_ms=float(np.median(walls)) * 1e3, kernels_ms=total, first_moments_ms=moments)
        rows.append(row)
        print("%-14s batch %d: add %.2f ms (median of %d), kernels %.2f ms, of which first moments %.3f ms"
              % (name, N, row["add_ms"], args.reps, total, moments))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), root=os.path.abspath(args.root), rows=rows), f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
