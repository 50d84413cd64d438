"""Times the damped copies of PqStats.refine_damped (DESIGN.md 4e, "Damping toward the original weights") for AlexNet
conv1 and fc6: a target object holding one add of a seeded Gaussian batch, then refine_damped at sweeps = 0 in the target
form, without and with the bias (the raw sums copied and damped, or the centered copies damped in place).  Per layer and
form, from one call under torch.profiler (CUDA activities) after a warm-up call: the duration of every damping kernel
(pqr_damp_lambda_kernel, pqr_damp_kernel, pqr_damp_tt_kernel, and the |W_g|^2 sums of pqr_sqnorm_*), the copy of the raw
sums and the upload of the weights, next to the median wall time of the damped and the undamped call over --reps calls.
Prints the card, its power limit and max SM clock.
    python tools/pq_damp_time.py [--reps 5] [--out f.json]"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pq_refine_time import card   # noqa: E402

LAYERS = {   # name: FC (Din, Dout, K, d, N) or conv (Cin, H, Cout, k, pad, stride, grp, K, d, N)
    "alexnet_conv1": (3, 227, 96, 11, 0, 4, 1, 32, 4, 16),
    "alexnet_fc6": (9216, 4096, 16, 8, 256),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--damp", type=float, default=1e-2)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "needs a GPU"
    q = importlib.import_module("quantized-cnn_b200")
    print("card: %s (name, power limit, max SM clock)" % card())
    ctx = q.Context(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    rng = np.random.RandomState(2)
    rows = []
    for name, geo in LAYERS.items():
        if len(geo) == 5:
            Din, Dout, K, d, N = geo
            y = torch.randn((N, Din), generator=g, device="cuda")
            t = torch.randn((N, Dout), generator=g, device="cuda")
            st = q.PqStats.fc(ctx, Din, Dout, d, target=True)
            W = rng.randn(Dout, Din).astype(np.float32)
            S, asmt_shape = -(-Din // d), (Dout, -(-Din // d))
        else:
            Cin, H, Cout, k, pad, stride, grp, K, d, N = geo
            Ho = (H + 2 * pad - k) // stride + 1
            y = torch.randn((N, H, H, Cin), generator=g, device="cuda")
            t = torch.randn((N, Ho, Ho, Cout), generator=g, device="cuda")
            st = q.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
            W = rng.randn(Cout, Cin // grp, k, k).astype(np.float32)
            S = -(-(Cin // grp) // d)
            asmt_shape = (Cout, k, k, S)
        st.add(y, t)
        ctrd = rng.randn(S, K, d).astype(np.float32)
        asmt = rng.randint(0, K, size=asmt_shape).astype(np.uint8)
        outputs = W.shape[0]
        bias = rng.randn(outputs).astype(np.float32)
        for bb in (None, bias):
            def damped():
                return st.refine_damped(W, ctrd, asmt, args.damp, target=True, bias=bb, sweeps=0)

            def plain():
                return st.refine_target(ctrd, asmt, sweeps=0) if bb is None else st.refine_target_bias(ctrd, asmt, bb, sweeps=0)

            walls = {}
            for key, fn in (("damped", damped), ("undamped", plain)):
                fn()   # warm-up
                torch.cuda.synchronize()
                w = []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    fn()
                    w.append(time.perf_counter() - t0)
                walls[key] = float(np.median(w)) * 1e3
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                damped()
                torch.cuda.synchronize()
            ev = [(e.name, (e.time_range.end - e.time_range.start) / 1e3) for e in prof.events()
                  if e.device_type == DeviceType.CUDA]
            kernels = {}
            for n, ms in ev:
                for key in ("pqr_damp_lambda_kernel", "pqr_damp_kernel", "pqr_damp_tt_kernel", "pqr_sqnorm"):
                    if key in n:
                        kernels[key] = kernels.get(key, 0.0) + ms
            copies = {k: sum(ms for n, ms in ev if key in n) for k, key in (("DtoD", "DtoD"), ("HtoD", "HtoD"))}
            form = "target" if bb is None else "target+bias"
            row = dict(layer=name, form=form, damp=args.damp, kernels_ms=kernels, copies_ms=copies,
                       damped_ms=walls["damped"], undamped_ms=walls["undamped"])
            rows.append(row)
            print("%-14s %-12s damping kernels %s; copies %s; call at sweeps=0: damped %.1f ms, undamped %.1f ms"
                  % (name, form, ", ".join("%s %.3f ms" % kv for kv in sorted(kernels.items())),
                     ", ".join("%s %.3f ms" % kv for kv in sorted(copies.items())), walls["damped"], walls["undamped"]))
        st.close()
        del y, t
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
