"""BASELINE.json configs[4]: per-layer synthetic sweep of the conv2..conv5 PQ kernels.
subspaces per group S in {4, 8, 16} (d = Cg / S), codebook size K in {64, 128, 256}, batch N in {1, 256};
reports time (CUDA events, median of reps), achieved GB/s on the algorithmic bytes of SURVEY.md 8(d) against the
measured HBM peak, lookups/s against the shared-memory gather bound and -- when the layer ran as a decode-at-use GEMM --
the executed tensor-core TFLOP/s.  EVERY row (N = 1 and N = 256) is checked against the CPU oracle (tolerance of the
path; both error metrics of tests/test_gpu_parity_b256.py are recorded).
    python tools/sweep.py [--reps 5] [--strict] [--out sweep.csv]
--strict: tensor_core = 0 (LUT + gather kernels only)
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEOM = {  # name: (Hi, Cin, Cout, k, pad, G)   SURVEY.md 8(d) config 5
    "conv2": (27, 96, 256, 5, 2, 2),
    "conv3": (13, 256, 384, 3, 1, 1),
    "conv4": (13, 384, 384, 3, 1, 2),
    "conv5": (13, 384, 256, 3, 1, 2),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="sweep.csv")
    ap.add_argument("--no-check", action="store_true")
    ap.add_argument("--strict", action="store_true")
    args = ap.parse_args()
    import torch
    q = importlib.import_module("quantized-cnn_b200")
    from oracle import pyoracle as po      # checker only
    ctx = q.Context(0)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except (OSError, ValueError):
        pass
    # without MEASURED_PEAKS.json: H100 SXM data sheet (3350 GB/s of HBM3) and the H100's maximum SM clock
    hbm = float(peaks.get("hbm_gbs", 3350.0))
    hbm_src = "MEASURED_PEAKS.json" if "hbm_gbs" in peaks else "H100 SXM data sheet, not measured"
    gather_peak = 32.0 * ctx.sm_count * float(peaks.get("sm_max_mhz", 1980.0)) * 1e6
    import re
    tol = 1e-4 if args.strict else 3e-4
    from concurrent.futures import ThreadPoolExecutor
    workers = max(1, min(32, (os.cpu_count() or 2) - 1))
    rows = ["layer,S_per_group,K,d,N,ms,alg_MB,alg_GBps,frac_hbm_peak,lookups_per_s,frac_smem_gather_bound,tensor_TFLOPs_executed,"
            "max_err_vs_oracle,max_err_e1,kernel"]
    for name, (Hi, Cin, Cout, k, pad, G) in GEOM.items():
        Cg = Cin // G
        for S in (4, 8, 16):
            d = Cg // S
            for K in (64, 128, 256):
                seed = sum(map(ord, name)) * 1000 + S * 10 + K // 64
                rng = np.random.RandomState(seed)
                ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
                asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
                bias = (rng.randn(Cout) * 0.1).astype(np.float32)
                layer = q.ConvLayer(ctx, Cin, Hi, Hi, Cout, k, pad, 1, G, ctrd, asmt, bias)
                if args.strict:
                    layer.set_param("tensor_core", 0)
                for N in (1, 256):
                    x = (np.abs(rng.randn(N, Hi, Hi, Cin)) * 20).astype(np.float32)
                    xd = torch.from_numpy(x).cuda()
                    y = layer.forward(xd)           # warm-up + tiling choice
                    torch.cuda.synchronize()
                    err = err1 = float("nan")
                    if not args.no_check:
                        Lr = po.conv(pad, k, Cout, G, 1)
                        with ThreadPoolExecutor(workers) as ex:      # ctypes releases the GIL: one image per thread
                            ref = np.concatenate(list(ex.map(lambda i: po.conv_aprx(x[i:i + 1], Lr, ctrd, asmt, bias), range(N))))
                        diff = np.abs(y.cpu().numpy().astype(np.float64) - ref)
                        scale = np.maximum(np.maximum(1.0, np.abs(ref)), 0.1 * np.abs(ref).max())
                        err = float((diff / scale).max())
                        err1 = float((diff / np.maximum(1.0, np.abs(ref))).max())
                        assert err <= tol, (name, S, K, N, err)
                    ms = []
                    for _ in range(args.reps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        layer.forward(xd)
                        e1.record()
                        torch.cuda.synchronize()
                        ms.append(e0.elapsed_time(e1))
                    t = float(np.median(ms))
                    w = layer.work(N)
                    full = layer.describe(N)
                    desc = full.split(" ")[0].split("(")[0]
                    m = re.search(r"pq_gemm_tc.*?NT=(\d+).*?grid=(\d+).*?ksteps=(\d+)", full)
                    tfl = 2.0 * float(m.group(2)) * float(m.group(3)) * (2 * 16 if "bf16x2" in full else 3 * 8) * 128 * float(m.group(1)) / (t * 1e-3) / 1e12 if m else 0.0
                    rows.append("%s,%d,%d,%d,%d,%.4f,%.2f,%.1f,%.4f,%.3e,%.4f,%.1f,%.2e,%.2e,%s" % (
                        name, S, K, d, N, t, w["alg_bytes"] / 1e6, w["alg_bytes"] / (t * 1e-3) / 1e9,
                        w["alg_bytes"] / (t * 1e-3) / 1e9 / hbm, w["lookups"] / (t * 1e-3),
                        w["lookups"] / (t * 1e-3) / gather_peak, tfl, err, err1, desc))
                    print(rows[-1], flush=True)
                layer.close()
    with open(args.out, "w") as f:
        f.write("# BASELINE.json configs[4] sweep; HBM peak %.1f GB/s (%s), smem-gather bound %.3e lookups/s\n" % (hbm, hbm_src, gather_peak))
        f.write("\n".join(rows) + "\n")


if __name__ == "__main__":
    main()
