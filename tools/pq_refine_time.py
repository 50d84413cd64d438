"""Times the error-correcting FC quantizer (qcnn_pq_refine_fc) on AlexNet fc6 / fc7 / fc8 (N = 4 Din inputs) and VGG16
fc6 (N = 8192) with seeded Gaussian weights (std 1/sqrt(Din)) and inputs, started from pq_quantize_fc (iters = 20) at
the shipped AlexNet (K, d).  Per layer, from one run under torch.profiler (CUDA activities): the Gram kernel's time, the
median per sweep of the sum of kernel durations (the sweeps are split at their loss kernels), how that splits between
the per-block cooperative kernel and the trailing GEMMs, achieved fp64 TFLOP/s from shape-based flop counts
(Gram: N Din (Din + 1), the useful lower triangle; sweep: 2 Dout Din^2, its GEMM work), and the loss trace.  Then, with
the profiler off, the wall time of a whole call.  Prints the card, its power limit and max SM clock.
The conv layers (qcnn_pq_refine_conv) of AlexNet (conv1-conv5, N = 64 images) and VGG16 (13 layers, N = 8) run at the
shipped AlexNet (K, d) and the VGG16 table of tests/test_oracle_vgg16.py (K = 128, d = 8; conv1_1 d = 4) on seeded
Gaussian maps and weights (std 1/sqrt(fan-in)), started from pq_quantize_conv (iters = 20).  Per layer: the time of
the patch and Gram kernels; per sweep (median) the sum of kernel durations split into the Cholesky (ridge, diagonal
blocks, panels, their trailing GEMMs, the solve), the assignment step, the response and GE GEMMs, and the building of
the joint system (member lists, M, b); fp64 TFLOP/s of the Gram (positions Dg (Dg + 1) per group), of the GEMMs
(2 Cout (sum_m (k^2 w_m)^2 + Dg^2)) and of the Cholesky ((K w_m)^3 / 3 per subspace, every cluster in use); the wall
time of a whole call with the profiler off.
With --target the same layers run the target form (qcnn_pq_refine_fc_target / _conv_target) on targets
t = (the layer's response) + 0.3 (a seeded Gaussian), and each layer also reports the cross-product GEMM P = T^T Y next
to the Gram, with its fp64 TFLOP/s (2 N Din Dout for FC, 2 positions Cout Cg k^2 for conv).
The conv Gram and cross product read the patches straight from the maps; a library that builds them with an im2col
kernel (pqrc_patch_kernel) has that kernel counted with the Gram, so two builds compare.  --digest prints the sha256 of
every layer's (ctrd, asmt, loss) bytes, and --root loads the package (and so the library) from another tree, so that
one script checks two builds for identical results:
    python tools/pq_refine_time.py [--sweeps 3] [--target] [--digest] [--root TREE] [--layers alexnet_fc6 ...]"""
import argparse
import hashlib
import importlib
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LAYERS = {   # name: (Din, Dout, K, d, N)
    "alexnet_fc6": (9216, 4096, 32, 4, 4 * 9216),
    "alexnet_fc7": (4096, 4096, 32, 4, 4 * 4096),
    "alexnet_fc8": (4096, 1000, 16, 1, 4 * 4096),
    "vgg16_fc6": (25088, 4096, 32, 4, 8192),
}
CONV_LAYERS = {   # name: (Cin, H, Cout, k, pad, stride, grp, K, d, N)
    "alexnet_conv1": (3, 227, 96, 11, 0, 4, 1, 128, 8, 64),
    "alexnet_conv2": (96, 27, 256, 5, 2, 1, 2, 128, 8, 64),
    "alexnet_conv3": (256, 13, 384, 3, 1, 1, 1, 128, 8, 64),
    "alexnet_conv4": (384, 13, 384, 3, 1, 1, 2, 128, 8, 64),
    "alexnet_conv5": (384, 13, 256, 3, 1, 1, 2, 128, 8, 64),
}
for _i, (_cin, _cout, _h) in enumerate([(3, 64, 224), (64, 64, 224), (64, 128, 112), (128, 128, 112), (128, 256, 56),
                                        (256, 256, 56), (256, 256, 56), (256, 512, 28), (512, 512, 28), (512, 512, 28),
                                        (512, 512, 14), (512, 512, 14), (512, 512, 14)]):
    _blk, _n = [(1, 1), (1, 2), (2, 1), (2, 2), (3, 1), (3, 2), (3, 3), (4, 1), (4, 2), (4, 3), (5, 1), (5, 2), (5, 3)][_i]
    CONV_LAYERS["vgg16_conv%d_%d" % (_blk, _n)] = (_cin, _h, _cout, 3, 1, 1, 1, 128, 4 if _cin == 3 else 8, 8)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def kernels(prof):
    """(name, start us, duration us) of every CUDA kernel of the trace, in start order"""
    from torch.autograd import DeviceType
    ev = [(e.name, e.time_range.start, e.time_range.end - e.time_range.start) for e in prof.events()
          if e.device_type == DeviceType.CUDA and ("pqr_" in e.name or "pqrc_" in e.name)]
    return sorted(ev, key=lambda x: x[1])


def gemm_mode(name):
    """pqr_gemm_kernel's template argument (0: fp64 GEMM, 1: Gram, 2: cross product, 3 / 4: the Gram / cross product
    on an NHWC map), or None for another kernel"""
    m = re.search(r"pqr_gemm_kernel<(?:\(int\))?(\d)>", name)
    return int(m.group(1)) if m else None


def loss_ends(ev):
    """indices of the loss kernels that close the start and every sweep (not the |T|^2 reduction's final kernel)"""
    return [i for i, (n, _, _) in enumerate(ev) if "pqr_loss_final" in n and not (i > 0 and "pqr_sqnorm" in ev[i - 1][0])]


def digest(res):
    """sha256 of the (ctrd, asmt, loss) bytes of one call"""
    h = hashlib.sha256()
    for a in res:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def time_conv(q, ctx, name, sweeps, target):
    import torch
    import torch.nn.functional as F
    from torch.profiler import ProfilerActivity, profile
    Cin, H, Cout, k, pad, stride, grp, K, d, N = CONV_LAYERS[name]
    Cg = Cin // grp
    W = np.random.default_rng(1).standard_normal((Cout, Cg, k, k), dtype=np.float32) / np.float32(np.sqrt(Cg * k * k))
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((N, H, H, Cin), generator=g, device="cuda", dtype=torch.float32)
    c0, a0, _ = q.pq_quantize_conv(ctx, W, K, d, iters=20, seed=3)
    if target:
        tg = F.conv2d(x.permute(0, 3, 1, 2), torch.from_numpy(W).cuda(), stride=stride, padding=pad, groups=grp)
        tg = tg.permute(0, 2, 3, 1).contiguous()
        tg += 0.3 * torch.randn(tg.shape, generator=g, device="cuda", dtype=torch.float32)
        run = lambda xx, tt, s: q.pq_refine_conv_target(ctx, xx, tt, c0, a0, k, pad=pad, stride=stride, grp=grp, sweeps=s)
    else:
        tg = x
        run = lambda xx, tt, s: q.pq_refine_conv(ctx, W, xx, c0, a0, pad=pad, stride=stride, grp=grp, sweeps=s)
    run(x[:1], tg[:1], 1)   # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, _, loss = run(x, tg, sweeps)
        torch.cuda.synchronize()
    ev = kernels(prof)
    gram = sum(t for n, _, t in ev if gemm_mode(n) in (1, 3) or "pqrc_patch" in n)
    cross = sum(t for n, _, t in ev if gemm_mode(n) in (2, 4))
    ends = loss_ends(ev)
    split = dict(chol=[], assign=[], gemm=[], system=[], total=[])
    for a, b in zip(ends[:-1], ends[1:]):
        part, in_chol = ev[a + 1:b + 1], False
        acc = dict.fromkeys(split, 0.0)
        for n, _, t in part:
            if "pqrc_ridge" in n:
                in_chol = True
            if in_chol or "pqrc_solve" in n:
                acc["chol"] += t
            elif "pqrc_assign" in n or "pqrc_ccost" in n:
                acc["assign"] += t
            elif gemm_mode(n) == 0:
                acc["gemm"] += t
            elif "pqr_loss" not in n:
                acc["system"] += t
            if "pqrc_solve" in n:
                in_chol = False
            acc["total"] += t
        for key in split:
            split[key].append(acc[key])
    med = {key: float(np.median(v)) / 1e3 for key, v in split.items()}
    t0 = time.perf_counter()
    res = run(x, tg, sweeps)
    wall = time.perf_counter() - t0
    Ho = (H + 2 * pad - k) // stride + 1
    T, Dg, S = k * k, Cg * k * k, -(-Cg // d)
    ws = [min(d, Cg - m * d) for m in range(S)]
    gram_flop = grp * N * Ho * Ho * Dg * (Dg + 1)
    gemm_flop = 2.0 * Cout * (sum((T * w) ** 2 for w in ws) + Dg * Dg)
    chol_flop = sum((K * w) ** 3 / 3.0 for w in ws)
    r = dict(layer=name, Cin=Cin, H=H, Cout=Cout, k=k, pad=pad, stride=stride, grp=grp, K=K, d=d, N=N,
             gram_ms=gram / 1e3, gram_tflops=gram_flop / (gram * 1e-6) / 1e12,
             sweep_ms=med["total"], sweep_chol_ms=med["chol"], sweep_assign_ms=med["assign"], sweep_gemm_ms=med["gemm"],
             sweep_system_ms=med["system"], gemm_tflops=gemm_flop / (med["gemm"] * 1e-3) / 1e12,
             chol_tflops=chol_flop / (med["chol"] * 1e-3) / 1e12, call_wall_s=wall,
             loss=[float(v) for v in loss], loss_ratio=float(loss[-1] / loss[0]), target=target, digest=digest(res))
    if target:
        r.update(cross_ms=cross / 1e3, cross_tflops=2.0 * N * Ho * Ho * Cout * Dg / (cross * 1e-6) / 1e12)
        print("%-14s cross product %8.2f ms (%5.1f TFLOP/s)" % (name, r["cross_ms"], r["cross_tflops"]))
    print("%-14s Gram %8.2f ms (%5.1f TFLOP/s)  sweep %8.2f ms (Cholesky %.2f ms %.2f TFLOP/s, assignment %.2f ms, "
          "GEMMs %.2f ms %.1f TFLOP/s, system %.2f ms)  call %.2f s  loss x%.3f after %d sweeps"
          % (name, r["gram_ms"], r["gram_tflops"], r["sweep_ms"], r["sweep_chol_ms"], r["chol_tflops"],
             r["sweep_assign_ms"], r["sweep_gemm_ms"], r["gemm_tflops"], r["sweep_system_ms"], wall, r["loss_ratio"],
             sweeps))
    del x, tg
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=3)
    ap.add_argument("--layers", nargs="*", default=list(LAYERS) + list(CONV_LAYERS))
    ap.add_argument("--target", action="store_true", help="time the target form (with the cross-product GEMM)")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--digest", action="store_true", help="print the sha256 of every layer's (ctrd, asmt, loss)")
    ap.add_argument("--root", default=ROOT, help="tree to load quantized-cnn_b200 (and its library) from")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "needs a GPU"
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    print("card: %s (name, power limit, max SM clock)" % card())
    print("library: %s" % q.LIB_PATH)
    results = []
    for name in args.layers:
        if name in CONV_LAYERS:
            results.append(time_conv(q, ctx, name, args.sweeps, args.target))
            continue
        Din, Dout, K, d, N = LAYERS[name]
        W = (np.random.default_rng(1).standard_normal((Dout, Din), dtype=np.float32) / np.float32(np.sqrt(Din)))
        g = torch.Generator(device="cuda").manual_seed(2)
        x = torch.randn((N, Din), generator=g, device="cuda", dtype=torch.float32)
        c0, a0, _ = q.pq_quantize_fc(ctx, W, K, d, iters=20, seed=3)
        if args.target:
            tg = x @ torch.from_numpy(W).cuda().T + 0.3 * torch.randn((N, Dout), generator=g, device="cuda")
            run = lambda xx, tt, s: q.pq_refine_fc_target(ctx, xx, tt, c0, a0, sweeps=s)
        else:
            tg = x
            run = lambda xx, tt, s: q.pq_refine_fc(ctx, W, xx, c0, a0, sweeps=s)
        run(x[:64], tg[:64], 1)   # warm-up: module load, smem opt-in
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, _, loss = run(x, tg, args.sweeps)
            torch.cuda.synchronize()
        ev = kernels(prof)
        gram = sum(t for n, _, t in ev if gemm_mode(n) == 1)
        cross = sum(t for n, _, t in ev if gemm_mode(n) == 2)
        ends = loss_ends(ev)
        sweeps, blk, trail = [], [], []
        for a, b in zip(ends[:-1], ends[1:]):
            part = ev[a + 1:b + 1]
            sweeps.append(sum(t for _, _, t in part))
            blk.append(sum(t for n, _, t in part if "pqr_block_kernel" in n))
            trail.append(sum(t for n, _, t in part if gemm_mode(n) == 0))
        t0 = time.perf_counter()
        res = run(x, tg, args.sweeps)
        wall = time.perf_counter() - t0
        sweep_ms = float(np.median(sweeps)) / 1e3
        gram_ms = gram / 1e3
        r = dict(layer=name, Din=Din, Dout=Dout, K=K, d=d, N=N, gram_ms=gram_ms,
                 gram_tflops=N * Din * (Din + 1) / (gram_ms * 1e-3) / 1e12, sweep_ms=sweep_ms,
                 sweep_block_kernel_ms=float(np.median(blk)) / 1e3, sweep_gemm_ms=float(np.median(trail)) / 1e3,
                 sweep_tflops=2.0 * Dout * Din * Din / (sweep_ms * 1e-3) / 1e12, call_wall_s=wall,
                 loss=[float(v) for v in loss], loss_ratio=float(loss[-1] / loss[0]), target=args.target,
                 digest=digest(res))
        if args.target:
            r.update(cross_ms=cross / 1e3, cross_tflops=2.0 * N * Din * Dout / (cross * 1e-6) / 1e12)
            print("%-12s cross product %8.2f ms (%5.1f TFLOP/s)" % (name, r["cross_ms"], r["cross_tflops"]))
        results.append(r)
        print("%-12s Gram %8.2f ms (%5.1f TFLOP/s)  sweep %8.2f ms (%5.1f TFLOP/s; block kernels %.2f ms, GEMMs %.2f ms)  "
              "call %.2f s  loss x%.3f after %d sweeps"
              % (name, gram_ms, r["gram_tflops"], sweep_ms, r["sweep_tflops"], r["sweep_block_kernel_ms"],
                 r["sweep_gemm_ms"], wall, r["loss_ratio"], args.sweeps))
        print("  loss trace: " + " ".join("%.6g" % v for v in loss))
        del x, tg
        torch.cuda.empty_cache()
    if args.digest:
        for r in results:
            print("digest %-14s %s" % (r["layer"], r["digest"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), sweeps=args.sweeps, results=results), f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
